"""--auto-carrier on the device: fsk_b200_rx_batch_auto / _s16 (the per-candidate rx kernel with a tone
table per stream and the carrier scan) against the FLAT auto oracle (oracle/auto_oracle.c), whose LITERAL
twin tests/test_auto_carrier_cpu.py pins to the reference CLI.

Every AUTO_COMBOS instance of minimodem_b200/csrc/fsk_b200_kernels.cu runs, float and int16, on random
streams that each carry their own tone pairs, behind silent lead-ins, with a gap that drops the carrier
and a second transmission on other tones.  Every stream is screened first (autoorc.screen): a scan decision
within 1e-5 (relative) of a tie -- its two largest band magnitudes, or its largest and the threshold -- or a
frame search that tests/tie_screen.py's perturbed runs can tip marks the stream as not robust.  Robust
streams must give the oracle's records and bands exactly (confidences within the usual bar).

SCAN_TIE rests on test_band_decisions_match_a_float64_dft: every consumer of band_mag (FskPlan.detect_carrier,
detect_carrier_batch and the scan inside the rx loop, float and int16 rows) takes a float64 DFT's decision
between two bands 2e-6 apart, in every lane placement of every AUTO_COMBOS instance, at the exact threshold
and on a tie of every band."""
import zlib

import numpy as np
import pytest

import autoorc
import golden_util as gu
import orc
import refcases
from gpudev import dev, mm, pcm, rows, sync, torch, upload
from rxcases import COVER, KEYS, auto_combos, live_records, records_of, tone_stream
from rxfam import as_oracle_frames, compare_frames, compare_reports, reports_of


PRESETS = ["rtty", "tdd", "callerid", "uic-train", "uic-ground", "V.21", "2400", "1200", "600", "300", "110"]


def test_the_cover_table_is_the_auto_combo_list():
    assert set(COVER) == auto_combos()


_CASES = {}


def auto_case(mode, rate, inverted=False):
    """3..6 random streams of one mode (computed once): lead-ins of up to two sample rings, one or two
    transmissions on their own tone pairs with a gap between, low noise; with the FLAT oracle's
    result and the screen's verdict per stream: (mode, streams, [(want, robust)])."""
    key = (mode, rate) + ((True,) if inverted else ())
    if key in _CASES:
        return _CASES[key]
    m = orc.Mode(mode, sample_rate=rate)
    d = m.derived()
    S = int(d.samplebuf_size)
    spb = float(d.nsamples_per_bit)
    b_shift = autoorc.b_shift(m, inverted)
    nbands = int((rate + float(m.band_width) / 2) / float(m.band_width)) // 2 + 1
    rng = np.random.default_rng(zlib.crc32(repr(key).encode()))
    streams = []
    for s in range(int(rng.integers(3, 7))):
        parts = [np.zeros(int(rng.integers(0, 2 * S)), np.float32), tone_stream(rng, m, b_shift, nbands, 6)]
        if s % 2 == 0:
            parts += [np.zeros(int(rng.uniform(30, 50) * spb), np.float32), tone_stream(rng, m, b_shift, nbands, 5)]
        parts.append(np.zeros(int(rng.integers(0, S)), np.float32))
        x = np.concatenate(parts)
        x = (x + np.float32(1e-4) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
    screened = [autoorc.screen(m, x, inverted) for x in streams]
    _CASES[key] = (m, streams, screened)
    return _CASES[key]


def engine(mode, rate):
    e = mm().RxEngine.for_mode(mode, rate)
    e.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    return e


def run_auto(eng, buf, n, lens, states=None, auto_states=None):
    t = torch()
    frames, st, ast, bands = eng.rx_batch_auto(upload(buf), nsamples=n,
                                               nsamples_each=upload(lens), states=states,
                                               auto_states=auto_states, rec_band=True)
    sync()
    return frames, st, ast, bands


def check_against_oracle(screened, fr, st, bands, what):
    """rxfam.check_against_oracle's record and report checks on the robust streams, plus each record's band;
    kept apart on purpose: the auto call's screen (autoorc.screen) has no frame-count bar for the streams it
    screens out, and it may screen out one stream of a case, not half"""
    nok = 0
    for s, (w, robust) in enumerate(screened):
        if not robust:
            continue
        nok += 1
        k = int(st["nframes"][s])
        recs = fr[s, :k]
        compare_frames(as_oracle_frames(recs), w["frames"], "%s stream %d" % (what, s))
        compare_reports(reports_of(recs, st[s]), w["reports"], "%s stream %d" % (what, s))
        got_f = [int(b) for r, b in zip(recs, bands[s, :k]) if int(r["frame_start"]) != mm().FRAME_REPORT]
        got_r = [int(b) for r, b in zip(recs, bands[s, :k]) if int(r["frame_start"]) == mm().FRAME_REPORT]
        assert got_f == w["frame_band"], (what, s, got_f, w["frame_band"])
        assert got_r == w["report_band"][:len(got_r)], (what, s, got_r, w["report_band"])
    assert nok >= len(screened) - 1, (what, "screened out", len(screened) - nok)


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_auto_instance_matches_the_flat_oracle(key):
    """Float rows: every auto instance gives the FLAT oracle's records and bands."""
    mode, rate = COVER[key]
    m, streams, screened = auto_case(mode, rate)
    want = [w for w, _ in screened]
    assert sum(len(w["frames"]) for w in want) > 0 and any(len(set(w["report_band"])) > 1 for w in want)
    eng = engine(mode, rate)
    buf, n = rows(streams, np.float32, 4)
    lens = np.array([len(a) for a in streams], np.int32)
    frames, states, ast, bands = run_auto(eng, buf, n, lens)
    G, W, L = key
    assert "k_rx_auto<G=%d,W=%d,L=%d," % (G, W, L) in eng.last_kernel() and "src=f32" in eng.last_kernel()
    st = mm().states_to_numpy(states)
    assert (st["done"] == 1).all()
    check_against_oracle(screened, mm().frames_to_numpy(frames), st, bands.cpu().numpy(), str(key))


@pytest.mark.gpu
def test_inverted_negates_the_band_shift():
    """--inverted: the space band lies b_shift below the mark band (src/minimodem.c:1204-1205)."""
    m, streams, screened = auto_case("1200", 48000, inverted=True)
    assert sum(len(w["frames"]) for w, _ in screened) > 0
    eng = mm().RxEngine.for_mode("1200", 48000, inverted=True)
    eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD, inverted=True)
    buf, n = rows(streams, np.float32, 4)
    frames, states, ast, bands = run_auto(eng, buf, n, np.array([len(a) for a in streams], np.int32))
    st = mm().states_to_numpy(states)
    check_against_oracle(screened, mm().frames_to_numpy(frames), st, bands.cpu().numpy(), "inverted")


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_auto_instance_int16_rows_equal_the_float_rows(key):
    """int16 rows: the same records, states and bands as the float path on s16/32768, bit for bit, in one
    pass and resumed from position 13 with a fresh auto state."""
    mode, rate = COVER[key]
    m, streams, _ = auto_case(mode, rate)
    eng = engine(mode, rate)
    p16 = [pcm(a) for a in streams]
    b16, n = rows(p16, np.int16, 8)
    b32, _ = rows([a.astype(np.float32) * np.float32(1.0 / 32768.0) for a in p16], np.float32, 8)
    lens = np.array([len(a) for a in streams], np.int32)
    for resume in (0, 13):
        t = torch()
        outs = []
        for b in (b32, b16):
            st0 = np.zeros(len(streams), mm().STATE_DTYPE)
            st0["pos"][:] = resume
            states = upload(st0.view(np.int32).reshape(len(streams), -1).copy())
            outs.append(run_auto(eng, b, n, lens, states=states))
            G, W, L = key
            assert "k_rx_auto<G=%d,W=%d,L=%d," % (G, W, L) in eng.last_kernel()
        assert "src=s16" in eng.last_kernel()
        (fa, sa, aa, ba), (fb, sb, ab, bb) = outs
        sa, sb = mm().states_to_numpy(sa), mm().states_to_numpy(sb)
        assert sa.tobytes() == sb.tobytes() and aa.cpu().numpy().tobytes() == ab.cpu().numpy().tobytes(), key
        fa, fb = mm().frames_to_numpy(fa), mm().frames_to_numpy(fb)
        ba, bb = ba.cpu().numpy(), bb.cpu().numpy()
        for s in range(len(streams)):
            k = int(sa["nframes"][s])
            assert fa[s, :k].tobytes() == fb[s, :k].tobytes() and (ba[s, :k] == bb[s, :k]).all(), (key, s, resume)
        assert sa["nframes"].sum() >= len(streams)


@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_auto_state_carries_a_stream_across_calls(key, src):
    """A stream continued mid-way -- every call stops after 3 records and the next one resumes from the
    saved stream state and auto state (carrier band, ring count) -- gives the records and bands of one
    pass, bit for bit."""
    mode, rate = COVER[key]
    m, streams, _ = auto_case(mode, rate)
    eng = engine(mode, rate)
    t = torch()
    if src == "s16":
        buf, n = rows([pcm(a) for a in streams], np.int16, 8)
    else:
        buf, n = rows(streams, np.float32, 4)
    lens = np.array([len(a) for a in streams], np.int32)
    whole = records_of(*(lambda r: (r[0], r[1], r[3]))(run_auto(eng, buf, n, lens)))
    x = upload(buf)
    each = upload(lens)
    states = t.zeros((len(streams), mm().STATE_WORDS), dtype=t.int32).to(dev())
    auto = t.zeros((len(streams), mm().AUTO_STATE_BYTES), dtype=t.uint8).to(dev())
    got = [[] for _ in streams]
    for call in range(10000):
        frames, states, auto, bands = eng.rx_batch_auto(x, nsamples=n, nsamples_each=each, max_frames=3,
                                                        states=states, auto_states=auto, rec_band=True)
        sync()
        for s, r in enumerate(records_of(frames, states, bands)):
            got[s] += r
        st = mm().states_to_numpy(states)
        if (st["done"] == 1).all():
            break
        assert "src=%s" % src in eng.last_kernel()
        st["nframes"][:] = 0
        states = upload(st.view(np.int32).reshape(len(streams), -1).copy())
    assert call >= 2 and got == whole, (key, src)


@pytest.mark.gpu
def test_a_stream_on_the_configured_tones_gives_the_fixed_tone_records():
    """A stream that acquires at its first scan on the engine's own bands and never drops it decodes
    exactly as fsk_b200_rx_batch does: same records, bit for bit.  (The scan finds a Bell202 mark tone of
    1200 Hz in band 5, its window being one bit long; the engine is set to bands 5 and 5 + b_shift.)"""
    m = orc.Mode("1200", sample_rate=48000)
    rng = np.random.default_rng(11)
    words = rng.integers(0, 256, 40, dtype=np.uint64).astype(np.uint32)
    x = orc.tx_words(m, words, 0.8, 4096, True)
    assert autoorc.rx_run(m, x)["frame_band"] == [5] * 40 and autoorc.b_shift(m) == 4
    eng = mm().RxEngine.for_mode("1200", 48000, f_mark=1000.0, f_space=1800.0)
    eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    assert (eng.params.b_mark, eng.params.b_space) == (5, 9)
    buf, n = rows([x] * 4, np.float32, 4)
    lens = np.full(4, n, np.int32)
    fa, sa, ast, bands = run_auto(eng, buf, n, lens)
    auto_kernel = eng.last_kernel()
    t = torch()
    fb, sb = eng.rx_batch(upload(buf), nsamples=n)
    sync()
    assert eng.last_kernel().split("<")[1].split(",mode")[0] in auto_kernel, (eng.last_kernel(), auto_kernel)
    sa, sb = mm().states_to_numpy(sa), mm().states_to_numpy(sb)
    fa, fb = mm().frames_to_numpy(fa), mm().frames_to_numpy(fb)
    assert (bands.cpu().numpy()[:, :int(sa["nframes"][0])] == eng.params.b_mark).all()
    for s in range(4):
        k = int(sb["nframes"][s])
        assert k == int(sa["nframes"][s]) and k >= 40
        assert fa[s, :k].tobytes() == fb[s, :k].tobytes(), s


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cli-auto-carrier", "cli-auto-carrier-rtty"])
def test_cli_auto_carrier_vectors_decode_on_the_device(name):
    """The reference CLI's own --auto-carrier runs (tests/golden): the device's records decode to its
    stdout, and its CARRIER lines name the bands the device reports."""
    case = refcases.BY_NAME[name]
    g = gu.load(name)
    _, rx = gu.modes(case)
    a = gu.audio(case, g)
    eng = engine(case["rx_mode"], case["rx_mkw"].get("sample_rate", 48000))
    buf, n = rows([a], np.float32, 4)
    frames, states, ast, bands = run_auto(eng, buf, n, np.array([n], np.int32))
    fr, st = mm().frames_to_numpy(frames), mm().states_to_numpy(states)
    k = int(st["nframes"][0])
    recs = [r for r in fr[0, :k] if int(r["frame_start"]) != mm().FRAME_REPORT]
    assert orc.ref_decode(rx, as_oracle_frames(recs)) == bytes(g["stdout"])
    res = {"frames": as_oracle_frames(recs), "frame_band": [int(b) for r, b in zip(fr[0, :k], bands.cpu().numpy()[0, :k])
                                                              if int(r["frame_start"]) != mm().FRAME_REPORT]}
    want = [ln.strip() for ln in bytes(g["stderr"]).decode().splitlines() if ln.startswith("### CARRIER")]
    got = [autoorc.carrier_line(rx, b) for f, b in zip(res["frames"], res["frame_band"]) if f[4]]
    assert got == want


@pytest.mark.gpu
def test_live_stream_records_do_not_depend_on_the_cut():
    """Live streams with auto-carrier: the records and bands do not depend on how the streams are cut,
    and equal those of one call over the whole streams; LiveReceiver(auto_carrier=...) prints the same
    text for every cut, the FLAT oracle's on the robust streams."""
    from minimodem_b200.serving import LiveReceiver
    t = torch()
    mode, rate = "1200", 48000
    m, streams, screened = auto_case(mode, rate)
    eng = engine(mode, rate)
    buf, n = rows(streams, np.float32, 4)
    r = run_auto(eng, buf, n, np.array([len(a) for a in streams], np.int32))
    whole = records_of(r[0], r[1], r[3])
    for cut in (997, 4096, 20000):
        assert live_records(engine(mode, rate), streams, cut) == whole, cut
    buf, n = rows(streams, np.float32, 4)
    lens = np.array([len(a) for a in streams], np.int64)
    outs = []
    for cut in (997, 4096, 20000):
        lr = LiveReceiver(mode, rate, len(streams), max_chunk=cut, device=dev(), auto_carrier=autoorc.DEFAULT_THRESHOLD)
        texts = [b""] * len(streams)

        def take(res):
            text, counts = res
            text, counts = text.cpu().numpy(), counts.cpu().numpy()
            return [texts[s] + text[s, :counts[s]].tobytes() for s in range(len(streams))]
        for o in range(0, n, cut):
            w = min(cut, n - o)
            chunk = upload(np.ascontiguousarray(buf[:, o:o + w]))
            valid = upload(np.clip(lens - o, 0, w).astype(np.int32))
            texts = take(lr.feed(chunk, valid))
        texts = take(lr.finish())
        outs.append(texts)
    assert outs[0] == outs[1] == outs[2]
    for s, (w, robust) in enumerate(screened):
        if robust:
            assert outs[0][s] == orc.ref_decode(m, w["frames"]), s


@pytest.mark.gpu
def test_every_preset_runs_and_the_errors_launch_nothing():
    """Every preset of fsk_b200_rx_config_for_mode at 8 and 48 kHz runs with auto-carrier.  Errors, and no
    launch: SAME (band shift 0, where the reference asserts), a data rate above the sample rate (a scan
    window under one sample, where the reference's scan never advances), 0.5 baud (no per-candidate
    kernel)."""
    t = torch()
    x = t.zeros((2, 4096), dtype=t.float32).to(dev())
    for rate in (8000, 48000):
        for p in PRESETS:
            eng = engine(p, rate)
            eng.rx_batch_auto(x, nsamples=4096)
            assert "k_rx_auto<" in eng.last_kernel(), (p, rate)
        fast = mm().RxEngine.for_mode("12000", 8000, f_mark=1200.0, f_space=2200.0, band_width=100.0)
        fast.rx_batch(x, nsamples=4096)             # the fixed-tone loop takes this mode
        n0 = mm().launch_count()
        e = mm().RxEngine.for_mode("same", rate)
        with pytest.raises(RuntimeError, match="-22"):
            e.set_auto_carrier(0.001)
        with pytest.raises(RuntimeError, match="-22"):
            e.rx_batch_auto(x, nsamples=4096)
        e = fast
        with pytest.raises(RuntimeError, match="-22"):
            e.set_auto_carrier(0.001)
        with pytest.raises(RuntimeError, match="-22"):
            e.rx_batch_auto(x, nsamples=4096)
        e = mm().RxEngine.for_mode("0.5", rate)
        e.set_auto_carrier(0.001)
        for bad in (0.0, -1.0, float("inf"), float("nan")):
            with pytest.raises(RuntimeError, match="-22"):
                e.set_auto_carrier(bad)
        with pytest.raises(RuntimeError, match="-22"):     # a failed set_auto_carrier disables the calls
            e.rx_batch_auto(x, nsamples=4096)
        e.set_auto_carrier(0.001)
        with pytest.raises(RuntimeError, match="-95"):
            e.rx_batch_auto(x, nsamples=4096)
        assert mm().launch_count() == n0


# ---------------------------------------------------------------------------------------------------
# band decisions against a float64 DFT: every consumer of band_mag
# ---------------------------------------------------------------------------------------------------
EPSILONS = (2e-6, -2e-6, 1e-5, -1e-5, 1e-4, -1e-4)


class Window:
    """one preset's carrier-scan window: n samples zero-padded to fftsize F, bands 1 .. nbands-1; G the lanes
    of its AUTO_COMBOS instance; L = ceil(nsamples_per_scan), the shortest stream whose scan reads it"""

    def __init__(self, key):
        self.key = key
        self.mode, self.rate = COVER[key]
        self.G = key[0]
        m = orc.Mode(self.mode, sample_rate=self.rate)
        p = mm().rx_params(mm().rx_config_for_mode(self.mode, self.rate))
        self.F, self.nbands = int(p.fftsize), int(p.nbands)
        sf = np.float32(min(np.float32(m.derived().nsamples_per_bit), np.float32(self.F)))
        self.n, self.L = int(sf), int(np.ceil(sf))
        self.b_shift = autoorc.b_shift(m)
        self.m = m
        k = np.arange(self.nbands)[:, None] * np.arange(self.n)[None, :] % self.F
        self.w = np.exp(-2j * np.pi * k / self.F)          # [band, sample], exact integer phase

    def mags(self, x):
        """float64 band magnitudes of the exact samples x[:n], band_mag's scale (2 / n); band 0 is -1"""
        m = np.abs(self.w @ np.asarray(x[:self.n], np.float64)) * (2.0 / self.n)
        m[0] = -1.0
        return m

    def accepts(self, b):
        return 1 <= b + self.b_shift < self.nbands

    def placements(self):
        """(name, k1, k2): the two bands in one lane of a group (k2 = k1 + G), in neighbouring lanes, across the
        G-lane group (lane G-1, then lane 0), and, for the warp-wide scan of detect_carrier_batch, in one lane
        of the 32-lane stride and across it; both bands accepted by the scan"""
        lo = max(1, 1 - self.b_shift)
        hi = min(self.nbands - 1, self.nbands - 1 - self.b_shift)
        mid = (lo + hi) // 2
        G = self.G
        want = [("same-lane", mid - G // 2, mid - G // 2 + G), ("neighbour-lanes", mid, mid + 1),
                ("across-group", (mid // G) * G, (mid // G) * G + 1), ("same-lane-32", mid - 16, mid + 16),
                ("across-32", 32, 33), ("across-32", 64, 65)]
        return [(nm, a, b) for nm, a, b in want if lo <= a < b <= hi]

    def duel(self, rng, k1, k2, eps, s16):
        """x [L] float32 (s16: int16) whose window's float64 magnitudes have bands k1 and k2 on top, |k2| / |k1| - 1
        within 10 % of eps, and every other band below both by more than 1e-3 of them; (x, the eps it has)"""
        i = np.arange(self.n)
        q = 1.0 / 32768.0
        for _ in range(64):
            p1, p2 = rng.uniform(0, 2 * np.pi, 2)
            build = lambda a2: 0.4 * np.cos(2 * np.pi * (k1 * i % self.F) / self.F + p1) + \
                a2 * np.cos(2 * np.pi * (k2 * i % self.F) / self.F + p2)
            r = lambda a2: (lambda mg: mg[k2] / mg[k1] - 1.0)(self.mags(build(a2)))
            lo, hi = 0.05, 0.55             # |x| < 1: int16 holds it
            if not r(lo) < eps < r(hi):
                continue
            for _ in range(80):
                mid = (lo + hi) / 2
                lo, hi = (mid, hi) if r(mid) < eps else (lo, mid)
            x = build((lo + hi) / 2)
            x = np.round(x / q).astype(np.float64) * q if s16 else x.astype(np.float32).astype(np.float64)
            # single-step nudges (one LSB or one ulp of one sample) toward eps
            D1, D2 = self.w[k1] @ x, self.w[k2] @ x
            for _ in range(200):
                e = abs(D2) / abs(D1) - 1.0
                if abs(e - eps) <= 0.05 * abs(eps):
                    break
                step = np.full(self.n, q) if s16 else np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)
                cand = []
                for sgn in (1.0, -1.0):
                    d1 = D1 + sgn * step * self.w[k1]
                    d2 = D2 + sgn * step * self.w[k2]
                    cand.append(np.abs(np.abs(d2) / np.abs(d1) - 1.0 - eps))
                cand = np.array(cand)
                j = np.unravel_index(np.argmin(cand), cand.shape)
                if cand[j] >= abs(e - eps):
                    break
                sgn = 1.0 if j[0] == 0 else -1.0
                x[j[1]] += sgn * step[j[1]]
                D1, D2 = self.w[k1] @ x, self.w[k2] @ x
            mg = self.mags(x)
            e = mg[k2] / mg[k1] - 1.0
            others = np.delete(mg, [0, k1, k2])
            if abs(e - eps) <= 0.1 * abs(eps) and others.max() < (1 - 1e-3) * min(mg[k1], mg[k2]) \
                    and min(mg[k1], mg[k2]) > 10 * autoorc.DEFAULT_THRESHOLD:
                out = np.zeros(self.L, np.float64)
                out[:self.n] = x
                if s16:
                    return np.round(out * 32768).astype(np.int16), e
                return out.astype(np.float32), e
        raise AssertionError(("no duel", self.key, k1, k2, eps))

    def impulse(self, a, s16=False):
        x = np.zeros(self.L, np.int16 if s16 else np.float32)
        x[0] = a
        return x

    def threshold_amplitude(self):
        """the float32 a > 0 with fl(a * magscalar) == threshold exactly (magscalar = 1 / (n / 2), src/fsk.c:553),
        or None; an impulse of a at the window start gives every band that magnitude"""
        ms = np.float32(1) / (np.float32(self.n) / np.float32(2))
        thr = np.float32(autoorc.DEFAULT_THRESHOLD)
        a = np.float32(thr / ms)
        for k in range(-64, 65):
            b = np.float32(a + np.float32(k) * np.spacing(a))
            if np.float32(b * ms) == thr:
                return b
        return None


WINDOWS = {}


def window(key):
    if key not in WINDOWS:
        WINDOWS[key] = Window(key)
    return WINDOWS[key]


def band_cases(key):
    """[(name, x float32 [L] or int16, the float64 decision: a band or -1, the band decision's eps or None)] of
    one preset: every placement at every eps (float32 and int16 samples), the exact threshold and 2e-6 either
    side, and the tie of every band (an impulse at the window start)"""
    w = window(key)
    rng = np.random.default_rng(zlib.crc32(repr(("duels",) + key).encode()))
    out = []
    for nm, k1, k2 in w.placements():
        for eps in EPSILONS:
            for s16 in (False, True):
                x, e = w.duel(rng, k1, k2, eps, s16)
                out.append(("%s %d/%d eps=%g%s" % (nm, k1, k2, eps, " s16" if s16 else ""), x, k2 if e > 0 else k1, e))
    a = w.threshold_amplitude()
    if a is not None:
        out.append(("threshold", w.impulse(a), 1, None))
        out.append(("threshold-2e-6", w.impulse(np.float32(a * np.float32(1 - 2e-6))), -1, None))
        out.append(("threshold+2e-6", w.impulse(np.float32(a * np.float32(1 + 2e-6))), 1, None))
    # every band at fl(|a| magscalar): band 1 where that reaches the threshold
    ms = np.float32(1) / (np.float32(w.n) / np.float32(2))
    tie = lambda a: 1 if np.float32(np.float32(a) * ms) >= np.float32(autoorc.DEFAULT_THRESHOLD) else -1
    out.append(("tie", w.impulse(0.875), tie(0.875), None))
    out.append(("tie s16", w.impulse(28672, s16=True), tie(0.875), None))
    return out


def widened(x):
    return x.astype(np.float32) * np.float32(1.0 / 32768.0) if x.dtype == np.int16 else x


def scan_band(w, want):
    """what the scan leaves in the auto state for the float64 decision `want`: the band if the scan accepts it, 0
    for none or a rejected band"""
    return want if want > 0 and w.accepts(want) else 0


def test_band_cases_are_what_they_claim():
    """The duels' float64 winners and margins, the exact threshold (every band's float32 magnitude equals it),
    the tie; and the auto oracle's scan (its scan log) takes the float64 decision on every one."""
    nthr = 0
    for key in KEYS:
        w = window(key)
        assert w.placements(), key
        for name, x, want, e in band_cases(key):
            y = widened(x)
            mg = w.mags(y)
            if e is not None:
                assert int(np.argmax(mg)) == want, (key, name)
            elif name.startswith("threshold"):
                nthr += 1
                ms = np.float32(1) / (np.float32(w.n) / np.float32(2))
                got = np.float32(abs(np.float32(y[0])) * ms)
                thr = np.float32(autoorc.DEFAULT_THRESHOLD)
                assert (got == thr) if name == "threshold" else (got < thr) == name.endswith("-2e-6"), (key, name)
            r = autoorc.rx_run(w.m, y, scans=True)
            assert r["scans"][0]["band"] == want and r["scans"][0]["window"] == (0 if want > 0 else 1), (key, name)
        if w.nbands > 33:
            assert any(nm.startswith("across-32") for nm, _, _ in w.placements()), key
    assert nthr >= 3 * (len(KEYS) - 1), nthr
    assert any(window(k).nbands > 32 for k in KEYS) and any(window(k).b_shift < 0 for k in KEYS)


@pytest.mark.ref
def test_the_reference_fft_ties_every_band_on_an_impulse():
    """The reference's own fsk_detect_carrier (oracle/_ref) on the impulse windows: the tie and the exact
    threshold pick band 1, 2e-6 below the threshold nothing."""
    import ctypes as C
    fn = orc.ref().fsk_detect_carrier
    fn.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_uint, C.c_float]
    fn.restype = C.c_int
    for key in KEYS:
        w = window(key)
        rp = orc.RefPlan(w.rate, w.m.mark_f, w.m.space_f, w.m.band_width)
        for name, x, want, e in band_cases(key):
            if e is None:
                y = np.ascontiguousarray(widened(x)[:w.n])
                assert fn(rp.h, orc.fptr(y), w.n, autoorc.DEFAULT_THRESHOLD) == want, (key, name)


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_band_decisions_match_a_float64_dft(key):
    """Every consumer of band_mag takes the float64 DFT's decision: FskPlan.detect_carrier (k_band_mags),
    detect_carrier_batch (k_detect_carrier) and the scan of rx_batch_auto on float and int16 rows (detect_group;
    the stream is shorter than a frame, so the loop scans once and stops, its decision in the auto state) --
    on duels of two bands eps apart, the exact threshold and the tie of every band."""
    w = window(key)
    cases = band_cases(key)
    t = torch()
    plan = mm().FskPlan(w.rate, float(w.m.mark_f), float(w.m.space_f), float(w.m.band_width))
    assert (plan.fftsize, plan.nbands) == (w.F, w.nbands)
    eng = engine(w.mode, w.rate)
    bad = []
    fl = [(nm, widened(x), want, e) for nm, x, want, e in cases]
    buf, _ = rows([x for _, x, _, _ in fl], np.float32, 4)
    got_b = mm().detect_carrier_batch(w.F, upload(buf), w.n, autoorc.DEFAULT_THRESHOLD).cpu().numpy()
    for i, (nm, x, want, e) in enumerate(fl):
        got = plan.detect_carrier(np.ascontiguousarray(x[:w.n]), autoorc.DEFAULT_THRESHOLD)
        if got != want:
            bad.append(("detect_carrier", nm, e, got, want))
        if int(got_b[i]) != want:
            bad.append(("detect_carrier_batch", nm, e, int(got_b[i]), want))
    for src in ("f32", "s16"):
        sub = [(nm, x, want, e) for nm, x, want, e in cases if (x.dtype == np.int16) == (src == "s16")]
        xs = [x for _, x, _, _ in sub]
        buf, _ = rows(xs, xs[0].dtype, 8)
        lens = np.full(len(xs), w.L, np.int32)
        _, st, ast, _ = run_auto(eng, buf, w.L, lens)
        assert "k_rx_auto<G=%d,W=%d,L=%d," % key in eng.last_kernel() and "src=%s" % src in eng.last_kernel()
        assert (mm().states_to_numpy(st)["nframes"] == 0).all()
        band = ast.cpu().numpy().view(np.uint32)[:, 0]
        for (nm, x, want, e), b in zip(sub, band):
            if int(b) != scan_band(w, want):
                bad.append(("scan " + src, nm, e, int(b), scan_band(w, want)))
    plan.destroy()
    eps = [abs(b[2]) for b in bad if b[2] is not None]
    print("%s: %d decisions, %d disagree with the float64 DFT; smallest |eps| disagreeing: %s" % (
        key, 3 * len(cases), len(bad), "%.2g" % min(eps) if eps else "none"))
    assert not bad, bad[:8]
