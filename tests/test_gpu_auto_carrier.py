"""--auto-carrier on the device: fsk_b200_rx_batch_auto / _s16 (the per-candidate rx kernel with a tone
table per stream and the carrier scan) against the FLAT auto oracle (oracle/auto_oracle.c), whose LITERAL
twin tests/test_auto_carrier_cpu.py pins to the reference CLI.

Every AUTO_COMBOS instance of minimodem_b200/csrc/fsk_b200_kernels.cu runs, float and int16, on random
streams that each carry their own tone pairs, behind silent lead-ins, with a gap that drops the carrier
and a second transmission on other tones.  Every stream is screened first (autoorc.screen): a scan decision
within 1e-5 (relative) of a tie -- its two largest band magnitudes, or its largest and the threshold -- or a
frame search that tests/tie_screen.py's perturbed runs can tip marks the stream as not robust.  Robust
streams must give the oracle's records and bands exactly (confidences within the usual bar); the device's
band magnitudes are the fsk_b200_detect_carrier_batch ones, within about 1e-6 of the oracle's."""
import zlib

import numpy as np
import pytest

import autoorc
import golden_util as gu
import orc
import refcases
from gpudev import dev, mm, pcm, rows, sync, torch, upload
from rxcases import COVER, KEYS, auto_combos, tone_stream
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


def records_of(frames, states, bands):
    """per stream: [(record bytes, band)] of the records a call wrote"""
    fr, st, b = mm().frames_to_numpy(frames), mm().states_to_numpy(states), bands.cpu().numpy()
    return [[(fr[s, i].tobytes(), int(b[s, i])) for i in range(int(st["nframes"][s]))] for s in range(len(st))]


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


def live_records(mode, rate, streams, cut):
    """The live-stream recipe of include/fsk_b200.h with auto-carrier: fsk_b200_stream_push, then
    fsk_b200_rx_batch_auto with the auto holdback, chunk by chunk; the holdback off for the last call.
    Returns every stream's records and bands in order."""
    t = torch()
    eng = engine(mode, rate)
    window = eng.auto_stream_window()
    eng.set_holdback(window)
    stride = (window + eng.params.frame_nsamples + cut + 3) & ~3
    max_frames = eng.max_frames(stride)
    S = len(streams)
    buf, n = rows(streams, np.float32, 4)
    lens = np.array([len(a) for a in streams], np.int64)
    z = lambda shape, dt: t.zeros(shape, dtype=dt).to(dev())
    rows_, fill = z((S, stride), t.float32), z((S,), t.int32)
    states, auto = z((S, mm().STATE_WORDS), t.int32), z((S, mm().AUTO_STATE_BYTES), t.uint8)
    dropped = z((S,), t.int32)
    got = [[] for _ in streams]

    def step(chunk, valid):
        mm().stream_push(rows_, fill, states, chunk, valid, dropped=dropped)
        frames, _, _, bands = eng.rx_batch_auto(rows_, nsamples=stride, nsamples_each=fill, max_frames=max_frames,
                                                states=states, auto_states=auto, rec_band=True)
        sync()
        for s, r in enumerate(records_of(frames, states, bands)):
            got[s] += r
    for o in range(0, n, cut):
        w = min(cut, n - o)
        step(upload(np.ascontiguousarray(buf[:, o:o + w])),
             upload(np.clip(lens - o, 0, w).astype(np.int32)))
    eng.set_holdback(0)
    step(z((S, 4), t.float32), 0)
    assert int(dropped.cpu().numpy().sum()) == 0
    return got


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
        assert live_records(mode, rate, streams, cut) == whole, cut
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
