"""Samples outside well-behaved audio: NaN, +-inf, clicks far above the signal, clipped int16 full scale,
streams scaled towards the fp32 overflow of a bin and down to subnormal values.

What the unmodified reference does with them (test_oracle_find_frame_is_the_reference_on_bad_samples, on
every find_frame call of clean streams, with the bad samples put into the call's own windows):
- A window that holds a NaN has NaN in both tone bins, whatever the FFT, so `mag_mark > mag_space` is false:
  a required '1' rejects the candidate (src/fsk.c:211) and otherwise its confidence is NaN, which never wins
  `best_c < c` (:492).  The oracle's direct sums give the same: a NaN costs exactly the candidates whose
  windows hold it, and the search's bits, frame start and confidence are the reference's.
- A window that holds +-inf has a non-finite value in both bins; which one (inf, or NaN where a twiddle is
  exactly 0 or a butterfly forms inf - inf) depends on the transform.  Both are implementation-independent in
  one respect only: the bit reads as a space and the confidence is 0 or NaN, so the candidate is never chosen.
  The bars below rest on that alone, and the search results then agree exactly.
- A click of 1e17 and more in a window swamps the reference's float FFT: its rounding decides the other bins
  there, and its choice among the candidates that hold the click differs from the oracle's.  Every such
  candidate stays below the confidence threshold in both (a lone impulse puts the same magnitude into the mark
  and the space bin, so its SNR is about 1), and the rx loop only acts on a confidence above the threshold
  (src/minimodem.c:1292), so the records do not depend on it.  A click of 1e4 gives the reference's result.
- Subnormal and 1e-20-scale windows: every off-tone magnitude is below FLT_EPSILON, so the confidence is the
  `inf` class in both, with the same bits and frame start.

The kernels against the oracle's FLAT rx loop, on every rx launch family (test_bad_samples_in_every_family):
clean and noisy streams with every kind of bad sample at every place.  Float rows: a NaN, a NaN burst of one
bit period, one +inf or -inf, clicks of 1e4 and 1e30; int16 rows: full-scale clicks and a full-scale burst.
The places: inside a frame's window; ending three samples before a window (the same lane-run of the prefix
table); in the first window of the lowest candidate of a fine search (the call without a search limit,
src/minimodem.c:1357-1389), which that window loses at the sliding search's first step; in the stop bit (the
pass-1 reject); in the lead-in (two bit windows before the first frame, or, for the auto call, the last half
bit of its silent lead-in, which the carrier scan reads).  Streams are screened with tests/tie_screen.py: a
robust stream must give the oracle's records and session reports, a screened-out one the frame count within
one.  The clean streams of the same launch must give the records of a launch whose other rows are clean.
This found two bugs.  The prefix table took a window as a difference of prefix values, so a NaN, inf or loud
click earlier in the same lane-run spoilt windows that do not hold it (an -inf three samples ahead of an RTTY
frame lost the frame).  The sliding fine search kept a NaN, inf or click that had left a window in that
window's sums, so a NaN in its lowest candidate kept the coarse frame start where the reference refines.

The fp32 bin overflow of DESIGN.md 5 item 4 is pinned by value (test_scaled_streams_stop_decoding_at_the_
documented_bound and its reference twin).  int16 rows at full scale equal the float path on the widened rows
in every int16 family, the host-slab call and LiveReceiver(pcm16=True).  LiveReceiver (plain, tones=,
channels_per_row=2, auto_carrier=) fed the poisoned streams in random chunks, with a cut inside every NaN
burst, prints the text of one rx pass over the same rows, and every poisoned stream keeps decoding.

The CPU test runs the `gpu` tests of this file on the host SIMT emulation of the kernels (tests/emu); the
TMA bulk fill is not modelled there and its row is skipped."""
import zlib

import numpy as np
import pytest

import autoorc
import orc
import rxfam
import tie_screen
import gpudev
from gpudev import dev, mm, pcm, records, sync, torch, upload, widen
from rxcases import check_channels_against_oracle, live_text, on_pair, one_pass_text, random_pair, run_channels
from rxfam import as_oracle_frames, compare_frames, compare_reports, reports_of

f32 = np.float32
NAN, INF = f32(np.nan), f32(np.inf)


# --------------------------------------------------------------------------------------------------
# CPU
# --------------------------------------------------------------------------------------------------
def test_sample_domain_file_on_the_emulated_kernels():
    """The `gpu` tests below on the host SIMT emulation of the kernels (the TMA bulk fill excepted)."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 3000, module="test_gpu_sample_domain.py")
    assert " passed" in tail and "failed" not in tail


def clean_stream(m, seed, nwords=8, amplitude=0.7):
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
    lead = np.zeros(int(3 * m.derived().nsamples_per_bit), np.float32)
    return np.concatenate([lead, orc.tx_words(m, words, amplitude, 4096, True)])


def windows(t, spb, n):
    """the bit windows [begin, end) of the candidate at t (src/fsk.c:183, :205)"""
    bn = int(f32(spb + f32(0.5)))
    return [(t + int(f32(f32(spb * f32(b)) + f32(0.5))), t + int(f32(f32(spb * f32(b)) + f32(0.5))) + bn)
            for b in range(n)]


def visiting_order(first, tmax, step):
    out, j = [], 0
    while True:
        up = 1 if j % 2 else -1
        t = first + up * ((j + 1) // 2) * step
        j += 1
        if t >= tmax:
            return out
        if t >= 0:
            out.append(t)


ANCHOR_MODES = [("1200", 48000), ("300", 48000), ("rtty", 8000), ("same", 48000)]
ANCHOR_KINDS = ["nan-one", "nan-several", "nan-every", "inf-per-window", "click-1e4", "click-1e17", "click-1e18",
                "click-1e19", "click-1e20", "click-1e30", "scale-1e-20", "subnormal"]


def poison_call(x, kind, win, spb_n, rng):
    """x: the call's samples (from its position); win: the windows of its winning candidate"""
    x = x.copy()
    bad = []
    if kind.startswith("scale") or kind == "subnormal":
        s = 1e-20 if kind == "scale-1e-20" else 1e-40
        return (x.astype(np.float64) * s).astype(np.float32), bad
    if kind == "nan-every":
        for p in range(0, x.size, max(1, spb_n // 2)):
            x[p] = NAN
            bad.append(p)
        return x, bad
    pick = {"nan-one": [int(rng.integers(len(win)))], "nan-several": sorted(rng.choice(len(win), 3, False))}
    ws = pick.get(kind, range(len(win)) if kind == "inf-per-window" else [int(rng.integers(len(win)))])
    for i, b in enumerate(ws):
        lo, hi = win[b]
        p = int(rng.integers(lo, hi))
        if kind.startswith("nan"):
            x[p] = NAN
        elif kind == "inf-per-window":
            x[p] = INF if i % 2 == 0 else -INF
        else:
            x[p] = f32(float(kind.split("-")[1])) * (1 if rng.integers(2) else -1)
        bad.append(p)
    return x, bad


@pytest.mark.ref
@pytest.mark.parametrize("mode,rate", ANCHOR_MODES, ids=["%s@%d" % m for m in ANCHOR_MODES])
def test_oracle_find_frame_is_the_reference_on_bad_samples(mode, rate):
    """Every find_frame call of the oracle's rx loop over a clean stream, replayed on the call's samples
    with bad ones put into its winning candidate's windows: orc_find_frame against the unmodified src/fsk.c
    (libfsk_ref).  NaN, inf, 1e4 clicks, 1e-20 and subnormal scales: bits and frame start equal, confidence
    to the parity bar with inf as a class.  Every candidate whose windows hold NaN or inf is never chosen by
    either (a one-candidate search returns 0) and has confidence NaN or 0 in the oracle.  Clicks of 1e17 and
    more: every candidate that holds one stays below the threshold in both, and a search whose best reaches
    the threshold in either agrees exactly."""
    import golden_util as gu
    m = orc.Mode(mode, sample_rate=rate)
    d = m.derived()
    x0 = clean_stream(m, zlib.crc32(mode.encode()))
    calls = orc.rx_run(m, x0, want_calls=True)["calls"]
    assert len(calls) >= 8
    plan = orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
    ref = orc.RefPlan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
    thr = f32(m.confidence_threshold)
    rng = np.random.default_rng(7)
    counts = dict.fromkeys(ANCHOR_KINDS, 0)
    for ci, c in enumerate(calls):
        fnum, first, tmax, step, limit, sync = c[:6]
        pos = c[10]
        expect = bytes(d.expect_sync if sync else d.expect_data)
        n = len(expect)
        spb = f32(f32(fnum) / f32(n))
        span = tmax + fnum + int(spb) + 8
        seg = np.zeros(span, np.float32)
        have = x0[pos:pos + span]
        seg[:have.size] = have
        win = windows(c[9] if c[6] > 0 else first, spb, n)
        for kind in ANCHOR_KINDS:
            x, bad = poison_call(seg, kind, win, int(spb), rng)
            o = plan.find_frame(x, fnum, first, tmax, step, limit, expect)
            r = ref.find_frame(x, fnum, first, tmax, step, limit, expect)
            what = (mode, ci, kind, o, r)
            hit = lambda t: any(lo <= p < hi for p in bad for lo, hi in windows(t, spb, n))
            if kind.startswith("click-1e") and kind != "click-1e4":
                for t in visiting_order(first, tmax, step):
                    if hit(t):
                        assert not (plan.find_frame(x, fnum, t, t + 1, 1, limit, expect)[0] > thr), what
                        assert not (ref.find_frame(x, fnum, t, t + 1, 1, limit, expect)[0] > thr), what
                if not (o[0] > thr or r[0] > thr):
                    counts[kind] += 1
                    continue
            elif kind.startswith("nan") or kind.startswith("inf"):
                for t in visiting_order(first, tmax, step):
                    if hit(t):
                        one_o = plan.find_frame(x, fnum, t, t + 1, 1, limit, expect)
                        one_r = ref.find_frame(x, fnum, t, t + 1, 1, limit, expect)
                        assert one_o[0] == 0 and one_r[0] == 0 and one_o[1] == one_r[1] == 0, (what, t)
                        cf = plan.frame_analyze(x[t:].copy(), float(spb), expect)[0]
                        assert not (cf > 0), (what, t, cf)
                if o[0] > 0:
                    assert not hit(o[3]), what
            assert o[1] == r[1] and o[3] == r[3], what
            assert gu.close(o[0], r[0], cond=gu.CONF_COND), what
            assert gu.close(o[2], r[2]), what
            counts[kind] += 1
    print("%s: %d calls; %s" % (mode, len(calls), counts))


# the frames the reference's own search (libfsk_ref behind the FLAT rx loop) finds on clean_stream(m, 11) at
# each scale of the samples: recorded here so that the device test, which cannot load the reference, holds it
SCALES = [1e-45, 1e-40, 1e-20, 1e16, 1e17, 1e18, 1e19, 1e36, 1e37]
SCALE_MODES = [("1200", 48000), ("300", 48000), ("rtty", 8000)]
REF_FRAMES = {"1200": [0, 8, 8, 8, 8, 8, 8, 8, 8], "300": [0, 8, 8, 8, 8, 8, 8, 8, 0],
              "rtty": [0, 8, 8, 8, 8, 8, 8, 8, 0]}


def scaled(m, scale):
    return (clean_stream(m, 11).astype(np.float64) * scale).astype(np.float32)


@pytest.mark.ref
def test_the_references_frames_at_each_scale_are_the_recorded_ones():
    got = {}
    for mode, rate in SCALE_MODES:
        m = orc.Mode(mode, sample_rate=rate)
        got[mode] = []
        for s in SCALES:
            x = scaled(m, s)
            got[mode].append(orc.rx_many(m, x[None, :].copy(), kind="reference")[0])
    print(got)
    assert got == REF_FRAMES


# --------------------------------------------------------------------------------------------------
# the device against the FLAT oracle, per launch family
# --------------------------------------------------------------------------------------------------
FAMILIES = {f: v for f, v in rxfam.FAMILIES.items() if not f.startswith("channels")}
PRESET = {"per-candidate": ("1200", 48000), "shared-segment": ("300", 48000), "prefix-table": ("rtty", 8000),
          "tones": ("1200", 48000), "auto": ("1200", 48000), "generic": ("25", 48000)}
FLOAT_KINDS = ["nan", "nan-burst", "+inf", "-inf", "click-1e4", "click-1e30"]
S16_KINDS = ["+32767", "-32768", "-32768-burst"]
PLACES = ["window", "before", "slide", "stop", "lead"]
REPORT = {}


def preset(fam):
    return next(v for k, v in PRESET.items() if fam.startswith(k))


def places(m, x, seed, lead=None):
    """sample positions of x by role, from the oracle's records and find_frame calls on x (on m's tones):
    the middle of frame j's third window, three samples before its first window, the first window of the
    lowest candidate of a fine search (src/minimodem.c:1357-1389: the call with no search limit), which
    leaves it at the sliding search's first step, the middle of the stop bit, and the lead-in: two bit
    windows before the first frame, or, given `lead` (the auto call's silent lead-in), the last half bit of
    it, where the carrier scan still looks"""
    d = m.derived()
    res = orc.rx_run(m, x, want_calls=True)
    fr = res["frames"]
    assert len(fr) >= 4, (m.mode, len(fr))
    n = int(d.expect_n_bits)
    spb = f32(f32(d.expect_nsamples) / f32(n))
    j = 1 + seed % (len(fr) - 2)
    start = int(fr[j][5]) + int(fr[j][3])          # (frame_start, pos): relative to the call's position
    win = windows(start, spb, n)
    bn = win[0][1] - win[0][0]
    pos = {f[5] for f in fr}
    refine = [c for c in res["calls"] if np.isinf(c[4]) and c[10] in pos]
    assert refine, (m.mode, "no fine search")
    c = refine[seed % len(refine)]
    lowest = c[10] + min(visiting_order(c[1], c[2], c[3]))
    first = int(fr[0][5]) + int(fr[0][3])
    return {"window": win[2][0] + bn // 2, "before": start - 3, "slide": lowest + min(c[3], bn) // 2,
            "stop": win[-1][0] + bn // 2,
            "lead": max(0, first - 2 * bn) if lead is None else lead - bn // 2}, bn


def poison(x, kind, p, bn):
    """x float32 (or int16 for the int16 kinds) with `kind` at p"""
    x = x.copy()
    if kind == "nan":
        x[p] = NAN
    elif kind == "nan-burst":
        x[p:p + bn] = NAN
    elif kind in ("+inf", "-inf"):
        x[p] = INF if kind[0] == "+" else -INF
    elif kind.startswith("click"):
        x[p] = f32(float(kind.split("-")[1])) * (1 if p % 2 else -1)
    elif kind == "-32768-burst":
        x[p:p + bn] = -32768
    else:
        x[p] = int(kind)
    return x


class Case:
    """streams (float32; int16 families: int16 rows and their exact widening), the oracle Mode per stream,
    the tone pairs (tone call) and what each stream is"""

    def __init__(self, fam):
        f = FAMILIES[fam]
        self.fam, self.call, self.s16 = fam, f["call"], f["src"] == "s16"
        mode, rate = preset(fam)
        self.mode, self.rate = mode, rate
        # seeded by the first family that shares these streams, so that a row runs the same data alone
        seed = zlib.crc32(next(g for g in FAMILIES if case_key(g) == case_key(fam)).encode())
        rng = np.random.default_rng(seed)
        base = orc.Mode(mode, sample_rate=rate)
        self.base = base
        kinds = S16_KINDS if self.s16 else FLOAT_KINDS
        clean, modes, pairs, leads = [], [], [], []
        for s in range(3):
            m = base
            lead = None
            if self.call in ("tones", "auto"):
                nb = int(mm().RxEngine.for_mode(mode, rate).params.nbands)
            if self.call == "tones":
                fm, fs = random_pair(rng, float(base.band_width), nb)
                m = on_pair(mode, rate, fm, fs)
                pairs.append((fm, fs))
            if self.call == "auto":
                # a pair on the band grid that the scan finds: the places come from the oracle on that pair
                bs = autoorc.b_shift(base)
                bw = float(base.band_width)
                bm = int(rng.integers(max(2, 2 - bs), min(nb - 3, nb - 3 - bs)))
                m = orc.Mode(mode, sample_rate=rate, mark=bm * bw, space=(bm + bs) * bw)
                lead = int(rng.integers(20000, 26000))
                a = np.concatenate([np.zeros(lead, np.float32), clean_stream(m, seed + s, nwords=9)])
            elif mode == "25":
                a = clean_stream(m, seed + s, nwords=5)
            else:
                a = clean_stream(m, seed + s, nwords=9, amplitude=float(rng.uniform(0.3, 1.0)))
            sigma = [0.0, 1e-4 if self.call == "auto" else 0.02, 0.002][s]
            a = (a + f32(sigma) * rng.standard_normal(a.size).astype(np.float32)).astype(np.float32)
            if self.s16:
                a = widen(pcm(a))
            clean.append(a)
            modes.append(m)
            leads.append(lead)
        self.clean = clean
        self.items = []            # (base index, kind, place, samples): every kind at every place
        for pi, place in enumerate(PLACES):
            for ki, kind in enumerate(kinds):
                b = (pi + ki) % 3
                pm, bn = places(modes[b], clean[b], pi + ki, leads[b])
                p = pm[place]
                if place == "before" and kind.endswith("burst"):
                    p -= bn - 1                 # the burst ends three samples before the window
                x = pcm(clean[b]) if self.s16 else clean[b]
                self.items.append((b, kind, place, poison(x, kind, p, bn)))
        self.modes = [base] * 3 if self.call == "auto" else modes
        self.pairs = pairs or None
        self.screened = [self.screen(self.modes[b], self.as_float(x)) for b, _, _, x in self.items]

    def as_float(self, x):
        return widen(x) if self.s16 else x

    def screen(self, m, x):
        if self.call == "auto":
            return autoorc.screen(m, x)
        return tie_screen.screen(m, x)


_CASES = {}


def case_key(fam):
    return FAMILIES[fam]["call"], preset(fam), FAMILIES[fam]["src"]


def case_of(fam):
    key = case_key(fam)
    if key not in _CASES:
        _CASES[key] = Case(fam)
    return _CASES[key]


def engine_for(fam, c, monkeypatch):
    return rxfam.new_engine(monkeypatch, fam, lambda: mm().RxEngine.for_mode(c.mode, c.rate))


def launch(eng, c, rows_, bases):
    """rows_: float32 or int16 arrays, bases: the clean stream each row comes from (its tone pair) ->
    (records per row, states, bands per row or None, last_kernel)"""
    bands = None
    if c.call == "tones":
        pairs = [c.pairs[b] for b in bases]
        bands = eng.tone_bands([p[0] for p in pairs], [p[1] for p in pairs], device=dev())
    r = rxfam.call(eng, c.fam, rows_, [x.size for x in rows_], bands=bands, rec_band=True)
    assert (r.st["done"] == 1).all()
    return [r.fr[s, :int(r.st["nframes"][s])] for s in range(len(rows_))], r.st, r.rec_band, r.k["text"]


def compare(c, i, recs, st, bands, what):
    want, robust = c.screened[i]
    got = as_oracle_frames(recs)
    if not robust:
        assert abs(len(got) - len(want["frames"])) <= 1, (what, len(got), len(want["frames"]))
        return False
    compare_frames(got, want["frames"], what)
    compare_reports(reports_of(recs, st), want["reports"], what)
    if bands is not None:
        fb = [int(b) for r, b in zip(recs, bands) if int(r["frame_start"]) != mm().FRAME_REPORT]
        assert fb == want["frame_band"], (what, fb, want["frame_band"])
    return True


FAM_ROWS = list(FAMILIES)


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAM_ROWS)
def test_bad_samples_in_every_family(fam, monkeypatch):
    """Per family: the poisoned streams (every kind at every place) against the screened FLAT oracle; the clean
    streams of the launch byte for byte those of a launch whose other rows are the unpoisoned streams."""
    rxfam.skip_tma(fam)
    c = case_of(fam)
    eng = engine_for(fam, c, monkeypatch)
    src = lambda a: pcm(a) if c.s16 else a
    rows = [src(a) for a in c.clean] + [x for _, _, _, x in c.items]
    bases = list(range(len(c.clean))) + [b for b, _, _, _ in c.items]
    recs, st, bands, k = launch(eng, c, rows, bases)
    rxfam.check_family(fam, rxfam.parse_launch(k))
    ref_rows = [src(a) for a in c.clean] + [src(c.clean[b]) for b, _, _, _ in c.items]
    recs0, st0, bands0, k0 = launch(eng, c, ref_rows, bases)
    assert k0 == k
    for s in range(len(c.clean)):
        assert recs[s].tobytes() == recs0[s].tobytes() and st[s].tobytes() == st0[s].tobytes(), (fam, s)
        if bands is not None:
            assert bands[s, :len(recs[s])].tobytes() == bands0[s, :len(recs0[s])].tobytes(), (fam, s)
    out = REPORT.setdefault(fam, dict(robust=0, screened=0, kinds={}))
    for i, (b, kind, place, _) in enumerate(c.items):
        s = len(c.clean) + i
        ok = compare(c, i, recs[s], st[s], None if bands is None else bands[s], (fam, kind, place, k))
        out["robust" if ok else "screened"] += 1
        out["kinds"][kind] = out["kinds"].get(kind, 0) + 1
    assert out["robust"] >= out["screened"], (fam, out)
    print("%s: %s; %d poisoned streams held to the oracle, %d screened out; %s"
          % (fam, k, out["robust"], out["screened"], out["kinds"]))


@pytest.mark.gpu
def test_a_poisoned_row_in_tone_pair_channels():
    """rx_batch_channels, k = 2, on rows that carry a Bell103 originate and answer pair: one row with a NaN
    burst in a frame of its originate channel, one with a 1e30 click; both channels of each row against the
    screened oracle on their pair, and the clean row's channels byte for byte those of the launch without the
    poisoned rows."""
    rng = np.random.default_rng(3103)
    pairs = [(1270.0, 1070.0), (2225.0, 2025.0)]
    lines = []
    for r in range(3):
        x = np.zeros(0, np.float32)
        for fm, fs in pairs:
            m = on_pair("300", 48000, fm, fs)
            a = clean_stream(m, 50 + 2 * r + len(x), nwords=8, amplitude=float(rng.uniform(0.3, 0.8)))
            a = np.concatenate([np.zeros(int(rng.integers(0, 2000)), np.float32), a])
            if a.size > x.size:
                a, x = x, a
            x = x.copy()
            x[:a.size] += a
        lines.append((x + f32(1e-3) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32))
    m0 = on_pair("300", 48000, *pairs[0])
    p1, bn = places(m0, lines[1], 1)
    p2, _ = places(m0, lines[2], 2)
    bad = [lines[0], poison(lines[1], "nan-burst", p1["window"], bn), poison(lines[2], "click-1e30", p2["slide"], bn)]
    eng = mm().RxEngine.for_mode("300", 48000)
    for src in ("f32", "s16"):
        conv = pcm if src == "s16" else (lambda a: a)
        rows_bad = [conv(a) for a in bad]
        fl = [widen(r) for r in rows_bad] if src == "s16" else rows_bad
        if src == "f32":
            texts = check_channels_against_oracle(eng, "300", 48000, fl, [pairs] * 3, 2, ("channels", src))
            assert all(len(t) >= 3 for t in texts), texts
        buf, n = gpudev.rows(rows_bad, rows_bad[0].dtype, 8)
        buf0, _ = gpudev.rows([conv(a) for a in lines], rows_bad[0].dtype, 8)
        flat = [p for _ in range(3) for p in pairs]
        tb = eng.tone_bands([p[0] for p in flat], [p[1] for p in flat], device=dev())
        lens = np.array([a.size for a in lines], np.int32)
        fa, sa = run_channels(eng, buf, n, lens, tb, 2)
        assert eng.last_kernel().startswith("k_rx_tones") and eng.last_kernel().endswith("channels=2")
        assert ("src=" + src) in eng.last_kernel(), eng.last_kernel()
        fb, sb = run_channels(eng, buf0, n, lens, tb, 2)
        ra, sa = records(fa, sa)
        rb, sb = records(fb, sb)
        assert ra[:2] == rb[:2] and sa[:2].tobytes() == sb[:2].tobytes(), src
        if src == "s16":
            ff, sf = run_channels(eng, gpudev.rows(fl, np.float32, 8, n=n)[0], n, lens, tb, 2)
            rf, sf = records(ff, sf)
            assert rf == ra and sf.tobytes() == sa.tobytes()


# --------------------------------------------------------------------------------------------------
# the fp32 overflow of a bin, and the small end
# --------------------------------------------------------------------------------------------------
# the frames the device finds at each scale of SCALES (emulator and H100 alike); the oracle and the
# reference find REF_FRAMES.  The top: `re*re + im*im` overflows fp32 once a bin passes ~1.8e19, i.e. at
# samples of about 1e18 at 1200 baud (40-sample windows) and 2.5e17 at 300 baud and RTTY (160 and 176); the
# reference's hypotf does not, and it decodes until its FFT itself overflows (~1e37).  The bottom: the
# square underflows once a bin falls below ~1e-19 (samples of about 1e-21), where hypotf keeps subnormal
# magnitudes, so a subnormal-scale stream decodes in the reference and not here.
DEVICE_FRAMES = {"1200": [0, 0, 8, 8, 8, 8, 0, 0, 0], "300": [0, 0, 8, 8, 8, 0, 0, 0, 0],
                 "rtty": [0, 0, 8, 8, 8, 0, 0, 0, 0]}


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate", SCALE_MODES, ids=["%s@%d" % m for m in SCALE_MODES])
def test_scaled_streams_stop_decoding_at_the_documented_bound(mode, rate):
    """A clean stream scaled by 1e-45 (the smallest subnormal) to 1e37 on the default kernel: wherever the
    device decodes, its records are the oracle's; where `re*re + im*im` overflows fp32 it gives no frame."""
    m = orc.Mode(mode, sample_rate=rate)
    eng = mm().RxEngine.for_mode(mode, rate)
    rows = [scaled(m, s) for s in SCALES]
    t = torch()
    n = max(r.size for r in rows)
    fr, st = eng.rx_batch(upload(gpudev.rows(rows, np.float32, 8, n=n)[0]), nsamples=n)
    sync()
    fr, st = mm().frames_to_numpy(fr), mm().states_to_numpy(st)
    got = []
    for i, s in enumerate(SCALES):
        recs = fr[i, :int(st["nframes"][i])]
        g = as_oracle_frames(recs)
        got.append(len(g))
        want = orc.rx_run(m, rows[i])
        if g:
            compare_frames(g, want["frames"], (mode, s))
            compare_reports(reports_of(recs, st[i]), want["reports"], (mode, s))
    print("%s: %s frames per scale %s (reference %s)" % (eng.last_kernel(), got, SCALES, REF_FRAMES[mode]))
    assert got == DEVICE_FRAMES[mode], (mode, got)


# --------------------------------------------------------------------------------------------------
# int16 rows at full scale
# --------------------------------------------------------------------------------------------------
S16_FAMS = [f for f in FAMILIES if FAMILIES[f]["src"] == "s16"]


def full_scale_rows(c):
    """hard-clipped FSK (+32767 / -32768, no sample in between) of each clean stream, and a row that is
    -32768 throughout"""
    rows = [np.where(a >= 0, 32767, -32768).astype(np.int16) for a in c.clean]
    rows.append(np.full(c.clean[0].size, -32768, np.int16))
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("fam", S16_FAMS)
def test_int16_full_scale_equals_the_float_path(fam, monkeypatch):
    """Every int16 family on clipped square-wave FSK and a constant -32768 row: records and states byte for
    byte those of the float rows x / 32768 on the same instance; the clipped streams still decode."""
    c = case_of(fam)
    eng = engine_for(fam, c, monkeypatch)
    rows = full_scale_rows(c)
    bases = list(range(len(c.clean))) + [0]
    a, sa, ba, ka = launch(eng, c, rows, bases)
    rxfam.check_family(fam, rxfam.parse_launch(ka))
    b, sb, bb, kb = launch(eng, c, [widen(r) for r in rows], bases)
    assert kb.split(",src=")[0] == ka.split(",src=")[0], (ka, kb)
    assert sa.tobytes() == sb.tobytes(), fam
    assert [r.tobytes() for r in a] == [r.tobytes() for r in b], fam
    assert min(len(r) for r in a[:-1]) >= 3, fam


@pytest.mark.gpu
def test_int16_full_scale_through_the_host_slab_call():
    """rx_batch_host_s16 on the clipped rows equals rx_batch_host on their widening, byte for byte."""
    c = case_of("per-candidate-s16")
    eng = mm().RxEngine.for_mode(c.mode, c.rate)
    rows = full_scale_rows(c)
    n = max(r.size for r in rows)
    q = gpudev.rows(rows, np.int16, 8, n=n)[0]
    fa, sa = eng.rx_batch_host_s16(q, nsamples=n)
    fb, sb = eng.rx_batch_host(widen(q), nsamples=n)
    assert sa.tobytes() == sb.tobytes()
    for s in range(len(rows)):
        k = int(sa["nframes"][s])
        assert fa[s, :k].tobytes() == fb[s, :k].tobytes(), s
    assert (sa["nframes"][:-1] >= 3).all()


# --------------------------------------------------------------------------------------------------
# live streams
# --------------------------------------------------------------------------------------------------
LIVE_KINDS = ("nan", "nan-burst", "+inf", "-inf", "click-1e30")


def live_rows(form):
    """(mode, rate, rows, tone pairs per channel or None, k, burst [(row, sample)]): the clean streams of a
    family case and its poisoned streams of LIVE_KINDS at the window, before and slide places"""
    if form == "channels":
        return channel_lines()
    c = case_of({"plain": "per-candidate", "tones": "tones", "auto": "auto"}[form])
    pick = [i for i, (_, kind, place, _) in enumerate(c.items)
            if kind in LIVE_KINDS and place in ("window", "before", "slide")]
    rows = list(c.clean) + [c.items[i][3] for i in pick]
    bases = list(range(len(c.clean))) + [c.items[i][0] for i in pick]
    bursts = [(len(c.clean) + n, int(np.flatnonzero(np.isnan(c.items[i][3]))[0]))
              for n, i in enumerate(pick) if c.items[i][1] == "nan-burst"]
    pairs = [c.pairs[b] for b in bases] if c.pairs else None
    return c.mode, c.rate, rows, pairs, 1, bursts


def channel_lines():
    """Bell103 lines carrying originate and answer, k = 2: a clean line, a NaN burst, an inf and a 1e30 click
    in a frame of the originate channel"""
    rng = np.random.default_rng(3104)
    pairs = [(1270.0, 1070.0), (2225.0, 2025.0)]
    m0 = on_pair("300", 48000, *pairs[0])
    lines = []
    for r in range(4):
        x = np.zeros(0, np.float32)
        for fm, fs in pairs:
            a = clean_stream(on_pair("300", 48000, fm, fs), 70 + 2 * r + len(x), nwords=8,
                             amplitude=float(rng.uniform(0.3, 0.8)))
            a = np.concatenate([np.zeros(int(rng.integers(0, 2000)), np.float32), a])
            if a.size > x.size:
                a, x = x, a
            x = x.copy()
            x[:a.size] += a
        lines.append((x + f32(1e-3) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32))
    bursts = []
    for r, kind in ((1, "nan-burst"), (2, "+inf"), (3, "click-1e30")):
        pm, bn = places(m0, lines[r], r)
        lines[r] = poison(lines[r], kind, pm["window"], bn)
        if kind == "nan-burst":
            bursts.append((r, pm["window"]))
    return "300", 48000, lines, [p for _ in lines for p in pairs], 2, bursts


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "tones", "channels", "auto"])
def test_live_receiver_fed_bad_samples_in_random_chunks(form):
    """LiveReceiver (plain, tones=, channels_per_row=2, auto_carrier=) fed streams that carry NaN, a NaN
    burst, inf and 1e30 clicks, in random chunks with a cut inside every NaN burst: the text of one rx pass
    over the same rows (whose records test_bad_samples_in_every_family holds to the oracle), for two chunk
    sizes, and every poisoned stream keeps decoding after its bad stretch."""
    mode, rate, rows, pairs, k, bursts = live_rows(form)
    whole = one_pass_text(mode, rate, rows, pairs, k, form == "auto")
    assert sum(len(w) for w in whole) >= 3 * len(rows), whole
    cut = [(r, p + 5) for r, p in bursts]
    assert cut
    for max_chunk, seed in ((701, 1), (4000, 2)):
        got = live_text(mode, rate, rows, pairs, k, form == "auto", max_chunk, seed, cut)
        assert got == whole, (form, max_chunk, [(a, b) for a, b in zip(got, whole) if a != b][:2])
    clean = whole[:3 * k] if form != "channels" else whole[:k]
    for s, w in enumerate(whole):
        if form == "channels" and s % k:
            continue                            # the answer channel carries no bad sample of its own
        assert len(w) >= min(len(c) for c in clean) - 4, (form, s, w)


@pytest.mark.gpu
def test_live_pcm16_receiver_at_full_scale():
    """LiveReceiver(pcm16=True) fed clipped square-wave FSK and a -32768 row in random int16 chunks prints
    what the float receiver prints on the exactly widened chunks, and the clipped streams decode."""
    c = case_of("per-candidate-s16")
    rows = full_scale_rows(c)
    a = live_text(c.mode, c.rate, rows, None, 1, False, 997, 5, pcm16=True)
    b = live_text(c.mode, c.rate, [widen(r) for r in rows], None, 1, False, 997, 5)
    assert a == b
    assert all(len(x) >= 5 for x in a[:-1]), a
