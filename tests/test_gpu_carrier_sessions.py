"""Streams that lose and regain the carrier, in every rx family, against the screened FLAT oracle.

The rx loop's carrier state machine (src/minimodem.c:1278-1407) decides a refine on `confidence <
peak_confidence * 0.75`, a squelch on `amplitude < track_amplitude * 0.25`, a strike on `confidence <=
confidence_threshold`, a drop with a session report on the 21st strike, and keeps a refined frame on
`confidence2 > confidence`.  The fast kernels restate some of these decisions ahead of the state machine
(the search loop's refine predicate, the FILL 0 look-ahead's advance, the ring restart after a long
strike run), so every stream below keeps crossing them: bursts at random amplitudes, silent gaps, noise-only
segments (false acquisitions and drops), fades (squelched strikes, or a held carrier at a third of the
level), noise bursts inside a burst (in-session refines), frames cut short, and per preset two gaps just
short of and just past the 21-strike drop.  test_every_case_reaches_every_loop_event proves on the CPU,
from the oracle's own call list, that each preset's case reaches every such event.

Robust streams (tests/tie_screen.py, whose replay of the loop's bookkeeping adds margins for the squelch,
the refine trigger and refine-keep, and decides each comparison inside its margin the other way once) must give the oracle's records and session reports; the others only
the frame count within one.  Resumed at every record (max_frames = 1) and fed to LiveReceiver in random
chunks, every family must give its own one-pass result.

The CPU test runs this file's `gpu` tests on the host SIMT emulation of the kernels (tests/emu); the TMA
bulk fill is not modelled there and its rows skip."""
import copy
import zlib

import numpy as np
import pytest

import minimodem_b200 as mm
import orc
import test_gpu_instantiations as I
import test_gpu_launch_shapes as L
import tie_screen

f32 = np.float32
SIGMA_BG = 0.003
NOISE_SIGMAS = (0.05, 0.2, 0.5)
NSTREAMS = 8
KINDS = ("burst", "gap", "noise", "fade", "sag", "cut")

# the families of test_gpu_launch_shapes but its auto call, the generic kernel (a ring too large for any
# fast shape) and tone-pair channels, k = 2
FAMILIES = {f: dict(v) for f, v in L.FAMILIES.items() if v["call"] != "auto"}
for _src in ("f32", "s16"):
    FAMILIES["generic" + ("-s16" if _src == "s16" else "")] = dict(
        call="rx", src=_src, env=L.PER_CAND, kern=("k_rx", 1, 0), cls="long", n=11,
        tune=dict(ring_floats=L.SMEM_MAX // 4 + 128))
FAMILIES["channels"] = dict(call="channels", src="f32", env={}, kern=("k_rx_tones", 0, 0))
NOT_LAUNCHED = {k: v for k, v in L.NOT_LAUNCHED.items() if k[0] in FAMILIES}
NOT_LAUNCHED[("channels", "same")] = "as the tone call"
ROWS = [(fam, w) for fam in FAMILIES for w in L.PRESETS + (["random"] if "cls" in FAMILIES[fam] else [])
        if (fam, w[0]) not in NOT_LAUNCHED]


def _rid(r):
    return L._rid(r)


# ---------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------
def session_stream(rng, m, end_in_gap):
    """(samples, noise-only ranges [(start, end)]): every kind of segment once (noise twice) and up to two more, in
    random order, under sigma = 0.003 background"""
    spb = float(m.derived().nsamples_per_bit)
    words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
    # a burst of 3..10 frames; SAME's counts its one sync byte (the transmitter's preamble is 16 of them)
    tm = copy.copy(m)
    tm.do_tx_sync_bytes = min(m.do_tx_sync_bytes, 1)
    burst = lambda amp: orc.tx_words(tm, words(int(rng.integers(3, 11)) - tm.do_tx_sync_bytes), amp, 4096, True)
    parts, noise, at = [], [], 0
    kinds = list(rng.permutation(KINDS + ("noise",))) + list(rng.choice(KINDS, int(rng.integers(0, 3))))
    kinds.append("gap" if end_in_gap else "burst")
    for kind in kinds:
        amp = float(rng.uniform(0.2, 1.0))
        if kind == "gap":
            a = np.zeros(int(rng.uniform(1, 60) * spb), np.float32)
        elif kind == "noise":           # long enough to acquire a false carrier in every preset's case; longer
            # ones pile up near-ties of the threshold and the search limit on noise candidates
            a = (float(rng.choice(NOISE_SIGMAS)) * rng.standard_normal(int(rng.uniform(20, 120) * spb))).astype(np.float32)
            noise.append((at, at + a.size))
        elif kind == "fade":            # squelched at 1/8..1/5 of the level, held at 1/3
            ratio = float(rng.uniform(1 / 8, 1 / 5)) if rng.random() < 0.6 else 1 / 3
            a = np.concatenate([burst(amp), burst(amp * ratio)])
        elif kind == "sag":             # a noise burst at the signal's level inside a running burst
            a = burst(amp)
            n = int(rng.uniform(2, 6) * spb)
            p = int(rng.integers(a.size // 4, a.size // 2))
            a[p:p + n] += (0.7 * amp * rng.standard_normal(a[p:p + n].size)).astype(np.float32)
        elif kind == "cut":
            a = burst(amp)
            a = a[:int(rng.integers(a.size // 3, a.size))]
        else:
            a = burst(amp)
        parts.append(a)
        at += a.size
    x = np.concatenate(parts)
    return (x + f32(SIGMA_BG) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32), noise


def drops(m, x):
    """carrier drops (session reports before the end of the stream) of the oracle on x"""
    r = orc.rx_run(m, x, literal=False)
    return len(r["reports"]) - (1 if r["reports"] and r["reports"][-1][4] == len(r["frames"]) else 0)


def boundary_streams(m, seed):
    """Two streams burst + silent gap + burst whose gaps are the longest without a carrier drop and the
    shortest with one (a bisection on the gap length on the oracle)."""
    rng = np.random.default_rng(seed)
    words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
    a, b = orc.tx_words(m, words(4), 0.6, 4096, True), orc.tx_words(m, words(3), 0.6, 4096, True)
    hi = int(80 * float(m.derived().nsamples_per_bit))
    bg = (f32(SIGMA_BG) * rng.standard_normal(a.size + b.size + hi)).astype(np.float32)
    make = lambda gap: (np.concatenate([a, np.zeros(gap, np.float32), b]) + bg[:a.size + gap + b.size]).astype(np.float32)
    lo = 0
    assert drops(m, make(lo)) == 0 and drops(m, make(hi)) > 0
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if drops(m, make(mid)):
            hi = mid
        else:
            lo = mid
    return make(lo), make(hi)


class Case:
    """channels (one per stream, or per (row, pair) for the channel call): oracle modes, rows, lengths, tone
    bands, the oracle's results with the screen's verdicts, noise ranges; `make` builds the engine"""


_CASES = {}


def case(fam, which):
    f = FAMILIES[fam]
    call = "tones" if f["call"] == "channels" else f["call"]
    key = (f["call"], f["src"], which) if which != "random" else (f["call"], f["src"], f["cls"], f["n"])
    if key in _CASES:
        return _CASES[key]
    seed = key[:1] + key[2:]                    # int16 rows: the float streams, quantized
    rng = np.random.default_rng(zlib.crc32(repr(("sessions",) + seed).encode()))
    c = Case()
    if which == "random":
        mode, kw, exp = I.framing(f["cls"], f["n"], 7000 + f["n"])
        m = I.oracle_mode(mode, kw, exp)
        c.make = lambda: I.engine(mode, kw, exp)
        c.mode, c.rate = mode, kw["sample_rate"]
    else:
        c.mode, c.rate = which
        m = orc.Mode(c.mode, sample_rate=c.rate)
        c.make = lambda: mm.RxEngine.for_mode(which[0], which[1])
    k = 2 if f["call"] == "channels" else 1
    nch = NSTREAMS + 2 if k == 1 else 2 * (NSTREAMS // 2 + 2)
    c.modes, c.hz, c.bands, c.noise, chans = [], [], [], [], []
    if call == "tones":
        import test_gpu_stream_tones as ST
        p = mm.rx_params(mm.rx_config_for_mode(c.mode, c.rate))
        nb = int(p.nbands)
        for j in range(nch):
            fm, fs = ST.random_pair(rng, float(m.band_width), nb)
            c.hz.append((fm, fs))
            c.bands.append([int(v) for v in mm.tone_bands(p, fm, fs)])
            tm = ST.on_pair(m.mode, m.sample_rate, fm, fs)
            tm.__dict__.update({kk: v for kk, v in m.__dict__.items() if kk not in ("mark_f", "space_f")})
            c.modes.append(tm)
    else:
        c.modes = [m] * nch
    for j in range(nch):
        chans.append(session_stream(rng, c.modes[j], j % 2 == 0))
    # the boundary streams: channels 8 and 9 (k = 1), or alone on rows 4 and 5 (k = 2)
    nb_at = [NSTREAMS, NSTREAMS + 1] if k == 1 else [NSTREAMS, NSTREAMS + 3]
    short, _ = boundary_streams(c.modes[nb_at[0]], zlib.crc32(repr(seed).encode()))
    _, past = boundary_streams(c.modes[nb_at[1]], zlib.crc32(repr(seed).encode()) + 1)
    chans[nb_at[0]] = (short, [])
    chans[nb_at[1]] = (past, [])
    if k == 2:
        for j in (NSTREAMS + 1, NSTREAMS + 2):      # the other channel of those rows carries nothing
            chans[j] = (np.zeros(1, np.float32), [])
    c.k = k
    c.rows = []
    for r in range(nch // k):
        xs = [chans[r * k + j][0] for j in range(k)]
        x = np.zeros(max(v.size for v in xs), np.float32)
        for v in xs:
            x[:v.size] += v
        c.rows.append(x)
    if f["src"] == "s16":                       # what the int16 rows carry, exactly
        c.rows = [L._pcm(x).astype(np.float32) / f32(32768) for x in c.rows]
    c.noise = [ch[1] for ch in chans]
    c.lens = np.array([x.size for x in c.rows], np.int32)
    c.row_of = [j // k for j in range(nch)]
    c.screened = [tie_screen.screen(c.modes[j], c.rows[c.row_of[j]]) for j in range(nch)]
    c.boundary = [(nb_at[0], 0), (nb_at[1], 1)]
    _CASES[key] = c
    return c


# ---------------------------------------------------------------------------------------------------
# CPU: the loop events every case reaches
# ---------------------------------------------------------------------------------------------------
EVENTS = ("acquire", "refine-in-session", "strike-threshold", "strike-squelch", "drop", "held-15-strikes",
          "acquire-in-noise", "open-at-end", "ends-mid-count")
# the events a preset's case cannot reach, with the reason
NOT_REACHED = {}


def events_of(m, x, noise):
    """the loop events of the oracle's run on x, from its call list"""
    r = orc.rx_run(m, x, literal=False, want_calls=True)
    calls = [(cl[6], cl[8], 0.0, cl[7], cl[9], cl[3]) for cl in r["calls"]]
    ev = []
    frames, reports, _ = tie_screen.replay(m, calls, events=ev)
    assert [f[:5] for f in r["frames"]] == frames and r["reports"] == reports
    kinds = set()
    for kind, i in ev:
        if kind == "acquire":
            at = r["calls"][i][10] + r["calls"][i][9]
            if any(a <= at < b for a, b in noise):
                kinds.add("acquire-in-noise")
        kinds.add(kind)
    return kinds


def test_every_case_reaches_every_loop_event():
    """From the oracle's call list: every preset's case (plain, tone and channel calls) reaches every loop
    event, but those NOT_REACHED names; the boundary streams straddle the 21-strike drop."""
    seen = {}
    for fam in ("per-candidate", "tones", "channels"):
        for which in L.PRESETS:
            if (fam, which[0]) in NOT_LAUNCHED:
                continue
            c = case(fam, which)
            got = set()
            for j, (want, _) in enumerate(c.screened):
                got |= events_of(c.modes[j], c.rows[c.row_of[j]], c.noise[j])
            for j, ndrop in c.boundary:
                assert min(drops(c.modes[j], c.rows[c.row_of[j]]), 1) == ndrop, (fam, which, j)
            seen[(FAMILIES[fam]["call"], which[0])] = got
            missing = [e for e in EVENTS if e not in got and (FAMILIES[fam]["call"], which[0], e) not in NOT_REACHED]
            print("%s %s: %s" % (fam, which[0], " ".join(e for e in EVENTS if e in got)))
            assert not missing, (fam, which, missing)
    for (call, preset, e), why in NOT_REACHED.items():
        assert e not in seen.get((call, preset), set()), (call, preset, e, "reached after all", why)


# ---------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------
def new_engine(monkeypatch, fam, c):
    f = FAMILIES[fam]
    L.set_env(monkeypatch, f["env"])
    eng = c.make()
    if "tune" in f:
        eng.tune(**f["tune"])
    return eng


def run(eng, fam, c, max_frames=None, states=None):
    """records per channel (bytes), the states, the launch"""
    f = FAMILIES[fam]
    t = I.torch()
    n = int(c.lens.max())
    buf = I._rows(c.rows, n, np.float32, 8)
    if f["src"] == "s16":
        buf = L._pcm(buf)
    x = t.from_numpy(buf).to(I.dev())
    le = t.from_numpy(c.lens).to(I.dev())
    if f["call"] == "rx":
        fr, st = eng.rx_batch(x, nsamples=n, nsamples_each=le, max_frames=max_frames, states=states)
    else:
        tb = t.from_numpy(np.array(c.bands, np.int32)).to(I.dev())
        fr, st = eng.rx_batch_tones(x, tb, nsamples=n, nsamples_each=le, max_frames=max_frames, states=states,
                                    channels_per_row=c.k)
    I.sync()
    fr, sn = mm.frames_to_numpy(fr), mm.states_to_numpy(st)
    text = eng.last_kernel()
    if c.k > 1:
        assert text.endswith(" channels=%d" % c.k), text
        text = text[:-len(" channels=%d" % c.k)]
    eng_k = L.LK.match(text)
    assert eng_k, text
    name, mode, fill = f["kern"]
    k = dict(zip(("name", "mode", "fill", "src"), (eng_k.group(1), int(eng_k.group(5)), int(eng_k.group(6)),
                                                    eng_k.group(7))))
    assert (k["name"], k["mode"], k["fill"]) == (name, mode, fill), (fam, text)
    assert k["src"].split(",")[0] == f["src"], (fam, text)
    if fam in ("per-candidate", "per-candidate-noslide"):
        assert k["src"] == ("f32,slide" if fam == "per-candidate" else "f32"), text
    return [fr[s, :int(sn["nframes"][s])].tobytes() for s in range(len(sn))], sn.copy(), text


def skip_tma(fam):
    if I.emulated() and FAMILIES[fam]["kern"][2] == 1:
        pytest.skip("the host emulation does not model cp.async.bulk / mbarrier")


SCREEN_COUNT = {}


@pytest.mark.gpu
@pytest.mark.parametrize("fam,which", ROWS, ids=[_rid(r) for r in ROWS])
def test_carrier_sessions_against_the_screened_oracle(fam, which, monkeypatch):
    """Robust channels give the oracle's records and session reports, screened-out ones its frame count
    within one."""
    skip_tma(fam)
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    recs, st, text = run(eng, fam, c)
    what = "%s %s %s" % (fam, which, text)
    I.compare_rx((None,) * 5 + (c.screened,), [np.frombuffer(r, mm.FRAME_DTYPE) for r in recs], st, what)
    bad = sum(1 for _, r in c.screened if not r)
    cnt = SCREEN_COUNT.setdefault(fam, [0, 0])
    cnt[0] += bad
    cnt[1] += len(c.screened)
    print("%s: %d records, %d of %d channels screened out" % (what, int(st["nframes"].sum()), bad, len(c.screened)))


@pytest.mark.gpu
def test_carrier_sessions_screen_out_few_streams():
    """Runs after the oracle tests: at most 10 % of each family's channels are screened out."""
    if not SCREEN_COUNT:
        pytest.skip("no carrier-session test ran in this session")
    for fam, (bad, total) in sorted(SCREEN_COUNT.items()):
        print("%s: %d of %d streams screened out" % (fam, bad, total))
        assert bad <= 0.1 * total, (fam, bad, total)


RESUME_ROWS = [(fam, ("300", 48000) if FAMILIES[fam]["call"] == "rx" else ("1200", 48000)) for fam in FAMILIES]


@pytest.mark.gpu
@pytest.mark.parametrize("fam,which", RESUME_ROWS, ids=[_rid(r) for r in RESUME_ROWS])
def test_carrier_sessions_resumed_at_every_record(fam, which, monkeypatch):
    """max_frames = 1: every call ends at a frame or a session report; the records joined equal one pass
    byte for byte and the final states equal its states but nframes."""
    skip_tma(fam)
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    one, st1, _ = run(eng, fam, c)
    joined = [b""] * len(one)
    states = None
    for i in range(100000):
        got, st, _ = run(eng, fam, c, max_frames=1, states=states)
        assert (st["nframes"] <= 1).all()
        for s in range(len(joined)):
            joined[s] += got[s]
        if (st["done"] == 1).all():
            break
        st = st.copy()
        st["nframes"][:] = 0
        states = I.torch().from_numpy(st.view(np.int32).reshape(len(st), -1).copy()).to(I.dev())
    assert joined == one, fam
    nrep = sum(1 for r in one for rec in np.frombuffer(r, mm.FRAME_DTYPE) if int(rec["frame_start"]) == mm.FRAME_REPORT)
    assert nrep >= 2 and i + 1 >= max(len(r) for r in one) // mm.FRAME_DTYPE.itemsize, (fam, nrep, i)
    st = st.copy()
    st["nframes"] = st1["nframes"]
    assert st.tobytes() == st1.tobytes(), fam
    print("%s: %d calls, %d records (%d session reports) equal to one pass" % (
        fam, i + 1, int(st1["nframes"].sum()), nrep))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "tones", "channels", "pcm16"])
def test_live_receiver_on_carrier_sessions(form):
    """LiveReceiver fed the session streams in random chunks, with a cut inside every silent gap and
    noise segment while the strikes are counting: the text of one rx pass over the same rows."""
    import test_gpu_sample_domain as SD
    fam = {"plain": "per-candidate", "tones": "tones", "channels": "channels", "pcm16": "per-candidate-s16"}[form]
    c = case(fam, ("1200", 48000))
    rows = [L._pcm(x) for x in c.rows] if form == "pcm16" else c.rows
    pairs = c.hz if c.hz else None
    cuts = [(c.row_of[j], (a + b) // 2) for j, ns in enumerate(c.noise) for a, b in ns]
    for j, x in enumerate(c.rows):             # and inside the silent gaps
        quiet = np.flatnonzero(np.abs(x) < 0.02)
        if quiet.size:
            cuts.append((j, int(quiet[quiet.size // 2])))
    whole = SD.one_pass_text(c.mode, c.rate, rows, pairs, c.k, False)
    assert sum(len(w) for w in whole) >= 3 * len(rows), whole
    got = SD.live_text(c.mode, c.rate, rows, pairs, c.k, False, 1501, 7, cuts, pcm16=form == "pcm16")
    assert got == whole, (form, [(a, b) for a, b in zip(got, whole) if a != b][:2])


def test_carrier_sessions_on_the_emulated_kernels():
    """The `gpu` tests above on the host SIMT emulation of the kernels, copies landing late."""
    import test_emu_parity
    tail = test_emu_parity.run_emulated("gpu", "late", 3000, module="test_gpu_carrier_sessions.py")
    assert " passed" in tail and "failed" not in tail
