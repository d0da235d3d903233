"""Every rx, find-frame and transmitter kernel instantiation the launchers can dispatch, on random
framings, against the oracle.

The rest of the `gpu` suite drives the kernels through a few fixed geometries; `rx_batch_any` and
`fsk_b200_find_frame_batch` (minimodem_b200/csrc/fsk_b200_kernels.cu) can launch some 140 distinct
template instances, and `tx_launch` eight.  The tables below map each launchable instance to a framing
and an environment that reach it, each test asserts that `last_kernel()` names the instance its row
claims (the launcher falls back silently otherwise), and test_the_tables_cover_every_instantiation
checks that the tables cover exactly what the kernel source instantiates, minus UNREACHABLE.

Random streams are screened for near-ties first (tests/tie_screen.py): a robust stream must give the
oracle's records under the usual parity bar, a stream whose records hinge on a knife-edge decision
only the frame count.  The screen is deterministic, so no case is flaky.

Under FSK_B200_EMU=1 (tests/emu) the same tests run on the host emulation (under a minute); the TMA bulk
fills (cp.async.bulk + mbarrier) are not modelled there and their rows are skipped."""
import os
import re

import numpy as np
import pytest

import emu_fuzz
import minimodem_b200 as mm
import orc
import tie_screen
import txorc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "minimodem_b200", "csrc", "fsk_b200_kernels.cu")
EPS = np.float32(1.1920928955078125e-07)


def emulated():
    import conftest
    return conftest.EMU_DEVICE is not None


def torch():
    return pytest.importorskip("torch")


def dev():
    import conftest
    if conftest.EMU_DEVICE is not None:
        return conftest.EMU_DEVICE
    assert torch().cuda.is_available(), "GPU tests need a CUDA device"
    return torch().device("cuda:0")


def sync():
    if not emulated():
        torch().cuda.synchronize()


# ---------------------------------------------------------------------------------------------------
# the coverage tables
# ---------------------------------------------------------------------------------------------------
# Framing classes: "short" = bit periods of 10..60 samples (the per-candidate kernels), "tile" = whole
# bit periods of 40..160 samples, so that the windows tile (shared-segment and prefix-table kernels),
# "long" = bit periods over 1536 samples (the twiddle table leaves shared memory: the generic kernels).
# n = the window count (expect string length) that makes the launcher pick the shape.
PER_CAND = {"FSK_B200_MULTI": "0", "FSK_B200_PREFIX": "0"}


def _fast(G, W, L, n):
    return dict(n=n, cls="short", env=dict(PER_CAND, FSK_B200_LANES=str(G), FSK_B200_SPLIT=str(L)))


def _n_for(G, W, L):
    """a window count for which W windows per lane are needed: in ((W - 1) G/L, W G/L]"""
    per = G // L
    return max(2, (W - 1) * per + 1 + (per - 1) // 2)


FAST_SHAPES = [(4, 1, 1), (4, 2, 1), (4, 3, 1), (4, 4, 1), (4, 2, 2), (4, 4, 2),
               (8, 1, 1), (8, 2, 1), (8, 3, 1), (8, 4, 1), (8, 1, 2), (8, 2, 2), (8, 3, 2), (8, 4, 2), (8, 4, 4),
               (16, 1, 1), (16, 2, 1), (16, 3, 1), (16, 4, 1), (16, 1, 2), (16, 2, 2), (16, 3, 2), (16, 4, 2),
               (16, 1, 4), (16, 2, 4), (16, 3, 4), (16, 4, 4),
               (32, 1, 1), (32, 2, 1), (32, 1, 2), (32, 2, 2), (32, 3, 2), (32, 4, 2), (32, 1, 4), (32, 2, 4),
               (32, 3, 4), (32, 4, 4)]
S16_SHAPES = [(8, 1, 1), (8, 2, 1), (8, 3, 1), (8, 2, 2), (8, 3, 2), (8, 4, 2), (8, 4, 4),
              (16, 1, 2), (16, 2, 2), (16, 2, 4), (16, 3, 4), (16, 4, 4), (32, 2, 4)]
# shared-segment (mode 2): the launcher takes the (W, L) of the fewest period slots W G/L >= n + 1
MULTI_ROWS = {(8, 2, 2): 7, (8, 3, 2): 10, (8, 4, 2): 14, (16, 2, 4): 6, (16, 3, 4): 11, (16, 4, 4): 13,
              (16, 3, 2): 20, (16, 4, 2): 28, (32, 2, 4): 14, (32, 3, 4): 19, (32, 4, 4): 27}
# prefix-table (mode 3): W codes the candidate slot of n + 1 window boundaries
PFX_ROWS = {1: 8, 3: 7, 4: 11, 5: 20}


def _multi(G, n):
    return dict(n=n, cls="tile", env=dict(FSK_B200_LANES=str(G), FSK_B200_MULTI="2", FSK_B200_PREFIX="0"))


def _pfx(n, fill):
    return dict(n=n, cls="tile", env=dict(FSK_B200_PREFIX="1", FSK_B200_PFX_FILL=str(fill)))


RX_TABLE = {}
for (G, W, L) in FAST_SHAPES:
    RX_TABLE[(G, W, L, 0, 0, "f32")] = _fast(G, W, L, _n_for(G, W, L))
for (G, W, L) in S16_SHAPES:
    RX_TABLE[(G, W, L, 0, 0, "s16")] = _fast(G, W, L, _n_for(G, W, L))
for (G, W, L), n in MULTI_ROWS.items():
    for src in ("f32", "s16"):
        RX_TABLE[(G, W, L, 2, 0, src)] = _multi(G, n)
for W, n in PFX_ROWS.items():
    RX_TABLE[(32, W, 1, 3, 1, "f32")] = _pfx(n, 1)
    RX_TABLE[(32, W, 1, 3, 0, "f32")] = _pfx(n, 0)
    RX_TABLE[(32, W, 1, 3, 0, "s16")] = _pfx(n, 0)
for src in ("f32", "s16"):
    RX_TABLE[("generic", src)] = dict(n=11, cls="long", env=dict(PER_CAND))

FF_TABLE = {(G, W, L, 0): _fast(G, W, L, _n_for(G, W, L)) for (G, W, L) in FAST_SHAPES}
FF_TABLE[("generic",)] = dict(n=11, cls="long", env={})

UNREACHABLE = {
    (16, 2, 2, 2, 0, "f32"): "mode 2 takes the fewest period slots and lets a later shape win a tie: "
                             "(16, 4, 4) has the same 16 slots as (16, 2, 2) and is listed after it",
    (16, 2, 2, 2, 0, "s16"): "as the float build: (16, 4, 4) wins the 16-slot tie",
}

# the transmitter: <T, VEC, LUT> by construction, plus where the sine table lives
TX_LUTS = [0, 16, 1000, 4095, 8193, 16384, 65536]
TX_ROWS = [(fmt, align, lut) for fmt in ("f32", "s16") for align in ("aligned", "odd-stride", "offset-base")
           for lut in TX_LUTS]


def tx_key(fmt, align, lut):
    """the k_tx_synth instance tx_launch picks for this construction, and the table's placement"""
    size = 4 if fmt == "f32" else 2
    vec = 16 // size if align == "aligned" else 1
    place = "none" if lut == 0 else "smem" if lut * size <= 32768 else "global"
    return (fmt, vec, lut > 0, place)


def kernel_key(s):
    """last_kernel() -> the key of the tables"""
    m = re.match(r"(k_rx|k_find_frame)<G=(\d+),W=(\d+),L=(\d+),mode=(\d)\(([a-z-]+)\)(?:,fill=(\d),src=(\w+))?", s)
    assert m, s
    G, W, L, mode = (int(m.group(i)) for i in (2, 3, 4, 5))
    if m.group(1) == "k_find_frame":
        return ("generic",) if mode == 1 else (G, W, L, mode)
    src = m.group(8)
    return ("generic", src) if mode == 1 else (G, W, L, mode, int(m.group(7)), src)


def launchable():
    """(rx keys, find-frame keys, tx keys) the kernel source can dispatch, from its combo lists"""
    src = open(KERNELS).read()

    def combos(name):
        m = re.search(r"#define %s\(X\)((?:[^\n]*\\\n)*[^\n]*)" % name, src)
        return [tuple(int(v) for v in t.split(",")) for t in re.findall(r"X\(([\d, ]+)\)", m.group(1))]
    fast, multi, s16 = combos("FAST_COMBOS"), combos("MULTI_COMBOS"), combos("S16_FAST_COMBOS")
    pfx = [w for (w,) in combos("PFX_SLOTS")]
    rx = {(G, W, L, 0, 0, "f32") for G, W, L in fast} | {(G, W, L, 0, 0, "s16") for G, W, L in s16}
    rx |= {(G, W, L, 2, 0, s) for G, W, L in multi for s in ("f32", "s16")}
    rx |= {(32, W, 1, 3, f, "f32") for W in pfx for f in (0, 1)} | {(32, W, 1, 3, 0, "s16") for W in pfx}
    rx |= {("generic", "f32"), ("generic", "s16")}
    ff = {(G, W, L, 0) for G, W, L in fast} | {("generic",)}
    tx = {(t, v, lut, p) for t, v in (("f32", 4), ("f32", 1), ("s16", 8), ("s16", 1))
          for lut, p in ((False, "none"), (True, "smem"), (True, "global"))}
    return rx, ff, tx


def test_the_tables_cover_every_instantiation():
    """CPU: the tables = what rx_batch_any / the find-frame launcher / tx_launch can dispatch, minus
    UNREACHABLE (each with its reason)."""
    rx, ff, tx = launchable()
    assert set(UNREACHABLE) <= rx
    assert set(RX_TABLE) == rx - set(UNREACHABLE), (rx - set(RX_TABLE) - set(UNREACHABLE), set(RX_TABLE) - rx)
    assert not set(RX_TABLE) & set(UNREACHABLE)
    assert set(FF_TABLE) == ff, (ff ^ set(FF_TABLE))
    assert {tx_key(*r) for r in TX_ROWS} == tx
    print("instantiations: %d rx (%d unreachable), %d find_frame, %d tx"
          % (len(RX_TABLE), len(UNREACHABLE), len(FF_TABLE), len(tx)))


# ---------------------------------------------------------------------------------------------------
# random framings
# ---------------------------------------------------------------------------------------------------
PAIRS = {"short": [(b, r) for b in emu_fuzz.BAUDS for r in emu_fuzz.RATES if 10 <= r / b <= 60],
         "tile": [(600, 48000), (300, 48000), (1200, 48000)],
         "long": [(25, 48000), (20, 44100)]}


def framing(cls, n, seed):
    """(mode, kw, expect override or None): a random framing of class `cls` whose expect string has n
    windows -- its own if it has n, else its own cut to n or continued with don't-care windows"""
    rng = np.random.default_rng(seed)
    pairs = PAIRS[cls]
    while True:
        baud, rate = pairs[int(rng.integers(0, len(pairs)))]
        kw = dict(sample_rate=rate)
        kw["n_data_bits"] = int(rng.choice([5, 6, 7, 8, 9, 12, 16] if n < 24 else [n - 8, n - 6, n - 4]))
        kw["startbits"] = int(rng.choice([1, 1, 2]))
        kw["stopbits"] = float(rng.choice([1.0, 1.0, 1.5, 2.0]))
        kw["msb_first"] = bool(rng.integers(0, 2))
        kw["invert_start_stop"] = bool(rng.integers(0, 2))
        kw["inverted"] = bool(rng.integers(0, 2))
        if cls == "tile" and kw["stopbits"] == 1.5:
            continue
        try:
            m = orc.Mode(str(baud), **kw)
            d = m.derived()
            orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
        except Exception:
            continue
        if max(m.mark_f, m.space_f) >= rate / 2 - m.band_width:
            continue
        own = bytes(d.expect_data)
        exp = None if len(own) == n else (own[:n] if len(own) > n else own + b"d" * (n - len(own)))
        return str(baud), kw, exp


def oracle_mode(mode, kw, exp):
    m = orc.Mode(mode, **kw)
    m.expect_data_string = exp
    return m


def engine(mode, kw, exp):
    names = dict(startbits="nstartbits", stopbits="nstopbits")
    ov = {names.get(k, k): v for k, v in kw.items() if k != "sample_rate"}
    cfg = mm.rx_config_for_mode(mode, kw.get("sample_rate", 48000), **ov)
    if exp is not None:
        cfg.expect_data_string = exp
    return mm.RxEngine(mm.rx_params(cfg))


_CASES = {}


def rx_case(cls, n):
    """A random framing of class cls with n windows and 3..8 streams from the oracle's
    transmitter: ragged lead-in, sigma = 0.01 noise, the last stream cut in mid-frame; with the oracle's
    records and the screen's verdict per stream.  Computed once per (cls, n)."""
    key = (cls, n)
    if key in _CASES:
        return _CASES[key]
    seed = 4000 + 100 * ["short", "tile", "long"].index(cls) + n
    mode, kw, exp = framing(cls, n, seed)
    m = oracle_mode(mode, kw, exp)
    rng = np.random.default_rng(seed)
    spb = int(m.derived().nsamples_per_bit)
    nstreams = int(rng.integers(3, 9))
    nwords = 4 if cls == "long" else int(rng.integers(8, 16))
    streams = []
    for s in range(nstreams):
        words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
        a = orc.tx_words(m, words, float(rng.uniform(0.3, 1.0)), 4096, True)
        lead = int(rng.integers(0, 3 * spb + 1))
        x = np.concatenate([np.zeros(lead, np.float32), a])
        if s == nstreams - 1:
            x = x[:lead + int(a.size * rng.uniform(0.4, 0.9))]
        x = (x + np.float32(0.01) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
    screened = [tie_screen.screen(m, x) for x in streams]
    _CASES[key] = (mode, kw, exp, m, streams, screened)
    return _CASES[key]


SCREEN_COUNT = {}
REACHED = set()


def compare_rx(case, recs, st, what):
    import test_gpu_parity as T
    mode, kw, exp, m, streams, screened = case
    assert (st["done"] == 1).all(), what
    for s, (want, robust) in enumerate(screened):
        got = T.as_oracle_frames(recs[s])
        if robust:
            T.compare_frames(got, want["frames"], "%s stream %d" % (what, s))
            T.compare_reports(T.reports_of(recs[s], st[s]), want["reports"], "%s stream %d" % (what, s))
        else:
            assert abs(len(got) - len(want["frames"])) <= 1, (what, s, len(got), len(want["frames"]))


def _setenv(monkeypatch, env):
    for k in ("FSK_B200_LANES", "FSK_B200_SPLIT", "FSK_B200_MULTI", "FSK_B200_PREFIX", "FSK_B200_PFX_FILL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)                # read when the engine is created


def _rows(streams, n, dtype, align=4):
    stride = (n + align - 1) & ~(align - 1)
    buf = np.zeros((len(streams), stride), dtype)
    for i, a in enumerate(streams):
        buf[i, :len(a)] = a
    return buf


def _skip_tma(key):
    if emulated() and len(key) == 6 and key[3] == 3 and key[4] == 1:
        pytest.skip("the host emulation does not model cp.async.bulk / mbarrier")


RX_F32 = sorted((k for k in RX_TABLE if k[-1] == "f32"), key=str)
RX_S16 = sorted((k for k in RX_TABLE if k[-1] == "s16"), key=str)


@pytest.mark.gpu
@pytest.mark.parametrize("key", RX_F32, ids=[str(k) for k in RX_F32])
def test_rx_instantiation_on_random_framings(key, monkeypatch):
    """Float rows: every float k_rx instance against the screened oracle records."""
    _skip_tma(key)
    row = RX_TABLE[key]
    case = rx_case(row["cls"], row["n"])
    mode, kw, exp, m, streams, screened = case
    _setenv(monkeypatch, row["env"])
    eng = engine(mode, kw, exp)
    assert eng.params.expect_n_bits == row["n"]
    n = max(len(a) for a in streams)
    lens = np.array([len(a) for a in streams], np.int32)
    t = torch()
    frames, states = eng.rx_batch(t.from_numpy(_rows(streams, n, np.float32)).to(dev()), nsamples=n,
                                  nsamples_each=t.from_numpy(lens).to(dev()))
    sync()
    assert kernel_key(eng.last_kernel()) == key, eng.last_kernel()
    REACHED.add(key)
    fr, st = mm.frames_to_numpy(frames), mm.states_to_numpy(states)
    compare_rx(case, [fr[i, :st["nframes"][i]] for i in range(len(streams))], st, "%s %s %r" % (key, mode, kw))
    fam = "mode%d" % key[3] if key[0] != "generic" else "generic"
    c = SCREEN_COUNT.setdefault(fam, [0, 0])
    c[0] += sum(1 for _, r in screened if not r)
    c[1] += len(screened)
    print("%s: %d of %d streams screened out" % (key, sum(1 for _, r in screened if not r), len(screened)))


@pytest.mark.gpu
@pytest.mark.parametrize("key", RX_S16, ids=[str(k) for k in RX_S16])
def test_rx_instantiation_int16_rows_equal_the_float_rows(key, monkeypatch):
    """int16 rows: every int16 k_rx instance gives the float path's records on s16/32768 bit for bit,
    in one pass and resumed from a position that is not a multiple of 8."""
    row = RX_TABLE[key]
    mode, kw, exp, m, streams, _ = rx_case(row["cls"], row["n"])
    _setenv(monkeypatch, row["env"])
    eng = engine(mode, kw, exp)
    n = max(len(a) for a in streams)
    t = torch()
    pcm = _rows([np.clip(np.round(a * 32768.0), -32768, 32767) for a in streams], n, np.int16, 8)
    lens = t.from_numpy(np.array([len(a) for a in streams], np.int32)).to(dev())
    d16 = t.from_numpy(pcm).to(dev())
    f32 = mm.s16_to_f32(d16)
    fr_a, st_a = eng.rx_batch(f32, nsamples=n, nsamples_each=lens)
    fr_b, st_b = eng.rx_batch(d16, nsamples=n, nsamples_each=lens)
    sync()
    assert kernel_key(eng.last_kernel()) == key, eng.last_kernel()
    REACHED.add(key)
    sa, sb = mm.states_to_numpy(st_a), mm.states_to_numpy(st_b)
    assert sa.tobytes() == sb.tobytes(), key
    a, b = mm.frames_to_numpy(fr_a), mm.frames_to_numpy(fr_b)
    for s in range(len(streams)):
        k = int(sa["nframes"][s])
        assert a[s, :k].tobytes() == b[s, :k].tobytes(), (key, s)
    assert sa["nframes"].sum() >= len(streams), key
    resume = mm.states_to_numpy(st_b).copy()
    resume[:] = np.zeros(1, resume.dtype)
    resume["pos"][:] = 13
    st_c = t.from_numpy(resume.view(np.int32).reshape(len(streams), -1).copy()).to(dev())
    st_d = st_c.clone()
    fr_c, st_c = eng.rx_batch(f32, nsamples=n, nsamples_each=lens, states=st_c)
    fr_d, st_d = eng.rx_batch(d16, nsamples=n, nsamples_each=lens, states=st_d)
    sync()
    assert kernel_key(eng.last_kernel()) == key, eng.last_kernel()
    c, d = mm.frames_to_numpy(fr_c), mm.frames_to_numpy(fr_d)
    sc = mm.states_to_numpy(st_c)
    assert sc.tobytes() == mm.states_to_numpy(st_d).tobytes(), (key, "resumed")
    for s in range(len(streams)):
        k = int(sc["nframes"][s])
        assert c[s, :k].tobytes() == d[s, :k].tobytes(), (key, s, "resumed")


@pytest.mark.gpu
def test_screen_rejects_few_streams():
    """Runs after the rx tests: at most 10 % of each family's streams are screened out."""
    if not SCREEN_COUNT:
        pytest.skip("no rx instantiation ran in this session")
    print("%d k_rx instantiations reached" % len(REACHED))
    for fam, (bad, total) in sorted(SCREEN_COUNT.items()):
        print("%s: %d of %d streams screened out" % (fam, bad, total))
        assert bad <= 0.1 * total, (fam, bad, total)


# ---------------------------------------------------------------------------------------------------
# per-bit magnitudes of every k_find_frame instance against a float64 DFT
# ---------------------------------------------------------------------------------------------------
# The largest deviation of a window's magnitude from the float64 DFT, relative to the window's larger
# magnitude, over every instance and sigma: 3.3e-7 on the emulator and 3.7e-7 on an H100 80GB HBM3
# (700 W power limit).  The bar is 4x the larger of the two.
PERBIT_BAR = 1.5e-6
PERBIT_MAX = [0.0]

FF_KEYS = sorted(FF_TABLE, key=str)


@pytest.mark.gpu
@pytest.mark.parametrize("key", FF_KEYS, ids=[str(k) for k in FF_KEYS])
def test_find_frame_instantiation_per_bit_magnitudes_vs_fp64(key, monkeypatch):
    row = FF_TABLE[key]
    mode, kw, exp = framing(row["cls"], row["n"], 9000 + row["n"] + (500 if row["cls"] == "long" else 0))
    m = oracle_mode(mode, kw, exp)
    _setenv(monkeypatch, row["env"])
    eng = engine(mode, kw, exp)
    p = eng.params
    assert p.expect_n_bits == row["n"]
    rng = np.random.default_rng(17 + row["n"])
    words = rng.integers(0, 1 << m.n_data_bits, 40 if row["cls"] == "short" else 6, dtype=np.uint64).astype(np.uint32)
    clean = orc.tx_words(m, words, 1.0, 4096, True)
    spb = float(p.nsamples_per_bit)
    tmc = int(np.float32(np.float32(spb) * np.float32(0.75) + np.float32(0.5))) + p.nsamples_overscan
    wlen = (tmc + p.expect_nsamples + int(spb) + 8 + 3) & ~3
    nstreams = 48
    buf = np.zeros((nstreams, wlen), np.float32)
    sigmas = (0.0, 0.05, 0.3)
    for s in range(nstreams):
        pos = int(rng.integers(0, max(1, clean.size - wlen)))
        w = np.zeros(wlen, np.float32)
        seg = clean[pos:pos + wlen]
        w[:seg.size] = seg
        buf[s] = (w + sigmas[s % 3] * rng.standard_normal(wlen)).astype(np.float32)
    t = torch()
    T = lambda a, dt: t.from_numpy(np.ascontiguousarray(np.asarray(a).astype(dt))).to(dev())
    full = lambda v, dt: T(np.full(nstreams, v), dt)
    step = max(tmc // 8, 1)
    frames, mags = eng.find_frame_batch(T(buf, np.float32), full(wlen, np.int32), full(p.nsamples_overscan, np.int32),
                                        full(tmc, np.int32), full(step, np.int32), full(np.inf, np.float32),
                                        bit_mags=True)
    sync()
    assert kernel_key(eng.last_kernel()) == key, eng.last_kernel()
    fr, mg = mm.frames_to_numpy(frames), mags.cpu().numpy()
    plan = orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
    nb = int(p.expect_n_bits)
    spb_fsk = np.float32(np.float32(p.expect_nsamples) / np.float32(nb))           # src/fsk.c:465
    N = int(np.float32(spb_fsk + np.float32(0.5)))
    F = int(p.fftsize)
    tw_m = np.exp(-2j * np.pi * ((int(p.b_mark) * np.arange(N)) % F) / F)
    tw_s = np.exp(-2j * np.pi * ((int(p.b_space) * np.arange(N)) % F) / F)
    bar = PERBIT_BAR
    if emulated():      # FSK_EMU_ULP=n moves the emulated sqrt by up to n ulp
        bar += int(os.environ.get("FSK_EMU_ULP", "0")) * 2.0 ** -23
    worst = 0.0
    checked = 0
    for s in range(nstreams):
        if not fr[s]["confidence"] > 0:
            continue
        start = int(fr[s]["frame_start"])
        bits = int(fr[s]["bits_lo"]) | (int(fr[s]["bits_hi"]) << 32)
        x = buf[s, start:].astype(np.float64)
        for b in range(nb):
            beg = int(np.float32(np.float32(spb_fsk * np.float32(b)) + np.float32(0.5)))
            seg = np.zeros(N)
            have = x[beg:beg + N]
            seg[:have.size] = have
            mk = abs(np.dot(seg, tw_m)) * 2.0 / N
            sp = abs(np.dot(seg, tw_s)) * 2.0 / N
            top = max(mk, sp)
            if top == 0:
                continue
            dev_ = max(abs(mg[s, b, 0] - top), abs(mg[s, b, 1] - min(mk, sp))) / top
            worst = max(worst, dev_)
            assert dev_ <= bar, (key, s, b, dev_, mg[s, b], mk, sp)
            if abs(mk - sp) > 1e-5 * top:
                assert ((bits >> b) & 1) == (1 if mk > sp else 0), (key, s, b, mk, sp)
        _, _, _, sig, noise, _ = plan.frame_analyze(buf[s, start:].copy(), float(spb_fsk), b"d" * nb)
        assert np.array_equal(mg[s, :, 1] <= EPS, noise <= EPS), (key, s, mg[s, :, 1], noise)
        checked += 1
    assert checked >= max(2, nstreams // 12), (key, checked)
    PERBIT_MAX[0] = max(PERBIT_MAX[0], worst)
    print("%s: per-bit deviation from the fp64 DFT at most %.3g of the window's signal (all so far: %.3g)"
          % (key, worst, PERBIT_MAX[0]))


# ---------------------------------------------------------------------------------------------------
# the transmitter: every k_tx_synth instance and table placement on random configurations
# ---------------------------------------------------------------------------------------------------
VOLUMES = [1e-5, 0.3, 1.0, 1.7]


def tx_framing(seed):
    rng = np.random.default_rng(seed)
    while True:
        baud = int(rng.choice([45, 110, 300, 600, 1200, 2400]))
        rate = int(rng.choice([8000, 11025, 22050, 48000]))
        if not 4 <= rate / baud <= 400:
            continue
        kw = dict(sample_rate=rate, n_data_bits=int(rng.integers(1, 33)), startbits=int(rng.choice([0, 1, 2])),
                  stopbits=float(rng.choice([0.0, 1.0, 1.5, 2.0])), msb_first=bool(rng.integers(0, 2)),
                  invert_start_stop=bool(rng.integers(0, 2)))
        if rng.integers(0, 2):
            kw["mark"] = float(rng.integers(300, rate // 2 - 100))
            kw["space"] = float(rng.integers(300, rate // 2 - 100))
        return str(baud), kw, bool(rng.integers(0, 2) and kw["n_data_bits"] == 5)


def tx_out(n, stride, dtype, align, sentinel):
    """an output tensor with `align` rows; the whole allocation (one row before and after) = sentinel"""
    t = torch()
    off = 1 if align == "offset-base" else 0
    flat = t.full(((n + 2) * stride + 2 * off + 8,), sentinel, dtype=dtype, device=dev())
    base = stride + off
    return flat, flat[base:base + n * stride].view(n, stride), base


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,align,lut", TX_ROWS, ids=["%s-%s-lut%d" % r for r in TX_ROWS])
def test_tx_instantiation_on_random_configurations(fmt, align, lut):
    """TxEngine.text_batch for one (type, row alignment, --lut): random rates, baud rates, tones, 1..32
    data bits, start and stop bits (1.5 included), bit order, start/stop inversion, both encoders and
    the four volumes; ragged texts (0 included), then an empty tick with FSK_B200_TX_IDLE_IF_EMPTY.
    Equal to the oracle's transmitter (bit-exact for lut > 0, 1 ulp / 1 LSB for lut = 0); nothing is
    written outside [0, count) of a row."""
    t = torch()
    float_samples = fmt == "f32"
    dtype = t.float32 if float_samples else t.int16
    sentinel = -7.25 if float_samples else -7777
    nconf = 4
    for c in range(nconf):
        seed = 600 + 10 * TX_LUTS.index(lut) + c + (0 if float_samples else 5000)
        mode, kw, baudot = tx_framing(seed)
        rng = np.random.default_rng(seed)
        vol = VOLUMES[(c + TX_LUTS.index(lut)) % len(VOLUMES)]
        names = dict(mark="f_mark", space="f_space", startbits="nstartbits", stopbits="nstopbits")
        rx = mm.rx_config_for_mode(mode, kw["sample_rate"], **{names.get(k, k): v for k, v in kw.items()
                                                              if k != "sample_rate"})
        cfg = mm.tx_config_from(rx)
        m = orc.Mode(mode, **kw)
        kind = mm.ENCODE_BAUDOT if baudot else mm.ENCODE_ASCII8
        te = mm.TxEngine(cfg, kind, vol, lut, float_samples)
        okind = "baudot" if baudot else "ascii8"
        n, maxlen = 9, 12
        texts = [bytes(int(x) for x in rng.integers(1, 256, 0 if i == 1 else int(rng.integers(1, maxlen + 1))))
                 for i in range(n)]
        tstride = max(len(x) for x in texts)
        tb = np.zeros((n, tstride), np.uint8)
        for i, x in enumerate(texts):
            tb[i, :len(x)] = np.frombuffer(x, np.uint8)
        need = max(te.max_samples(tstride, 0), te.max_samples(tstride, mm.TX_IDLE_IF_EMPTY | mm.TX_FINAL))
        stride = need | 1 if align == "odd-stride" else (need + 7) & ~7
        flat, out, base = tx_out(n, stride, dtype, align, sentinel)
        assert (out.data_ptr() % 16 == 0 and (stride * out.element_size()) % 16 == 0) == (align == "aligned")
        states = te.new_states(n, dev())
        lens = t.tensor([len(x) for x in texts], dtype=t.int32).to(dev())
        _, cnt = te.text_batch(t.from_numpy(tb).to(dev()), lens, states, 0, out=out)
        sync()
        c1 = cnt.cpu().numpy().copy()
        a1 = flat.cpu().numpy().copy()
        # an empty tick: the idle tone where a byte went out, then the trailer
        zero = t.zeros((n,), dtype=t.int32, device=dev())
        flat.fill_(sentinel)
        _, cnt2 = te.text_batch(t.from_numpy(tb).to(dev()), zero, states, mm.TX_IDLE_IF_EMPTY | mm.TX_FINAL, out=out)
        sync()
        c2 = cnt2.cpu().numpy().copy()
        a2 = flat.cpu().numpy().copy()
        for i, x in enumerate(texts):
            want = txorc.tx_events(m, list(x) + [txorc.IDLE], okind, vol, lut, float_samples)
            got = []
            for a, cn in ((a1, c1[i]), (a2, c2[i])):
                r = a[base + i * stride: base + (i + 1) * stride]
                assert (r[cn:] == sentinel).all(), (mode, kw, i, "wrote past its count")
                got.append(r[:cn])
            got = np.concatenate(got)
            got = got.astype(np.float32) if float_samples else got.astype(np.float32) * np.float32(1 / 32768)
            assert got.size == want.size, (mode, kw, vol, lut, i, got.size, want.size)
            if lut > 0:
                assert np.array_equal(got, want), (mode, kw, vol, lut, i)
            elif float_samples:
                # the sine within 1 ulp; at a volume other than 1 the product is rounded once more
                ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
                ulps[(got == 0) & (want == 0)] = 0
                assert ulps.max(initial=0) <= (1 if vol == 1.0 else 2), (mode, kw, vol, i)
            else:
                assert np.abs(np.round(got * 32768.0) - np.round(want * 32768.0)).max(initial=0) <= 1, (mode, kw, vol, i)
        for a in (a1, a2):
            assert (a[:base] == sentinel).all() and (a[base + n * stride:] == sentinel).all(), "wrote outside the rows"


@pytest.mark.gpu
@pytest.mark.parametrize("lut", [16, 1000, 8193], ids=lambda v: "lut%d" % v)
def test_tx_batch_odd_stride(lut):
    """fsk_b200_tx_batch (the word encoder) with an odd row stride: scalar stores, bit-exact."""
    t = torch()
    mode, kw, _ = tx_framing(700 + lut)
    m = orc.Mode(mode, **kw)
    names = dict(mark="f_mark", space="f_space", startbits="nstartbits", stopbits="nstopbits")
    cfg = mm.tx_config_from(mm.rx_config_for_mode(mode, kw["sample_rate"], **{names.get(k, k): v for k, v in kw.items()
                                                                               if k != "sample_rate"}))
    rng = np.random.default_rng(lut)
    n, nwords = 17, 6
    words = rng.integers(0, 1 << m.n_data_bits, (n, nwords), dtype=np.uint64).astype(np.uint32)
    ref0 = orc.tx_words(m, words[0], 1.0, lut, True)
    nout = ref0.size + 5
    stride = nout | 1
    table = t.from_numpy(mm.sin_table(lut)).to(dev())
    out = t.full((n, stride), -3.0, dtype=t.float32, device=dev())
    mm.tx_batch(cfg, t.from_numpy(words.astype(np.int32)).to(dev()), nout, table=table, out=out, stride=stride)
    sync()
    o = out.cpu().numpy()
    for s in range(n):
        want = np.zeros(nout, np.float32)
        w = orc.tx_words(m, words[s], 1.0, lut, True)
        want[:w.size] = w
        assert np.array_equal(o[s, :nout], want), (mode, kw, s)
        assert (o[s, nout:] == -3.0).all(), s


# ---------------------------------------------------------------------------------------------------
# CPU: the screen itself, and the oracle's transmitter pinned at the new table lengths and volumes
# ---------------------------------------------------------------------------------------------------
def _same_result(a, b):
    return a["frames"] == b["frames"] and a["reports"] == b["reports"]


def test_tie_screen_replays_the_oracle_exactly():
    """delta = 0: the screen's search is the oracle's, records and reports bit for bit, on every golden
    vector and on 64 random framings."""
    import golden_util as gu
    import refcases
    for case in refcases.EVERY:
        g = gu.load(case["name"])
        _, rx = gu.modes(case)
        a = gu.audio(case, g)
        if case["rxnoise"]:
            a = (a + np.float32(-0.5) * np.float32(np.float32(case["rxnoise"]) * 2)).astype(np.float32)
        got, _ = tie_screen.run(rx, a, delta=0.0)
        assert _same_result(got, orc.rx_run(rx, a, literal=False)), case["name"]
    for seed in range(64):
        rng = np.random.default_rng(1000 + seed)
        mode, kw = emu_fuzz.random_mode(rng)
        m = orc.Mode(mode, **kw)
        words = rng.integers(0, 1 << m.n_data_bits, int(rng.integers(6, 18)), dtype=np.uint64).astype(np.uint32)
        x = np.concatenate([np.zeros(int(rng.integers(0, 3 * int(m.derived().nsamples_per_bit) + 1)), np.float32),
                            orc.tx_words(m, words, float(rng.uniform(0.3, 1.0)), 4096, True)])
        x = (x + np.float32(0.01) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        got, _ = tie_screen.run(m, x, delta=0.0)
        assert _same_result(got, orc.rx_run(m, x, literal=False)), (mode, kw)


def test_tie_screen_flags_a_constructed_tie():
    """With confidence_threshold set to the oracle's exact float32 confidence of its weakest frame, the rx loop's
    `confidence <= threshold` (src/minimodem.c:1292) sits on the tie: the stream is not robust.  The same
    stream at the default threshold is."""
    import golden_util as gu
    import refcases
    case = refcases.BY_NAME["small-1200"]
    g = gu.load(case["name"])
    _, rx = gu.modes(case)
    a = gu.audio(case, g)
    a = (a + np.float32(0.02) * np.random.default_rng(1).standard_normal(a.size).astype(np.float32)).astype(np.float32)
    want, robust = tie_screen.screen(rx, a)
    assert robust and len(want["frames"]) > 4
    c = min(f[1] for f in want["frames"] if np.isfinite(f[1]))       # the weakest frame: the others stay above
    tied = orc.Mode(case["rx_mode"], **dict(case["rx_mkw"], confidence=float(c)))
    assert tied.confidence_threshold == c
    _, robust = tie_screen.screen(tied, a)
    assert not robust


def test_the_screen_rejects_few_of_the_random_cases():
    """At most 10 % of the streams the rx tests draw are screened out, per family of instantiations
    (full sizes, as on the device)."""
    fams = {}
    for key, row in RX_TABLE.items():
        fam = "generic" if key[0] == "generic" else "mode%d" % key[3]
        fams.setdefault(fam, set()).add((row["cls"], row["n"]))
    import conftest
    if conftest.EMU_DEVICE is not None:
        pytest.skip("counted at the device's sizes, without the emulation")
    for fam, cases in sorted(fams.items()):
        bad = total = 0
        for cls, n in sorted(cases):
            screened = rx_case(cls, n)[5]
            bad += sum(1 for _, r in screened if not r)
            total += len(screened)
        print("%s: %d of %d random streams screened out" % (fam, bad, total))
        assert bad <= 0.1 * total, (fam, bad, total)


PIN = [("1200", {}, 1000, 0.3, False), ("300", dict(stopbits=1.5), 8193, 1.7, True),
       ("rtty", dict(sample_rate=8000), 4095, 1e-5, False), ("600", dict(sample_rate=22050), 65536, 1.0, True),
       ("1200", dict(startbits=2), 16384, 1.7, False), ("110", dict(sample_rate=11025), 16, 0.3, True)]


@pytest.mark.ref
@pytest.mark.parametrize("mode,kw,lut,vol,flt", PIN, ids=["%s-lut%d-vol%g%s" % (p[0], p[2], p[3], "-float" if p[4] else "")
                                                      for p in PIN])
def test_tx_oracle_matches_the_reference_cli_at_new_table_lengths(mode, kw, lut, vol, flt, tmp_path):
    """The oracle's transmitter against the unmodified reference CLI's `--tx --lut=N --volume V`, by hash,
    at table lengths that are not powers of two or that leave shared memory on the device, and at the
    volumes of the device tests."""
    import hashlib
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import read_wav
    m = orc.Mode(mode, **kw)
    args = [mode, "--samplerate", str(m.sample_rate), "--lut=%d" % lut, "--volume", repr(vol)]
    if "stopbits" in kw:
        args += ["--stopbits", str(kw["stopbits"])]
    if "startbits" in kw:
        args += ["--startbits", str(kw["startbits"])]
    if flt:
        args.append("--float-samples")
    text = bytes(np.random.default_rng(lut).integers(32, 127, 12, dtype=np.uint8)) + b"\n"
    wav = str(tmp_path / "x.wav")
    subprocess.run([orc.REF_CLI, "--tx", "--file", wav] + args, input=text, check=True)
    audio, _, _ = read_wav(wav)
    kind = "baudot" if mode == "rtty" else "ascii8"
    mine = txorc.tx_events(m, list(text), kind, vol, lut, flt)
    assert mine.size == audio.size, (args, mine.size, audio.size)
    assert hashlib.sha256(mine.tobytes()).digest() == hashlib.sha256(audio.astype(np.float32).tobytes()).digest(), args
