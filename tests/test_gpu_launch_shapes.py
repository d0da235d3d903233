"""The rx records do not depend on how a stream is launched: ring depth, warps per block, the stream's
place in the batch and what its neighbours do.

Ring depth (RxEngine.tune(ring_floats=...) / FSK_B200_RING), warps per block (warps_per_block /
FSK_B200_WPB) and batch position change when and where samples are copied into shared memory, never the
order of a sum:
- the per-candidate window sums are indexed from the window start (or, sliding, from the candidate
  offset), never from the ring offset;
- the shared-segment walk order (LaneWinM.rot0) depends on the geometry alone;
- the prefix table is cut into pieces counted from the search position's 16-byte piece, and every ring is
  a whole number of 128-float blocks.
The int16 rows widen each block in place before the search reads it, the TMA fill lands the same values
as the cp.async fill, and the tone and auto calls only add a per-stream table that is filled from the
unit-circle table at fixed indices.  So at a fixed (G, W, L, MODE) the records and every byte of
fsk_b200_stream_state (stat_candidates, stat_searches and reserved included) must be identical across
these knobs, and the tests below hold every family to exactly that.

A deeper ring turns on the look-ahead fill (Shape::lookahead = min(slack, the largest advance)): the
copies for the next iteration run up to a whole advance ahead of the one being searched.  Every run reads
last_kernel() and checks that the launch is the one the row asks for -- kernel family, (G, W, L),
threads=, ring= and lookahead= -- so a request the launcher overrode fails instead of passing on the
default shape.

Under FSK_B200_EMU=1 (tests/emu) the file runs on the host emulation of the kernels (test_emu_parity.py
runs it with copies landing early and late); the TMA bulk fill is not modelled there and its rows skip."""
import re
import zlib

import numpy as np
import pytest

import autoorc
import minimodem_b200 as mm
import orc
import test_gpu_instantiations as I
import tie_screen

SMEM_MAX = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (and of the emulation)
KNOBS = ("FSK_B200_LANES", "FSK_B200_SPLIT", "FSK_B200_MULTI", "FSK_B200_PREFIX", "FSK_B200_PFX_FILL",
         "FSK_B200_RING", "FSK_B200_WPB", "FSK_B200_NO_SLIDE")
PER_CAND = {"FSK_B200_MULTI": "0", "FSK_B200_PREFIX": "0"}
SHARED = {"FSK_B200_MULTI": "2", "FSK_B200_PREFIX": "0"}

# family -> the call, the rows, the environment, and the kernel it must launch: (last_kernel name, mode,
# fill); `cls` / `n`: the random framing of test_gpu_instantiations.framing that the family also runs
FAMILIES = {
    "per-candidate": dict(call="rx", src="f32", env=PER_CAND, kern=("k_rx", 0, 0), cls="short", n=10),
    "per-candidate-noslide": dict(call="rx", src="f32", env=dict(PER_CAND, FSK_B200_NO_SLIDE="1"),
                                  kern=("k_rx", 0, 0), cls="short", n=12),
    "per-candidate-s16": dict(call="rx", src="s16", env=PER_CAND, kern=("k_rx", 0, 0), cls="short", n=11),
    "shared-segment": dict(call="rx", src="f32", env=SHARED, kern=("k_rx", 2, 0), cls="tile", n=10),
    "shared-segment-s16": dict(call="rx", src="s16", env=SHARED, kern=("k_rx", 2, 0), cls="tile", n=11),
    "prefix-table-tma": dict(call="rx", src="f32", env={"FSK_B200_PREFIX": "1", "FSK_B200_PFX_FILL": "1"},
                             kern=("k_rx", 3, 1), cls="tile", n=8),
    "prefix-table-cp": dict(call="rx", src="f32", env={"FSK_B200_PREFIX": "1", "FSK_B200_PFX_FILL": "0"},
                            kern=("k_rx", 3, 0), cls="tile", n=7),
    "prefix-table-s16": dict(call="rx", src="s16", env={"FSK_B200_PREFIX": "1", "FSK_B200_PFX_FILL": "0"},
                             kern=("k_rx", 3, 0), cls="tile", n=11),
    "tones": dict(call="tones", src="f32", env={}, kern=("k_rx_tones", 0, 0)),
    "tones-s16": dict(call="tones", src="s16", env={}, kern=("k_rx_tones", 0, 0)),
    "auto": dict(call="auto", src="f32", env={}, kern=("k_rx_auto", 0, 0)),
    "auto-s16": dict(call="auto", src="s16", env={}, kern=("k_rx_auto", 0, 0)),
}
PRESETS = [("1200", 48000), ("300", 48000), ("rtty", 8000), ("same", 48000)]
# the presets a family cannot launch, with the reason
NOT_LAUNCHED = {
    ("shared-segment", "same"): "SAME's 10 windows have no shared-segment plan: the per-candidate kernel runs",
    ("shared-segment-s16", "same"): "as the float rows",
    ("tones", "same"): "SAME's shape (G=8, W=4, L=4) has no per-stream tone build (AUTO_COMBOS)",
    ("tones-s16", "same"): "as the float rows",
    ("auto", "same"): "as the tone call",
    ("auto-s16", "same"): "as the tone call",
}

LK = re.compile(r"(k_rx|k_rx_auto|k_rx_tones)<G=(\d+),W=(\d+),L=(\d+),mode=(\d)\([a-z-]+\),fill=(\d),src=([a-z0-9,]+)> "
                r"threads=(\d+) ring=(\d+) smem=(\d+) blocks=(\d+) lookahead=(\d+)$")


def launch(eng):
    """last_kernel() as a dict"""
    s = eng.last_kernel()
    m = LK.match(s)
    assert m, s
    k = dict(zip(("name", "G", "W", "L", "mode", "fill", "src", "threads", "ring", "smem", "blocks", "lookahead"),
                 m.groups()))
    for f in k:
        if f not in ("name", "src"):
            k[f] = int(k[f])
    k["text"] = s
    return k


def shape(k):
    return (k["name"], k["G"], k["W"], k["L"], k["mode"], k["fill"], k["src"])


def max_advance(p):
    """the largest advance of the rx loop, as the launcher bounds the look-ahead with it"""
    return max(p.try_max_nocarrier, p.try_max_carrier) - 1 + p.frame_nsamples


def set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)            # read when the engine is created


# ---------------------------------------------------------------------------------------------------
# cases: streams from the oracle's transmitter
# ---------------------------------------------------------------------------------------------------
_CASES = {}


def _pcm(a):
    return np.clip(np.round(a * 32768.0), -32768, 32767).astype(np.int16)


def case(fam, which):
    """(engine factory, streams, lengths, per-stream tone bands or None, oracle Mode) for a family and a
    preset (mode, rate) or "random".  6 streams: ragged lead-ins, sigma = 0.01 noise (1e-4 for the auto
    call, whose streams start with silence longer than the deepest ring), every third stream drops the
    carrier and finds it again, the last one is cut mid-frame.  Computed once per (call, which)."""
    f = FAMILIES[fam]
    key = (f["call"], f.get("cls"), f.get("n"), which)
    if key in _CASES:
        return _CASES[key]
    rng = np.random.default_rng(zlib.crc32(repr(key).encode()))
    if which == "random":
        mode, kw, exp = I.framing(f["cls"], f["n"], 7000 + f["n"])
        m = I.oracle_mode(mode, kw, exp)
        make = lambda: I.engine(mode, kw, exp)
    else:
        mode, rate = which
        m = orc.Mode(mode, sample_rate=rate)
        make = lambda: mm.RxEngine.for_mode(mode, rate)
    spb = float(m.derived().nsamples_per_bit)
    streams, bands = [], []
    probe = make()
    p = probe.params
    nb = int(p.nbands)
    for s in range(6):
        if f["call"] == "auto":
            import test_gpu_auto_carrier as AC
            bs = autoorc.b_shift(m)
            parts = [np.zeros(int(rng.integers(20000, 26000)), np.float32), AC.tone_stream(rng, m, bs, nb, 5)]
            if s % 3 == 1:
                parts += [np.zeros(int(rng.uniform(30, 50) * spb), np.float32), AC.tone_stream(rng, m, bs, nb, 4)]
            sigma = 1e-4
        else:
            tm = m
            if f["call"] == "tones":
                import test_gpu_stream_tones as ST
                fm, fs = ST.random_pair(rng, float(m.band_width), nb)
                bands.append([int(v) for v in mm.tone_bands(p, fm, fs)])
                tm = ST.on_pair(m.mode, m.sample_rate, fm, fs)
                tm.__dict__.update({k: v for k, v in m.__dict__.items() if k not in ("mark_f", "space_f")})
            words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
            parts = [np.zeros(int(rng.integers(0, 3 * spb + 1)), np.float32),
                     orc.tx_words(tm, words(int(rng.integers(6, 10))), float(rng.uniform(0.3, 1.0)), 4096, True)]
            if s % 3 == 1:
                parts += [np.zeros(int(rng.uniform(20, 40) * spb), np.float32),
                          orc.tx_words(tm, words(4), float(rng.uniform(0.3, 1.0)), 4096, True)]
            sigma = 0.01
        x = np.concatenate(parts)
        if s == 5:
            x = x[:int(x.size * rng.uniform(0.6, 0.9))]
        x = (x + np.float32(sigma) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
    _CASES[key] = (make, streams, np.array([x.size for x in streams], np.int32), bands or None, m)
    return _CASES[key]


class Run:
    """one call: records per stream (bytes), the states, the auto states and record bands, the launch"""

    def __init__(self, recs, st, extra, k):
        self.recs, self.st, self.extra, self.k = recs, st, extra, k

    def same_as(self, other, what):
        assert self.st.tobytes() == other.st.tobytes(), (what, "states", self.k["text"], other.k["text"])
        for s, (a, b) in enumerate(zip(self.recs, other.recs)):
            assert a == b, (what, "stream %d" % s, self.k["text"], other.k["text"])
        assert self.extra == other.extra, (what, "auto states / bands")

    def nrecs(self):
        return int(self.st["nframes"].sum())


def run(eng, fam, c, max_frames=None, states=None, auto_states=None):
    make, streams, lens, bands, m = c
    f = FAMILIES[fam]
    t = I.torch()
    n = int(lens.max())
    buf = I._rows(streams, n, np.float32, 8)
    if f["src"] == "s16":
        buf = _pcm(buf)
    x = t.from_numpy(buf).to(I.dev())
    le = t.from_numpy(lens).to(I.dev())
    extra = None
    if f["call"] == "rx":
        fr, st = eng.rx_batch(x, nsamples=n, nsamples_each=le, max_frames=max_frames, states=states)
    elif f["call"] == "tones":
        tb = t.from_numpy(np.array(bands, np.int32)).to(I.dev())
        fr, st = eng.rx_batch_tones(x, tb, nsamples=n, nsamples_each=le, max_frames=max_frames, states=states)
    else:
        fr, st, ast, rb = eng.rx_batch_auto(x, nsamples=n, nsamples_each=le, max_frames=max_frames, states=states,
                                            auto_states=auto_states, rec_band=True)
    I.sync()
    fr, sn = mm.frames_to_numpy(fr), mm.states_to_numpy(st)
    recs = [fr[s, :int(sn["nframes"][s])].tobytes() for s in range(len(streams))]
    if f["call"] == "auto":
        rb = rb.cpu().numpy()
        extra = (ast.cpu().numpy().tobytes(), [rb[s, :int(sn["nframes"][s])].tobytes() for s in range(len(streams))])
        return Run(recs, sn.copy(), extra, launch(eng)), st, ast
    return Run(recs, sn.copy(), extra, launch(eng)), st, None


def new_engine(monkeypatch, fam, c, extra_env=None, tune=None):
    f = FAMILIES[fam]
    set_env(monkeypatch, dict(f["env"], **(extra_env or {})))
    eng = c[0]()
    if f["call"] == "auto":
        eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    if tune:
        eng.tune(**tune)
    return eng


def check_family(fam, k):
    name, mode, fill = FAMILIES[fam]["kern"]
    assert (k["name"], k["mode"], k["fill"]) == (name, mode, fill), (fam, k["text"])
    assert k["src"].split(",")[0] == FAMILIES[fam]["src"], (fam, k["text"])
    if fam == "per-candidate":
        assert k["src"] == "f32,slide", k["text"]
    if fam == "per-candidate-noslide":
        assert k["src"] == "f32", k["text"]


def skip_tma(fam):
    if I.emulated() and FAMILIES[fam]["kern"][2] == 1:
        pytest.skip("the host emulation does not model cp.async.bulk / mbarrier")


def ring_for_full_lookahead(base, p):
    """the first ring (whole 128-float blocks) at which lookahead= reaches the largest advance"""
    adv = max_advance(p)
    if base["lookahead"] >= adv:
        return base["ring"]
    return base["ring"] + (adv - base["lookahead"] + 127) // 128 * 128


def per_ring_float(k):
    """shared-memory bytes per ring float of a block of this launch"""
    return 4 * (k["threads"] // 32) * (32 // k["G"])


def deepest_ring(base, want):
    """`want`, or the largest ring below it at which this block still fits in shared memory"""
    room = (SMEM_MAX - base["smem"]) // per_ring_float(base)
    return min(want, base["ring"] + room // 128 * 128)


REPORT = {}


def report(fam, k, nrecs):
    r = REPORT.setdefault(fam, dict(launches=set(), records=0, full=False))
    r["launches"].add("ring=%d lookahead=%d threads=%d" % (k["ring"], k["lookahead"], k["threads"]))
    r["records"] += nrecs


# ---------------------------------------------------------------------------------------------------
# 1. ring depth at a pinned shape
# ---------------------------------------------------------------------------------------------------
FAM_KEYS = list(FAMILIES)
RING_ROWS = [(fam, w) for fam in FAM_KEYS for w in PRESETS + ["random"]
             if not (FAMILIES[fam]["call"] != "rx" and w == "random") and (fam, w[0]) not in NOT_LAUNCHED]


def _rid(r):
    return "%s-%s" % (r[0], r[1] if isinstance(r[1], str) else "%s@%d" % r[1])


@pytest.mark.gpu
@pytest.mark.parametrize("fam,which", RING_ROWS, ids=[_rid(r) for r in RING_ROWS])
def test_ring_depth_does_not_change_the_records(fam, which, monkeypatch):
    """At the default launch's (G, L) -- lanes pinned with tune(), the split with FSK_B200_SPLIT -- and its
    warps per block, rings of R0 + 128, R0 + 256, the first ring whose look-ahead is the largest advance,
    and 4x that (or the deepest ring that still fits the block) give the default run's records and states
    byte for byte, and the launch shows the ring and the look-ahead asked for."""
    skip_tma(fam)
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    base, _, _ = run(eng, fam, c)
    k0 = base.k
    check_family(fam, k0)
    assert base.nrecs() >= 6, (fam, which, k0["text"])
    p = eng.params
    report(fam, k0, base.nrecs())
    # the prefix-table kernel's own choice can exceed the 4 warps tune() takes: pin 4 there
    pin = dict(lanes_per_stream=k0["G"], warps_per_block=min(4, k0["threads"] // 32))
    env = {"FSK_B200_SPLIT": str(k0["L"])}
    if pin["warps_per_block"] != k0["threads"] // 32:
        e1 = new_engine(monkeypatch, fam, c, env, pin)
        got, _, _ = run(e1, fam, c)
        assert shape(got.k) == shape(k0) and got.k["threads"] == 128, got.k["text"]
        got.same_as(base, (fam, which, "4 warps"))
        report(fam, got.k, got.nrecs())
        k0 = got.k
    r_full = ring_for_full_lookahead(k0, p)
    rings = [k0["ring"] + 128, k0["ring"] + 256, r_full, deepest_ring(k0, 4 * r_full)]
    assert rings[-1] >= r_full + 128, (fam, which, rings, k0["text"])
    for ring in rings:
        e2 = new_engine(monkeypatch, fam, c, env, dict(pin, ring_floats=ring))
        got, _, _ = run(e2, fam, c)
        k = got.k
        assert shape(k) == shape(k0) and k["threads"] == k0["threads"], (fam, which, ring, k0["text"], k["text"])
        assert k["ring"] == ring, (fam, ring, k["text"])
        assert k["lookahead"] == min(max_advance(p), k0["lookahead"] + ring - k0["ring"]), (fam, ring, k["text"])
        assert k["smem"] == k0["smem"] + per_ring_float(k0) * (ring - k0["ring"]), (fam, ring, k["text"])
        got.same_as(base, (fam, which, ring))
        report(fam, k, got.nrecs())
        if k["lookahead"] == max_advance(p):
            REPORT[fam]["full"] = True
    print("%s %s: %s; %d records compared byte for byte per run" % (
        fam, which, ", ".join(sorted(REPORT[fam]["launches"])), base.nrecs()))


@pytest.mark.gpu
@pytest.mark.parametrize("fam", ["per-candidate", "shared-segment-s16", "prefix-table-cp", "tones", "auto"])
def test_an_overflowing_call_resumed_on_another_ring_gives_one_pass(fam, monkeypatch):
    """max_frames = 3: the call stops with the output full; the states then continue on an engine with
    a different ring (and look-ahead), in calls of 3 records, and the records joined equal one pass."""
    skip_tma(fam)
    c = case(fam, ("300", 48000) if fam != "tones" else ("1200", 48000))
    eng = new_engine(monkeypatch, fam, c)
    one, _, _ = run(eng, fam, c)
    k0 = one.k
    p = eng.params
    env = {"FSK_B200_SPLIT": str(k0["L"])}
    pin = dict(lanes_per_stream=k0["G"], warps_per_block=min(4, k0["threads"] // 32))
    engines = [eng, new_engine(monkeypatch, fam, c, env, dict(pin, ring_floats=ring_for_full_lookahead(k0, p)))]
    joined = [b""] * len(c[1])
    states = auto_states = None
    launches = set()
    for i in range(200):
        e = engines[i % 2]
        got, states, auto_states = run(e, fam, c, max_frames=3, states=states, auto_states=auto_states)
        launches.add((got.k["ring"], got.k["lookahead"]))
        assert shape(got.k) == shape(k0), got.k["text"]
        for s in range(len(joined)):
            joined[s] += got.recs[s]
        if (got.st["done"] == 1).all():
            break
        st = got.st.copy()
        st["nframes"][:] = 0            # the records of the next call start at its row's first slot
        states = I.torch().from_numpy(st.view(np.int32).reshape(len(st), -1).copy()).to(I.dev())
    assert len(launches) == 2 and i >= 3, (launches, i)
    assert joined == one.recs, fam
    st = got.st.copy()
    st["nframes"] = one.st["nframes"]
    assert st.tobytes() == one.st.tobytes(), fam
    print("%s: %d calls on rings %s, %d records equal to one pass" % (fam, i + 1, sorted(launches), one.nrecs()))


# ---------------------------------------------------------------------------------------------------
# 2. a ring deep enough to change the lane count
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which,env", [(("1200", 48000), PER_CAND), (("same", 48000), PER_CAND),
                                       (("300", 48000), SHARED)], ids=["1200", "same", "300-shared-segment"])
def test_a_deep_ring_with_free_lanes_moves_g_and_keeps_the_oracle_records(which, env, monkeypatch):
    """lanes_per_stream left at 0: the launcher derives G from the streams that fit per SM, so a ring 2048
    floats deeper raises G -- the L-way combine then sums in another order, so the records are held to the
    screened oracle (as test_gpu_instantiations.compare_rx does), not to the default run."""
    fam = "per-candidate" if env is PER_CAND else "shared-segment"
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    base, _, _ = run(eng, fam, c)
    e2 = new_engine(monkeypatch, fam, c, tune=dict(ring_floats=base.k["ring"] + 2048))
    got, _, _ = run(e2, fam, c)
    k = got.k
    assert k["ring"] == base.k["ring"] + 2048 and k["mode"] == base.k["mode"], k["text"]
    assert k["G"] > base.k["G"], (base.k["text"], k["text"])
    make, streams, lens, _, m = c
    screened = [tie_screen.screen(m, x) for x in streams]
    ocase = (m.mode, {}, None, m, streams, screened)
    I.compare_rx(ocase, [np.frombuffer(r, mm.FRAME_DTYPE) for r in got.recs], got.st, k["text"])
    print("%s: %s -> %s; %d of %d streams held to the oracle's records" % (
        fam, base.k["text"], k["text"], sum(1 for _, r in screened if r), len(screened)))


# ---------------------------------------------------------------------------------------------------
# 3. warps per block
# ---------------------------------------------------------------------------------------------------
WPB_ROWS = [(fam, w) for fam in FAM_KEYS for w in (("1200", 48000), ("300", 48000))
            if not (fam.startswith("tones") and w[0] == "300")]


@pytest.mark.gpu
@pytest.mark.parametrize("fam,which", WPB_ROWS, ids=[_rid(r) for r in WPB_ROWS])
def test_warps_per_block_do_not_change_the_records(fam, which, monkeypatch):
    """tune(warps_per_block=w), w = 1..4, and w = 3 at the ring of a full look-ahead: threads = 32 w and
    the default run's records and states byte for byte.  The prefix-table kernel honours w only under
    FSK_B200_PREFIX=1, which its families set."""
    skip_tma(fam)
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    base, _, _ = run(eng, fam, c)
    k0 = base.k
    check_family(fam, k0)
    env = {"FSK_B200_SPLIT": str(k0["L"])}
    r_full = ring_for_full_lookahead(k0, eng.params)
    rows = [dict(warps_per_block=w) for w in (1, 2, 3, 4)] + [dict(warps_per_block=3, ring_floats=r_full)]
    smem = {}
    for tv in rows:
        e2 = new_engine(monkeypatch, fam, c, env, dict(tv, lanes_per_stream=k0["G"]))
        got, _, _ = run(e2, fam, c)
        k = got.k
        assert shape(k) == shape(k0), (fam, tv, k0["text"], k["text"])
        assert k["ring"] == tv.get("ring_floats", k0["ring"]), (tv, k["text"])
        w = tv["warps_per_block"]
        if len(tv) == 1:
            smem[w] = k["smem"]
        # the block at w warps from the blocks at 1 and 2 warps (both fit at the default ring): the
        # streams' slots scale with the warps
        need = 0
        if w > 2:
            per_warp = smem[2] - smem[1]
            need = smem[1] - per_warp + w * (per_warp + (k["ring"] - k0["ring"]) * 4 * (32 // k0["G"]))
        if need <= SMEM_MAX:
            assert k["threads"] == 32 * w, (fam, tv, k["text"])
        else:
            assert k["threads"] < 32 * w, (fam, tv, k["text"])        # fewer warps first, the same G
        got.same_as(base, (fam, which, tv))
        report(fam, k, got.nrecs())
    print("%s %s: %s; %d records compared byte for byte per run" % (
        fam, which, ", ".join(sorted(REPORT[fam]["launches"])), base.nrecs()))


@pytest.mark.gpu
def test_the_prefix_table_kernel_ignores_warps_per_block_unless_forced(monkeypatch):
    """Without FSK_B200_PREFIX=1 the prefix-table kernel keeps its own warps per block for every w."""
    fam = "prefix-table-cp"
    c = case(fam, ("300", 48000))
    set_env(monkeypatch, {"FSK_B200_PFX_FILL": "0"})
    eng = c[0]()
    base, _, _ = run(eng, fam, c)
    assert base.k["mode"] == 3, base.k["text"]
    seen = set()
    for w in (1, 2, 3, 4):
        e2 = c[0]()
        e2.tune(warps_per_block=w)
        got, _, _ = run(e2, fam, c)
        assert got.k["threads"] == base.k["threads"] and shape(got.k) == shape(base.k), got.k["text"]
        got.same_as(base, w)
        seen.add(w * 32 == base.k["threads"])
    assert False in seen


# ---------------------------------------------------------------------------------------------------
# 4. fallbacks
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
def test_a_ring_too_large_for_one_stream_falls_back_to_the_generic_kernel(src, monkeypatch):
    """A ring that does not fit even one G = 32 stream: the generic kernel (ring=0, no look-ahead), and the
    screened oracle's records."""
    fam = "per-candidate" if src == "f32" else "per-candidate-s16"
    c = case(fam, ("1200", 48000))
    eng = new_engine(monkeypatch, fam, c, tune=dict(ring_floats=SMEM_MAX // 4 + 128))
    got, _, _ = run(eng, fam, c)
    k = got.k
    assert (k["mode"], k["G"], k["ring"], k["lookahead"]) == (1, 32, 0, 0), k["text"]
    assert "mode=1(generic)" in k["text"] and k["src"] == src, k["text"]
    make, streams, lens, _, m = c
    if src == "s16":
        streams = [_pcm(x).astype(np.float32) / np.float32(32768.0) for x in streams]
    screened = [tie_screen.screen(m, x) for x in streams]
    I.compare_rx((m.mode, {}, None, m, streams, screened), [np.frombuffer(r, mm.FRAME_DTYPE) for r in got.recs],
                 got.st, k["text"])


@pytest.mark.gpu
def test_a_ring_that_leaves_no_room_for_the_sliding_table_drops_slide(monkeypatch):
    """The sliding fine search stages an extended tone table; a ring that fits the block only without it
    launches without `slide`, and that run equals an FSK_B200_NO_SLIDE=1 run bit for bit (sliding rounds
    differently, DESIGN.md 3, so the sliding run is not the reference)."""
    c = case("per-candidate", ("1200", 48000))
    pin = dict(lanes_per_stream=32, warps_per_block=1)
    slide = new_engine(monkeypatch, "per-candidate", c, tune=pin)
    a, _, _ = run(slide, "per-candidate", c)
    flat = new_engine(monkeypatch, "per-candidate-noslide", c, tune=pin)
    b, _, _ = run(flat, "per-candidate-noslide", c)
    assert a.k["src"] == "f32,slide" and b.k["src"] == "f32", (a.k["text"], b.k["text"])
    extra = a.k["smem"] - b.k["smem"]
    step = per_ring_float(b.k) * 128
    assert extra > step, (extra, step)
    # the first ring whose block fits without the extension but not with it
    blocks = (SMEM_MAX - extra - b.k["smem"]) // step + 1
    ring = b.k["ring"] + 128 * blocks
    assert b.k["smem"] + step * blocks <= SMEM_MAX < b.k["smem"] + step * blocks + extra
    e1 = new_engine(monkeypatch, "per-candidate", c, tune=dict(pin, ring_floats=ring))
    got, _, _ = run(e1, "per-candidate", c)
    e2 = new_engine(monkeypatch, "per-candidate-noslide", c, tune=dict(pin, ring_floats=ring))
    want, _, _ = run(e2, "per-candidate-noslide", c)
    assert got.k["src"] == "f32" and shape(got.k) == shape(b.k) and got.k["ring"] == ring, got.k["text"]
    assert want.k["text"] == got.k["text"]
    got.same_as(want, "slide dropped")
    got.same_as(b, "no slide, ring %d" % ring)


# ---------------------------------------------------------------------------------------------------
# 5. neighbours
# ---------------------------------------------------------------------------------------------------
NEIGHBOUR_ROWS = [("per-candidate", 4), ("per-candidate", 8), ("per-candidate", 16), ("per-candidate", 32),
                  ("shared-segment", 0), ("prefix-table-cp", 0), ("tones", 0), ("auto", 0)]


def _nb_case(fam):
    """target streams, and one row of every kind of neighbour: (samples, length, state in, tone pair)"""
    which = ("300", 48000) if fam in ("shared-segment", "prefix-table-cp") else ("1200", 48000)
    make, streams, lens, bands, m = case(fam, which)
    rng = np.random.default_rng(zlib.crc32(fam.encode()))
    p = make().params
    zero = np.zeros(1, mm.STATE_DTYPE)[0]
    pair = lambda s: bands[s] if bands else None
    targets = [(streams[s], int(lens[s]), zero, pair(s)) for s in (0, 1, 5)]
    done = np.zeros(1, mm.STATE_DTYPE)[0]
    done["pos"], done["done"], done["nframes"], done["carrier"], done["track_amplitude"] = 777, 1, 3, 1, 0.25
    cut = int(lens[2]) // 2
    long = np.concatenate([streams[3]] * 4)
    noise = (np.float32(0.3) * rng.standard_normal(int(lens[4]) // 3)).astype(np.float32)
    nbrs = [("done", streams[2], int(lens[2]), done, pair(2)),
            ("empty", streams[2], 0, zero, pair(2)),
            ("short", streams[2], int(p.expect_nsamples) - 1, zero, pair(2)),
            ("noise", noise, noise.size, zero, pair(4)),
            ("resumed", streams[2], int(lens[2]), ("resume", cut), pair(2)),
            ("overflow", long, long.size, zero, pair(3))]
    if fam == "tones":
        nbrs.append(("invalid-pair", streams[2], int(lens[2]), zero, [int(p.nbands), 5]))
    if fam == "auto":
        nbrs.append(("silence", np.zeros(1, np.float32), None, zero, None))
    return make, m, targets, nbrs


def _batch(eng, fam, rows, max_frames):
    """rows: (samples, length or None for the whole stride, state) -> (records, states, sentinel left)"""
    t = I.torch()
    n = max(max(r[0].size for r in rows), max(r[1] or 0 for r in rows))
    stride = (n + 7) & ~7
    buf = np.zeros((len(rows), stride), np.float32)
    lens = np.zeros(len(rows), np.int32)
    st = np.zeros(len(rows), mm.STATE_DTYPE)
    for i, (x, ln, s0, _) in enumerate(rows):
        buf[i, :x.size] = x
        lens[i] = stride if ln is None else ln
        st[i] = s0
    x = t.from_numpy(buf).to(I.dev())
    le = t.from_numpy(lens).to(I.dev())
    states = t.from_numpy(st.view(np.int32).reshape(len(rows), -1).copy()).to(I.dev())
    frames = t.full((len(rows), max_frames, 5), 0x5A5A5A5A, dtype=t.int32).to(I.dev())
    call = FAMILIES[fam]["call"]
    if call == "rx":
        fr, so = eng.rx_batch(x, nsamples=stride, nsamples_each=le, max_frames=max_frames, frames=frames, states=states)
    elif call == "tones":
        tb = t.from_numpy(np.array([r[3] for r in rows], np.int64).astype(np.uint32).view(np.int32)).to(I.dev())
        fr, so = eng.rx_batch_tones(x, tb, nsamples=stride, nsamples_each=le, max_frames=max_frames, frames=frames,
                                    states=states)
    else:
        fr, so, _ = eng.rx_batch_auto(x, nsamples=stride, nsamples_each=le, max_frames=max_frames, frames=frames,
                                      states=states)
    I.sync()
    raw = fr.cpu().numpy()
    fr, so = mm.frames_to_numpy(fr), mm.states_to_numpy(so)
    out = []
    for i in range(len(rows)):
        out.append((fr[i, :int(so["nframes"][i])].tobytes(), so[i].tobytes(), bool((raw[i] == 0x5A5A5A5A).all())))
    return out, launch(eng)


@pytest.mark.gpu
@pytest.mark.parametrize("fam,G", NEIGHBOUR_ROWS, ids=["%s-G%d" % r if r[1] else r[0] for r in NEIGHBOUR_ROWS])
def test_a_streams_records_do_not_depend_on_its_place_or_its_neighbours(fam, G, monkeypatch):
    """A few target streams, each run alone, then placed at every group slot of every warp of the first
    block and in the last, partial block of a batch of a few hundred rows whose other rows are
    neighbours: a stream that is done on entry, a zero-length row, a row shorter than expect_nsamples,
    pure noise, a stream resumed from a mid-stream state, a long stream that alone overflows max_frames,
    an invalid tone pair (tone call), silence as long as the batch (auto call).  Every row's records and
    state equal its lone run byte for byte; the done and invalid-pair rows come back untouched."""
    make, m, targets, nbrs = _nb_case(fam)
    env = dict(FAMILIES[fam]["env"])

    def engine():
        set_env(monkeypatch, env)
        e = make()
        if FAMILIES[fam]["call"] == "auto":
            e.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
        if G:
            e.tune(lanes_per_stream=G)
        return e

    eng = engine()
    # the lone runs; max_frames: every target fits, the long neighbour does not
    mf = 1
    for x, ln, s0, bp in targets:
        r, k1 = _batch(eng, fam, [(x, ln, s0, bp)], 4096)
        mf = max(mf, len(r[0][0]) // mm.FRAME_DTYPE.itemsize)
    mf += 2
    lone_t = [_batch(eng, fam, [t_], mf)[0][0] for t_ in targets]
    # resumed neighbour: its state after the first half of its row
    rows_n = []
    for name, x, ln, s0, bp in nbrs:
        if isinstance(s0, tuple):
            r, _ = _batch(eng, fam, [(x, s0[1], np.zeros(1, mm.STATE_DTYPE)[0], bp)], mf)
            s0 = np.frombuffer(r[0][1], mm.STATE_DTYPE)[0].copy()
            s0["done"], s0["nframes"] = 0, 0
        rows_n.append((name, (x, ln, s0, bp)))
    lone_n = {}
    for name, row in rows_n:
        if name == "silence":
            continue
        lone_n[name] = _batch(eng, fam, [row], mf)[0][0]
    assert len(lone_n["overflow"][0]) // mm.FRAME_DTYPE.itemsize == mf, "the long neighbour must fill max_frames"
    k = launch(eng)
    assert k["G"] == (G or k["G"]), k["text"]
    spb = (k["threads"] // 32) * (32 // k["G"])        # streams per block
    part = max(1, spb // 2)                             # rows in the last, partial block
    nrows = max(5 * spb, 300 // spb * spb) + part
    layout = [None] * nrows
    targ_at = sorted(set(list(range(spb)) + [nrows - part, nrows - 1]))
    for j, i in enumerate(targ_at):
        layout[i] = ("t", j % len(targets))
    names = [nm for nm, _ in rows_n]
    j = 0
    for i in range(nrows):
        if layout[i] is None:
            layout[i] = ("n", names[j % len(names)])
            j += 1
    rows = [targets[v] if kind == "t" else dict(rows_n)[v] for kind, v in layout]
    if fam == "auto":
        # the silence row: as long as the batch
        rows = [(r[0], None, r[2], r[3]) if layout[i] == ("n", "silence") else r for i, r in enumerate(rows)]
    got, kb = _batch(eng, fam, rows, mf)
    assert shape(kb) == shape(k) and kb["threads"] == k["threads"], (k["text"], kb["text"])
    assert kb["blocks"] == (nrows + spb - 1) // spb and nrows % spb, kb["text"]
    checked = 0
    for i, (kind, v) in enumerate(layout):
        recs, st, untouched = got[i]
        if kind == "t":
            assert (recs, st) == lone_t[v][:2], (fam, G, "target", v, "row", i, "slot", i % spb, kb["text"])
        elif v == "silence":
            s = np.frombuffer(st, mm.STATE_DTYPE)[0]
            assert recs == b"" and s["done"] == 1, (fam, "silence row", i)
        else:
            assert (recs, st) == lone_n[v][:2], (fam, G, "neighbour", v, "row", i, kb["text"])
            if v in ("done", "invalid-pair"):
                assert untouched and st == rows[i][2].tobytes(), (fam, v, i)
        checked += len(recs) // mm.FRAME_DTYPE.itemsize
    print("%s G=%s: %s, %d rows (%d per block), %d records compared byte for byte" % (
        fam, G or "default", kb["text"], nrows, spb, checked))


# ---------------------------------------------------------------------------------------------------
# 6. tune() itself
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_tune_refuses_bad_values_and_keeps_the_previous_tuning(monkeypatch):
    """-EINVAL for ring_floats 1..127, lanes_per_stream 2, 3 or 64, warps_per_block 5 or -1; after a refused
    call the previous tuning stays (the same launch, the same records); tune(0, 0, 0) restores the default;
    a tune() between two calls on one engine takes effect at the next call."""
    fam = "per-candidate"
    c = case(fam, ("1200", 48000))
    eng = new_engine(monkeypatch, fam, c)
    base, _, _ = run(eng, fam, c)
    eng.tune(lanes_per_stream=16, warps_per_block=3, ring_floats=base.k["ring"] + 384)
    tuned, _, _ = run(eng, fam, c)
    assert (tuned.k["G"], tuned.k["threads"], tuned.k["ring"]) == (16, 96, base.k["ring"] + 384), tuned.k["text"]
    bad = [dict(ring_floats=r) for r in (1, 2, 64, 127)] + [dict(lanes_per_stream=v) for v in (2, 3, 64)]
    bad += [dict(warps_per_block=v) for v in (5, -1)]
    for tv in bad:
        with pytest.raises(RuntimeError, match="-22|EINVAL|must"):
            eng.tune(**tv)
        again, _, _ = run(eng, fam, c)
        assert again.k["text"] == tuned.k["text"], (tv, again.k["text"])
        again.same_as(tuned, tv)
    eng.tune(0, 0, 0)
    back, _, _ = run(eng, fam, c)
    assert back.k["text"] == base.k["text"]
    back.same_as(base, "tune(0, 0, 0)")


@pytest.mark.gpu
def test_every_family_reached_a_full_look_ahead():
    """Runs after the ring-depth tests: per family, the launches seen and the records compared byte for
    byte; every family that ran had a launch whose look-ahead is its largest advance."""
    if not REPORT:
        pytest.skip("no ring-depth test ran in this session")
    for fam, r in sorted(REPORT.items()):
        print("%s: %d records compared; %s" % (fam, r["records"], ", ".join(sorted(r["launches"]))))
        assert r["full"], (fam, "no launch with a full look-ahead")
