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
import zlib

import numpy as np
import pytest

import minimodem_b200 as mm
import tie_screen
from gpudev import dev, pcm, state_rows, torch, upload
from rxcases import shape_case as case
from rxfam import (FAMILIES, NOT_LAUNCHED, PER_CAND, PRESETS, SHAPE_FAMILIES, SHARED, SMEM_MAX, call, check_family,
                   compare_rx, launch, new_engine, set_env, skip_tma)


def shape(k):
    return (k["name"], k["G"], k["W"], k["L"], k["mode"], k["fill"], k["src"])


def max_advance(p):
    """the largest advance of the rx loop, as the launcher bounds the look-ahead with it"""
    return max(p.try_max_nocarrier, p.try_max_carrier) - 1 + p.frame_nsamples




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
    if FAMILIES[fam]["src"] == "s16":
        streams = [pcm(x) for x in streams]
    r = call(eng, fam, streams, lens, bands=bands, max_frames=max_frames, states=states, auto_states=auto_states,
             rec_band=True)
    extra = None
    if r.auto is not None:
        extra = (r.auto.cpu().numpy().tobytes(), [r.rec_band[s, :int(r.st["nframes"][s])].tobytes()
                                                  for s in range(len(streams))])
    return Run(r.recs, r.st, extra, r.k), r.states, r.auto


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
FAM_KEYS = SHAPE_FAMILIES
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
    eng = new_engine(monkeypatch, fam, c[0])
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
        e1 = new_engine(monkeypatch, fam, c[0], env, pin)
        got, _, _ = run(e1, fam, c)
        assert shape(got.k) == shape(k0) and got.k["threads"] == 128, got.k["text"]
        got.same_as(base, (fam, which, "4 warps"))
        report(fam, got.k, got.nrecs())
        k0 = got.k
    r_full = ring_for_full_lookahead(k0, p)
    rings = [k0["ring"] + 128, k0["ring"] + 256, r_full, deepest_ring(k0, 4 * r_full)]
    assert rings[-1] >= r_full + 128, (fam, which, rings, k0["text"])
    for ring in rings:
        e2 = new_engine(monkeypatch, fam, c[0], env, dict(pin, ring_floats=ring))
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
    eng = new_engine(monkeypatch, fam, c[0])
    one, _, _ = run(eng, fam, c)
    k0 = one.k
    p = eng.params
    env = {"FSK_B200_SPLIT": str(k0["L"])}
    pin = dict(lanes_per_stream=k0["G"], warps_per_block=min(4, k0["threads"] // 32))
    engines = [eng, new_engine(monkeypatch, fam, c[0], env, dict(pin, ring_floats=ring_for_full_lookahead(k0, p)))]
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
        states = state_rows(st)
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
    screened oracle (as rxfam.compare_rx does), not to the default run."""
    fam = "per-candidate" if env is PER_CAND else "shared-segment"
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c[0])
    base, _, _ = run(eng, fam, c)
    e2 = new_engine(monkeypatch, fam, c[0], tune=dict(ring_floats=base.k["ring"] + 2048))
    got, _, _ = run(e2, fam, c)
    k = got.k
    assert k["ring"] == base.k["ring"] + 2048 and k["mode"] == base.k["mode"], k["text"]
    assert k["G"] > base.k["G"], (base.k["text"], k["text"])
    make, streams, lens, _, m = c
    screened = [tie_screen.screen(m, x) for x in streams]
    compare_rx(screened, [np.frombuffer(r, mm.FRAME_DTYPE) for r in got.recs], got.st, k["text"])
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
    eng = new_engine(monkeypatch, fam, c[0])
    base, _, _ = run(eng, fam, c)
    k0 = base.k
    check_family(fam, k0)
    env = {"FSK_B200_SPLIT": str(k0["L"])}
    r_full = ring_for_full_lookahead(k0, eng.params)
    rows = [dict(warps_per_block=w) for w in (1, 2, 3, 4)] + [dict(warps_per_block=3, ring_floats=r_full)]
    smem = {}
    for tv in rows:
        e2 = new_engine(monkeypatch, fam, c[0], env, dict(tv, lanes_per_stream=k0["G"]))
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
    eng = new_engine(monkeypatch, fam, c[0], tune=dict(ring_floats=SMEM_MAX // 4 + 128))
    got, _, _ = run(eng, fam, c)
    k = got.k
    assert (k["mode"], k["G"], k["ring"], k["lookahead"]) == (1, 32, 0, 0), k["text"]
    assert "mode=1(generic)" in k["text"] and k["src"] == src, k["text"]
    make, streams, lens, _, m = c
    if src == "s16":
        streams = [pcm(x).astype(np.float32) / np.float32(32768.0) for x in streams]
    screened = [tie_screen.screen(m, x) for x in streams]
    compare_rx(screened, [np.frombuffer(r, mm.FRAME_DTYPE) for r in got.recs],
                 got.st, k["text"])


@pytest.mark.gpu
def test_a_ring_that_leaves_no_room_for_the_sliding_table_drops_slide(monkeypatch):
    """The sliding fine search stages an extended tone table; a ring that fits the block only without it
    launches without `slide`, and that run equals an FSK_B200_NO_SLIDE=1 run bit for bit (sliding rounds
    differently, DESIGN.md 3, so the sliding run is not the reference)."""
    c = case("per-candidate", ("1200", 48000))
    pin = dict(lanes_per_stream=32, warps_per_block=1)
    slide = new_engine(monkeypatch, "per-candidate", c[0], tune=pin)
    a, _, _ = run(slide, "per-candidate", c)
    flat = new_engine(monkeypatch, "per-candidate-noslide", c[0], tune=pin)
    b, _, _ = run(flat, "per-candidate-noslide", c)
    assert a.k["src"] == "f32,slide" and b.k["src"] == "f32", (a.k["text"], b.k["text"])
    extra = a.k["smem"] - b.k["smem"]
    step = per_ring_float(b.k) * 128
    assert extra > step, (extra, step)
    # the first ring whose block fits without the extension but not with it
    blocks = (SMEM_MAX - extra - b.k["smem"]) // step + 1
    ring = b.k["ring"] + 128 * blocks
    assert b.k["smem"] + step * blocks <= SMEM_MAX < b.k["smem"] + step * blocks + extra
    e1 = new_engine(monkeypatch, "per-candidate", c[0], tune=dict(pin, ring_floats=ring))
    got, _, _ = run(e1, "per-candidate", c)
    e2 = new_engine(monkeypatch, "per-candidate-noslide", c[0], tune=dict(pin, ring_floats=ring))
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
    t = torch()
    n = max(max(r[0].size for r in rows), max(r[1] or 0 for r in rows))
    stride = (n + 7) & ~7
    buf = np.zeros((len(rows), stride), np.float32)
    lens = np.zeros(len(rows), np.int32)
    st = np.zeros(len(rows), mm.STATE_DTYPE)
    for i, (x, ln, s0, _) in enumerate(rows):
        buf[i, :x.size] = x
        lens[i] = stride if ln is None else ln
        st[i] = s0
    frames = t.full((len(rows), max_frames, 5), 0x5A5A5A5A, dtype=t.int32).to(dev())
    bands = [r[3] for r in rows] if FAMILIES[fam]["call"] == "tones" else None
    r = call(eng, fam, upload(buf), lens, n=stride, bands=bands, states=st, max_frames=max_frames, frames=frames)
    raw = r.fr.view(np.int32).reshape(len(rows), -1)
    return [(r.recs[i], r.st[i].tobytes(), bool((raw[i] == 0x5A5A5A5A).all())) for i in range(len(rows))], r.k


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
    eng = new_engine(monkeypatch, fam, make, tune=dict(lanes_per_stream=G) if G else None)
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
    eng = new_engine(monkeypatch, fam, c[0])
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
