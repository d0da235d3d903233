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
import numpy as np
import pytest

import minimodem_b200 as mm
import orc
import rxfam
import tie_screen
from gpudev import pcm
from rxcases import drops, live_text, one_pass_text, session_case
from rxfam import PRESETS, compare_rx

# the families of test_gpu_launch_shapes but its auto call, the generic kernel (a ring too large for any
# fast shape) and tone-pair channels, k = 2
FAMILIES = {f: rxfam.FAMILIES[f] for f in rxfam.SHAPE_FAMILIES if rxfam.FAMILIES[f]["call"] != "auto"}
FAMILIES["generic"], FAMILIES["generic-s16"] = rxfam.FAMILIES["generic"], rxfam.FAMILIES["generic-s16"]
FAMILIES["channels"] = dict(rxfam.FAMILIES["channels-2"], call="channels")
NOT_LAUNCHED = {k: v for k, v in rxfam.NOT_LAUNCHED.items() if k[0] in FAMILIES}
NOT_LAUNCHED[("channels", "same")] = "as the tone call"
ROWS = [(fam, w) for fam in FAMILIES for w in PRESETS + (["random"] if "cls" in FAMILIES[fam] else [])
        if (fam, w[0]) not in NOT_LAUNCHED]


def _rid(r):
    return "%s-%s" % (r[0], r[1] if isinstance(r[1], str) else "%s@%d" % r[1])


def case(fam, which):
    return session_case(FAMILIES[fam], which)


def registry_name(fam):
    """this file's family name in rxfam.FAMILIES"""
    return "channels-2" if fam == "channels" else fam


def skip_tma(fam):
    rxfam.skip_tma(registry_name(fam))


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
        for which in PRESETS:
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
    return rxfam.new_engine(monkeypatch, registry_name(fam), c.make, tune=FAMILIES[fam].get("tune"))


def run(eng, fam, c, max_frames=None, states=None):
    """records per channel (bytes), the states, the launch"""
    rows_ = [pcm(x) for x in c.rows] if FAMILIES[fam]["src"] == "s16" else c.rows
    r = rxfam.call(eng, registry_name(fam), rows_, c.lens, bands=c.bands or None, max_frames=max_frames,
                   states=states)
    rxfam.check_family(registry_name(fam), r.k)
    text = r.k["text"][:len(r.k["text"]) - len(" channels=%d" % c.k)] if c.k > 1 else r.k["text"]
    return r.recs, r.st, text


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
    compare_rx(c.screened, [np.frombuffer(r, mm.FRAME_DTYPE) for r in recs], st, what)
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
        states = st
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
    fam = {"plain": "per-candidate", "tones": "tones", "channels": "channels", "pcm16": "per-candidate-s16"}[form]
    c = case(fam, ("1200", 48000))
    rows_ = [pcm(x) for x in c.rows] if form == "pcm16" else c.rows
    pairs = c.hz if c.hz else None
    cuts = [(c.row_of[j], (a + b) // 2) for j, ns in enumerate(c.noise) for a, b in ns]
    for j, x in enumerate(c.rows):             # and inside the silent gaps
        quiet = np.flatnonzero(np.abs(x) < 0.02)
        if quiet.size:
            cuts.append((j, int(quiet[quiet.size // 2])))
    whole = one_pass_text(c.mode, c.rate, rows_, pairs, c.k, False)
    assert sum(len(w) for w in whole) >= 3 * len(rows_), whole
    got = live_text(c.mode, c.rate, rows_, pairs, c.k, False, 1501, 7, cuts, pcm16=form == "pcm16")
    assert got == whole, (form, [(a, b) for a, b in zip(got, whole) if a != b][:2])


def test_carrier_sessions_on_the_emulated_kernels():
    """The `gpu` tests above on the host SIMT emulation of the kernels, copies landing late."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 3000, module="test_gpu_carrier_sessions.py")
    assert " passed" in tail and "failed" not in tail
