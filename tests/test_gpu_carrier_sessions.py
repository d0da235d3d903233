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

The auto call (--auto-carrier) runs every AUTO_COMBOS preset, float and int16 rows, and --inverted once.
Its loop also scans for the carrier: every burst is on its own random pair of the band grid, a burst on
one pair follows another directly (a retune), a burst's space band falls outside the grid (the scan rejects
it), and every strike past the 20th -- in noise too, without a carrier -- rescans.  Its boundary streams
straddle the drop twice, the second burst on the first one's pair and on another.  Its streams are held to
the screened FLAT auto oracle (tests/autoorc.py), bands included, and its scan events come from the
oracle's scan log.

Robust streams (tests/tie_screen.py, whose replay of the loop's bookkeeping adds margins for the squelch,
the refine trigger and refine-keep, and decides each comparison inside its margin the other way once) must give the oracle's records and session reports; the others only
the frame count within one.  Resumed at every record (max_frames = 1) and fed to LiveReceiver in random
chunks, every family must give its own one-pass result.

The CPU test runs this file's `gpu` tests on the host SIMT emulation of the kernels (tests/emu); the TMA
bulk fill is not modelled there and its rows skip."""
import numpy as np
import pytest

import autoorc
import minimodem_b200 as mm
import orc
import rxfam
import tie_screen
from gpudev import pcm
from rxcases import COVER, auto_drop_in_gap, drops, live_records, live_text, one_pass_text, session_case
from rxfam import PRESETS, compare_frames, compare_reports, compare_rx, reports_of

# the families of test_gpu_launch_shapes, the generic kernel (a ring too large for any fast shape), tone-pair
# channels, k = 2, and the auto call under --inverted
FAMILIES = {f: rxfam.FAMILIES[f] for f in rxfam.SHAPE_FAMILIES}
FAMILIES["generic"], FAMILIES["generic-s16"] = rxfam.FAMILIES["generic"], rxfam.FAMILIES["generic-s16"]
FAMILIES["channels"] = dict(rxfam.FAMILIES["channels-2"], call="channels")
FAMILIES["auto-inverted"] = dict(rxfam.FAMILIES["auto"], inverted=True)
NOT_LAUNCHED = {k: v for k, v in rxfam.NOT_LAUNCHED.items() if k[0] in FAMILIES}
NOT_LAUNCHED[("channels", "same")] = "as the tone call"
# the auto call runs every preset of the AUTO_COMBOS cover table (one per kernel instance), --inverted at 1200
AUTO_PRESETS = sorted(set(COVER.values()))
ROWS = [(fam, w) for fam in FAMILIES if FAMILIES[fam]["call"] != "auto"
        for w in PRESETS + (["random"] if "cls" in FAMILIES[fam] else []) if (fam, w[0]) not in NOT_LAUNCHED]
ROWS += [(fam, w) for fam in ("auto", "auto-s16") for w in AUTO_PRESETS] + [("auto-inverted", ("1200", 48000))]


def _rid(r):
    return "%s-%s" % (r[0], r[1] if isinstance(r[1], str) else "%s@%d" % r[1])


def case(fam, which):
    return session_case(FAMILIES[fam], which)


def registry_name(fam):
    """this file's family name in rxfam.FAMILIES"""
    return {"channels": "channels-2", "auto-inverted": "auto"}.get(fam, fam)


def skip_tma(fam):
    rxfam.skip_tma(registry_name(fam))


# ---------------------------------------------------------------------------------------------------
# CPU: the loop events every case reaches
# ---------------------------------------------------------------------------------------------------
EVENTS = ("acquire", "refine-in-session", "strike-threshold", "strike-squelch", "drop", "held-15-strikes",
          "acquire-in-noise", "open-at-end", "ends-mid-count")
# the auto call's scan events, from the auto oracle's scan log
SCAN_EVENTS = ("scan-none", "accept-after-window-0", "accept-in-noise", "reject-space", "rescan-after-drop-elsewhere",
               "rescan-on-strike-without-carrier", "retune", "scan-at-end")
# the events a preset's case cannot reach, with the reason
_SHORT_NOISE = "the auto call's noise segments are at most 60 bit periods (rxcases.session_stream): no search in them passes the threshold"
NOT_REACHED = {
    ("auto", "300@48000", "acquire-in-noise"): _SHORT_NOISE,
    ("auto", "uic-train@8000", "acquire-in-noise"): _SHORT_NOISE + " (a UIC frame is 47 bits and starts with a sync byte)",
    ("auto", "uic-ground@48000", "acquire-in-noise"): _SHORT_NOISE + " (a UIC frame is 47 bits and starts with a sync byte)",
    ("auto", "uic-ground@48000", "scan-none"): "one scan covers half the ring, 50 bit periods at 48 kHz, so a gap of at most 60 "
                                          "after the 21 strikes always reaches the next burst",
    ("auto", "uic-ground@48000", "scan-at-end"): "a 47-bit frame: the loop stops with less than a frame left before the last drop "
                                            "rescans",
    ("auto", "rtty@48000", "held-15-strikes"): "no stream holds a carrier across 15 strikes (the 8 kHz case does)",
}


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


def auto_events_of(m, x, noise, inverted):
    """the loop events of the auto oracle's run on x: the nine above from tie_screen.replay over its search
    calls, the scan events from its scan log"""
    r = autoorc.rx_run(m, x, inverted=inverted, scans=True)
    ev = []
    frames, reports, _ = tie_screen.replay(m, autoorc.calls(m, x, inverted), events=ev)
    assert [f[:5] for f in r["frames"]] == frames and r["reports"] == reports
    kinds = {kind for kind, _ in ev}
    inside = lambda at: any(a <= at < b for a, b in noise)
    if any(f[4] and inside(f[5] + f[3]) for f in r["frames"]):
        kinds.add("acquire-in-noise")
    d = m.derived()
    window = int(min(float(d.nsamples_per_bit), orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width).p.fftsize))
    for e in r["scans"]:
        ok = e["outcome"] == "accepted"
        dropped = r["report_band"][e["nreports"] - 1] if e["nreports"] else None
        kinds.add({"none": "scan-none", "rejected": "reject-space"}.get(e["outcome"], "accepted"))
        if ok and e["window"] > 0:
            kinds.add("accept-after-window-0")
        if ok and inside(e["pos"] + e["window"] * window):
            kinds.add("accept-in-noise")
        if ok and dropped is not None and e["band"] != dropped:
            kinds.add("rescan-after-drop-elsewhere")
            nf = e["nframes"]
            if e["cause"] == "after-drop" and e["window"] == 0 and nf < len(frames) and r["frame_band"][nf] == e["band"]:
                kinds.add("retune")
        if e["cause"] == "after-strike":
            kinds.add("rescan-on-strike-without-carrier")
    last = r["scans"][-1] if r["scans"] else None
    if last and last["outcome"] == "none" and last["nframes"] == len(frames):
        kinds.add("scan-at-end")         # the loop runs out of samples while it scans
    return kinds


def test_every_case_reaches_every_loop_event():
    """From the oracle's call list: every preset's case (plain, tone, channel and auto calls) reaches every loop
    event, but those NOT_REACHED names; the boundary streams straddle the 21-strike drop.  The auto call's
    cases also reach every scan event, from the auto oracle's scan log."""
    seen = {}
    rows = [(fam, w) for fam in ("per-candidate", "tones", "channels") for w in PRESETS]
    rows += [("auto", w) for w in AUTO_PRESETS] + [("auto-inverted", ("1200", 48000))]
    for fam, which in rows:
        if (fam, which[0]) in NOT_LAUNCHED:
            continue
        c = case(fam, which)
        auto = FAMILIES[fam]["call"] == "auto"
        events = EVENTS + (SCAN_EVENTS if auto else ())
        got = set()
        for j, (want, _) in enumerate(c.screened):
            if auto:
                got |= auto_events_of(c.modes[j], c.rows[c.row_of[j]], c.noise[j], c.inverted)
            else:
                got |= events_of(c.modes[j], c.rows[c.row_of[j]], c.noise[j])
        for j, ndrop in c.boundary:
            x = c.rows[c.row_of[j]]
            if auto:                    # the drop before the second burst, or none before it
                assert auto_drop_in_gap(c.modes[j], x, c.gap_end[j], c.inverted) == bool(ndrop), (fam, which, j)
            else:
                assert min(drops(c.modes[j], x), 1) == ndrop, (fam, which, j)
        call = "auto" if auto else FAMILIES[fam]["call"]
        preset = "%s@%d%s" % (which + ("-inverted" if c.inverted else "",)) if auto else which[0]
        seen[(call, preset)] = got
        missing = [e for e in events if e not in got and (call, preset, e) not in NOT_REACHED]
        print("%s %s: %s" % (fam, which[0], " ".join(e for e in events if e in got)))
        assert not missing, (fam, which, missing)
    for (call, preset, e), why in NOT_REACHED.items():
        assert e not in seen.get((call, preset), set()), (call, preset, e, "reached after all", why)


# ---------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------
def new_engine(monkeypatch, fam, c):
    eng = rxfam.new_engine(monkeypatch, registry_name(fam), c.make, tune=FAMILIES[fam].get("tune"))
    if FAMILIES[fam].get("inverted"):
        eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD, inverted=True)
    return eng


def run(eng, fam, c, max_frames=None, states=None, auto_states=None):
    """records per channel (bytes), the states, the launch; for the auto call also the record bands and the
    auto states"""
    rows_ = [pcm(x) for x in c.rows] if FAMILIES[fam]["src"] == "s16" else c.rows
    auto = FAMILIES[fam]["call"] == "auto"
    r = rxfam.call(eng, registry_name(fam), rows_, c.lens, bands=c.bands or None, max_frames=max_frames,
                   states=states, auto_states=auto_states, rec_band=auto)
    rxfam.check_family(registry_name(fam), r.k)
    text = r.k["text"][:len(r.k["text"]) - len(" channels=%d" % c.k)] if c.k > 1 else r.k["text"]
    if auto:
        return r.recs, r.st, text, r.rec_band, r.auto
    return r.recs, r.st, text


def compare_auto(screened, recs, st, rec_band, what):
    """every stream done; robust streams give the auto oracle's records, session reports and bands: the band
    of every frame record and of every report record"""
    assert (st["done"] == 1).all(), what
    for s, (want, robust) in enumerate(screened):
        if not robust:
            continue
        r = np.frombuffer(recs[s], mm.FRAME_DTYPE)
        compare_frames(rxfam.as_oracle_frames(r), want["frames"], "%s stream %d" % (what, s))
        compare_reports(reports_of(r, st[s]), want["reports"], "%s stream %d" % (what, s))
        rep = r["frame_start"] == mm.FRAME_REPORT
        b = rec_band[s, :len(r)]
        assert [int(v) for v in b[~rep]] == want["frame_band"], (what, s)
        assert [int(v) for v in b[rep]] == want["report_band"][:int(rep.sum())], (what, s)


SCREEN_COUNT = {}


@pytest.mark.gpu
@pytest.mark.parametrize("fam,which", ROWS, ids=[_rid(r) for r in ROWS])
def test_carrier_sessions_against_the_screened_oracle(fam, which, monkeypatch):
    """Robust channels give the oracle's records and session reports (and the auto call its bands),
    screened-out ones its frame count within one (the auto call: nothing, a scan near-tie can move a whole
    session)."""
    skip_tma(fam)
    c = case(fam, which)
    eng = new_engine(monkeypatch, fam, c)
    out = run(eng, fam, c)
    recs, st, text = out[:3]
    what = "%s %s %s" % (fam, which, text)
    if FAMILIES[fam]["call"] == "auto":
        compare_auto(c.screened, recs, st, out[3], what)
    else:
        compare_rx(c.screened, [np.frombuffer(r, mm.FRAME_DTYPE) for r in recs], st, what)
    bad = sum(1 for _, r in c.screened if not r)
    cnt = SCREEN_COUNT.setdefault(registry_name(fam), [0, 0])     # --inverted counts with the auto call
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
    byte for byte and the final states equal its states but nframes (the auto call: carrying the auto
    states, also the record bands and the final auto states)."""
    skip_tma(fam)
    c = case(fam, which)
    auto = FAMILIES[fam]["call"] == "auto"
    eng = new_engine(monkeypatch, fam, c)
    out1 = run(eng, fam, c)
    one, st1 = out1[:2]
    joined = [b""] * len(one)
    jband = [[] for _ in one]
    states = ast = None
    for i in range(100000):
        out = run(eng, fam, c, max_frames=1, states=states, auto_states=ast)
        got, st = out[:2]
        assert (st["nframes"] <= 1).all()
        for s in range(len(joined)):
            joined[s] += got[s]
            if auto:
                jband[s] += [int(v) for v in out[3][s, :int(st["nframes"][s])]]
        if auto:
            ast = out[4]
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
    if auto:
        assert jband == [[int(v) for v in out1[3][s, :int(st1["nframes"][s])]] for s in range(len(one))], fam
        assert ast.cpu().numpy().tobytes() == out1[4].cpu().numpy().tobytes(), fam
    print("%s: %d calls, %d records (%d session reports) equal to one pass" % (
        fam, i + 1, int(st1["nframes"].sum()), nrep))


def live_cuts(c, fam):
    """(row, sample) cuts inside every noise segment and a silent gap of every row, and for the auto call right
    after every carrier drop (where the rescan starts)"""
    cuts = [(c.row_of[j], (a + b) // 2) for j, ns in enumerate(c.noise) for a, b in ns]
    for j, x in enumerate(c.rows):             # and inside the silent gaps
        quiet = np.flatnonzero(np.abs(x) < 0.02)
        if quiet.size:
            cuts.append((j, int(quiet[quiet.size // 2])))
    if FAMILIES[fam]["call"] == "auto":
        for j, x in enumerate(c.rows):
            r = autoorc.rx_run(c.modes[j], x, inverted=c.inverted, scans=True)
            cuts += [(j, int(e["pos"])) for e in r["scans"] if e["cause"] == "after-drop"]
    return cuts


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "tones", "channels", "pcm16", "auto", "auto-pcm16"])
def test_live_receiver_on_carrier_sessions(form):
    """LiveReceiver fed the session streams in random chunks, with a cut inside every silent gap and
    noise segment while the strikes are counting (and, with auto-carrier, right after every drop): the text
    of one rx pass over the same rows."""
    fam = {"plain": "per-candidate", "tones": "tones", "channels": "channels", "pcm16": "per-candidate-s16",
           "auto": "auto", "auto-pcm16": "auto-s16"}[form]
    c = case(fam, ("1200", 48000))
    pcm16 = form.endswith("pcm16")
    auto = form.startswith("auto")
    rows_ = [pcm(x) for x in c.rows] if pcm16 else c.rows
    pairs = c.hz if c.hz else None
    cuts = live_cuts(c, fam)
    whole = one_pass_text(c.mode, c.rate, rows_, pairs, c.k, auto)
    assert sum(len(w) for w in whole) >= 3 * len(rows_), whole
    got = live_text(c.mode, c.rate, rows_, pairs, c.k, auto, 1501, 7, cuts, pcm16=pcm16)
    assert got == whole, (form, [(a, b) for a, b in zip(got, whole) if a != b][:2])


@pytest.mark.gpu
@pytest.mark.parametrize("fam", ["auto", "auto-s16"])
def test_live_auto_records_on_carrier_sessions(fam, monkeypatch):
    """The live-stream recipe with auto-carrier (rxcases.live_records) on the session streams, cut inside
    the gaps, inside the noise segments and right after every drop: the records and bands of one pass."""
    c = case(fam, ("1200", 48000))
    eng = new_engine(monkeypatch, fam, c)
    recs, st, _, rec_band, _ = run(eng, fam, c)
    size = mm.FRAME_DTYPE.itemsize
    whole = [[(r[i * size:(i + 1) * size], int(rec_band[s, i])) for i in range(len(r) // size)]
             for s, r in enumerate(recs)]
    rows_ = [pcm(x) for x in c.rows] if FAMILIES[fam]["src"] == "s16" else c.rows
    cuts = sorted({p for _, p in live_cuts(c, fam)})
    got = live_records(eng, rows_, 1501, cuts)
    assert got == whole, fam
    print("%s: %d records over %d cuts" % (fam, sum(len(w) for w in whole), len(cuts)))


def test_carrier_sessions_on_the_emulated_kernels():
    """The `gpu` tests above on the host SIMT emulation of the kernels, copies landing late."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 3000, module="test_gpu_carrier_sessions.py")
    assert " passed" in tail and "failed" not in tail
