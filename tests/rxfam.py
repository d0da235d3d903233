"""The rx launch families the `gpu` test files share, how a test asks for one and checks that it ran, and
the comparison of device records with the oracle's.

A family is a call (rx_batch, rx_batch_tones or rx_batch_auto), a sample type, the environment knobs that
select the kernel (read when the engine is created) and the kernel it must launch: (last_kernel name, mode,
fill).  `cls` / `n`: the random framing of rxcases.framing that the family also runs."""
import re

import numpy as np
import pytest

import autoorc
import golden_util as gu
import gpudev
import minimodem_b200 as mm
from gpudev import emulated

SMEM_MAX = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (and of the emulation)
KNOBS = ("FSK_B200_LANES", "FSK_B200_SPLIT", "FSK_B200_MULTI", "FSK_B200_PREFIX", "FSK_B200_PFX_FILL",
         "FSK_B200_RING", "FSK_B200_WPB", "FSK_B200_NO_SLIDE")
PER_CAND = {"FSK_B200_MULTI": "0", "FSK_B200_PREFIX": "0"}
SHARED = {"FSK_B200_MULTI": "2", "FSK_B200_PREFIX": "0"}

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
# the launch shapes' families; then tone-pair channels, k per row, and the generic kernel (a ring too large for
# any fast shape)
SHAPE_FAMILIES = list(FAMILIES)
for _k in (2, 3):
    FAMILIES["channels-%d" % _k] = dict(call="tones", src="f32", env={}, kern=("k_rx_tones", 0, 0), k=_k)
for _src in ("f32", "s16"):
    FAMILIES["generic" + ("-s16" if _src == "s16" else "")] = dict(
        call="rx", src=_src, env=PER_CAND, kern=("k_rx", 1, 0), cls="long", n=11,
        tune=dict(ring_floats=SMEM_MAX // 4 + 128))

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


def parse_launch(s):
    """a last_kernel() string as a dict; `k`: the channels per row of its ` channels=k` suffix (1 without)"""
    k = 1
    m = re.search(r" channels=(\d+)$", s)
    if m:
        k = int(m.group(1))
    m = LK.match(s[:len(s) - len(m.group(0))] if k > 1 else s)
    assert m, s
    d = dict(zip(("name", "G", "W", "L", "mode", "fill", "src", "threads", "ring", "smem", "blocks", "lookahead"),
                 m.groups()))
    for f in d:
        if f not in ("name", "src"):
            d[f] = int(d[f])
    d["k"] = k
    d["text"] = s
    return d


def launch(eng, k=1):
    """eng.last_kernel() as a dict; it must carry k channels per row (no ` channels=` suffix for k = 1)"""
    d = parse_launch(eng.last_kernel())
    assert d["k"] == k, (k, d["text"])
    return d


def check_family(fam, k):
    """the launch `k` is the kernel family `fam` asks for"""
    f = FAMILIES[fam]
    name, mode, fill = f["kern"]
    assert (k["name"], k["mode"], k["fill"]) == (name, mode, fill), (fam, k["text"])
    assert k["src"].split(",")[0] == f["src"], (fam, k["text"])
    assert k["k"] == f.get("k", 1), (fam, k["text"])
    if fam == "per-candidate":
        assert k["src"] == "f32,slide", k["text"]
    if fam == "per-candidate-noslide":
        assert k["src"] == "f32", k["text"]
    if mode == 1:
        assert "mode=1(generic)" in k["text"], k["text"]


def check_launch(eng, fam):
    """eng's last launch is the kernel family `fam` asks for"""
    check_family(fam, launch(eng, FAMILIES[fam].get("k", 1)))


def set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)            # read when the engine is created


def new_engine(monkeypatch, fam, make, extra_env=None, tune=None):
    """the engine `make()` builds under the family's environment (and `extra_env`), with the auto call's default
    threshold and `tune` applied"""
    f = FAMILIES[fam]
    set_env(monkeypatch, dict(f["env"], **(extra_env or {})))
    eng = make()
    if f["call"] == "auto":
        eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    if tune:
        eng.tune(**tune)
    return eng


class Call:
    """one rx call's outputs: `fr` and `st` (numpy frames and a copy of the states), `recs` (each channel's
    records as bytes), `states` / `auto` (the device states and auto states), `rec_band` (numpy, when asked
    for) and `k` (the parsed launch)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def call(eng, fam, rows, lens=None, n=None, bands=None, states=None, auto_states=None, max_frames=None,
         frames=None, rec_band=False, k=None):
    """One rx call of family `fam`: rx_batch, rx_batch_tones (k channels per row) or rx_batch_auto.  `rows`:
    host streams, copied into rows of a multiple of 8 samples in their own dtype (n: the longest, unless
    given), or a device tensor (n given).  `lens`, `bands` (per channel, [mark, space]) and `states` (numpy
    state records) are uploaded when they are host arrays.  `k`: channels per row of a tone call, if not the
    family's own."""
    f = FAMILIES[fam]
    k = f.get("k", 1) if k is None else k
    if isinstance(rows, (list, tuple)):
        buf, n0 = gpudev.rows(rows, rows[0].dtype, 8)
        x, n = gpudev.upload(buf), n0 if n is None else n
    else:
        x = rows
    if isinstance(lens, (list, tuple, np.ndarray)):
        lens = gpudev.upload(np.asarray(lens, np.int32))
    if isinstance(bands, (list, tuple, np.ndarray)):
        bands = gpudev.bands_tensor(bands)
    if isinstance(states, np.ndarray):
        states = gpudev.state_rows(states)
    kw = dict(nsamples=n, nsamples_each=lens, max_frames=max_frames, frames=frames, states=states)
    ast = rb = None
    if f["call"] == "rx":
        fr, st = eng.rx_batch(x, **kw)
    elif f["call"] == "tones":
        fr, st = eng.rx_batch_tones(x, bands, channels_per_row=k, **kw)
    elif rec_band:
        fr, st, ast, rb = eng.rx_batch_auto(x, auto_states=auto_states, rec_band=True, **kw)
    else:
        fr, st, ast = eng.rx_batch_auto(x, auto_states=auto_states, **kw)
    gpudev.sync()
    recs, sn = gpudev.records(fr, st)
    return Call(fr=mm.frames_to_numpy(fr), st=sn.copy(), recs=recs, states=st, auto=ast,
                rec_band=None if rb is None else rb.cpu().numpy(), k=launch(eng, k))


def skip_tma(fam):
    if emulated() and FAMILIES[fam]["kern"][2] == 1:
        pytest.skip("the host emulation does not model cp.async.bulk / mbarrier")


# ---------------------------------------------------------------------------------------------------
# device records against the oracle's
# ---------------------------------------------------------------------------------------------------
def as_oracle_frames(recs):
    out = []
    for r in recs:
        fs = int(r["frame_start"])
        if fs == mm.FRAME_REPORT:
            continue
        bits = int(r["bits_lo"]) | (int(r["bits_hi"]) << 32)
        out.append((bits, np.float32(r["confidence"]), np.float32(r["amplitude"]), fs & 0x7FFFFFFF,
                    1 if fs & mm.FRAME_ACQUIRED else 0, 0))
    return out


def reports_of(recs, st_row):
    """Carrier-session statistics exactly as the device accumulated them: the REPORT
    records (carrier drops, src/minimodem.c:1298-1307) plus the session still open at
    the end of the stream (:1469-1474), which lives in the stream state."""
    reps, count, nfr = [], 0, 0
    for r in recs:
        fs = int(r["frame_start"])
        if fs == mm.FRAME_REPORT:
            reps.append((count, int(r["bits_lo"]) | (int(r["bits_hi"]) << 32), np.float32(r["confidence"]),
                         np.float32(r["amplitude"]), nfr))
            count = 0
        else:
            count = 1 if fs & mm.FRAME_ACQUIRED else count + 1
            nfr += 1
    if st_row["carrier"]:
        assert int(st_row["nframes_decoded"]) == count
        reps.append((count, int(st_row["carrier_nsamples"]), np.float32(st_row["confidence_total"]),
                     np.float32(st_row["amplitude_total"]), nfr))
    return reps


def compare_reports(got, want, what=""):
    assert len(got) == len(want), (what, got, want)
    for a, b in zip(got, want):
        assert a[0] == b[0] and a[1] == b[1] and a[4] == b[4], (what, a, b)
        assert gu.close(a[2], b[2], cond=gu.CONF_COND) and gu.close(a[3], b[3]), (what, a, b)


def compare_frames(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (a, b) in enumerate(zip(got, want)):
        assert a[0] == b[0], (what, i, hex(a[0]), hex(b[0]))
        assert a[3] == b[3] and a[4] == b[4], (what, i, a, b)
        assert gu.close(a[1], b[1], cond=gu.CONF_COND), (what, i, a[1], b[1])
        assert gu.close(a[2], b[2]), (what, i, a[2], b[2])


def compare_rx(screened, recs, st, what):
    """every stream done; robust streams (tests/tie_screen.py) give the oracle's records and session reports,
    screened-out ones its frame count within one"""
    assert (st["done"] == 1).all(), what
    for s, (want, robust) in enumerate(screened):
        got = as_oracle_frames(recs[s])
        if robust:
            compare_frames(got, want["frames"], "%s stream %d" % (what, s))
            compare_reports(reports_of(recs[s], st[s]), want["reports"], "%s stream %d" % (what, s))
        else:
            assert abs(len(got) - len(want["frames"])) <= 1, (what, s, len(got), len(want["frames"]))


def check_against_oracle(screened, fr, st, what):
    """as compare_rx on the records of fr / st, and at least half the streams robust"""
    nok = 0
    for s, (w, robust) in enumerate(screened):
        recs = fr[s, :int(st["nframes"][s])]
        got = as_oracle_frames(recs)
        if not robust:
            assert abs(len(got) - len(w["frames"])) <= 1, (what, s, len(got), len(w["frames"]))
            continue
        nok += 1
        compare_frames(got, w["frames"], "%s stream %d" % (what, s))
        compare_reports(reports_of(recs, st[s]), w["reports"], "%s stream %d" % (what, s))
    assert 2 * nok >= len(screened), (what, "screened out", len(screened) - nok)
