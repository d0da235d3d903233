"""TEST INFRASTRUCTURE for --auto-carrier: ctypes bindings of oracle/auto_oracle.c (the reference's rx
loop with the carrier scan, in LITERAL and FLAT mode, and its optional scan log) and helpers that format its
records the way the reference CLI prints them, and the near-tie screen of tests/tie_screen.py for it (the
perturbed searches, the scan margin, and the replay of the loop's bookkeeping with its flipped re-runs).
The library is compiled on first use into a temporary directory, so the tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import orc
import tie_screen

DEFAULT_THRESHOLD = 0.001       # src/minimodem.c:659, -a
# a scan decision within this relative margin of a tie (two largest band magnitudes, or the largest and the
# threshold) can go either way between two correct DFTs; the device takes a float64 DFT's decision at 2e-6
# (tests/test_gpu_auto_carrier.py, test_band_decisions_match_a_float64_dft)
SCAN_TIE = 1e-5


class Scan(C.Structure):
    """orc_auto_scan of oracle/auto_oracle.c: one carrier scan"""
    _fields_ = [("pos", C.c_ulonglong), ("nvalid", C.c_ulonglong), ("window", C.c_int), ("band", C.c_int),
                ("outcome", C.c_int), ("cause", C.c_int), ("nframes", C.c_uint), ("nreports", C.c_uint)]


OUTCOMES = ("none", "accepted", "rejected")
CAUSES = ("start", "again", "after-drop", "after-strike")


class Bands(C.Structure):
    """orc_auto_bands of oracle/auto_oracle.c"""
    _fields_ = [("frame_band", C.POINTER(C.c_uint)), ("report_band", C.POINTER(C.c_uint)),
                ("cap_f", C.c_size_t), ("cap_r", C.c_size_t), ("min_margin", C.c_float)]


class ScanLog(C.Structure):
    """orc_auto_scan_log of oracle/auto_oracle.c"""
    _fields_ = [("scans", C.POINTER(Scan)), ("nscans", C.c_size_t), ("cap", C.c_size_t)]


SOURCES = [os.path.join(orc.ORACLE_DIR, f) for f in ("auto_oracle.c", "fsk_oracle.c", "fsk_oracle.h")]
_lib = None


def build():
    """Compile oracle/auto_oracle.c (gcc, as oracle/Makefile compiles the oracle) into a temporary
    directory, named after a hash of its sources."""
    h = hashlib.sha256()
    for f in SOURCES:
        with open(f, "rb") as fh:
            h.update(fh.read())
    out = os.path.join(tempfile.gettempdir(), "fsk_auto_oracle_%d_%s.so" % (os.getuid(), h.hexdigest()[:16]))
    if not os.path.exists(out):
        tmp = out + ".%d" % os.getpid()
        subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-Wno-unused-function", "-fPIC", "-ffp-contract=off",
                               "-shared", "-o", tmp, os.path.join(orc.ORACLE_DIR, "auto_oracle.c"), "-lm", "-lpthread"])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_rx_run_auto_log.argtypes = [C.POINTER(orc.OrcRxConfig), C.POINTER(C.c_float), C.c_size_t, C.c_int,
                                          C.c_float, C.c_int, C.c_int, C.c_void_p, C.POINTER(orc.OrcRxResult),
                                          C.POINTER(Bands), C.POINTER(ScanLog)]
        L.orc_rx_run_auto_log.restype = C.c_int
        L.orc_auto_scan_log_free.argtypes = [C.POINTER(ScanLog)]
        L.orc_rx_result_free.argtypes = [C.POINTER(orc.OrcRxResult)]
        L.orc_auto_bands_free.argtypes = [C.POINTER(Bands)]
        L.orc_auto_b_shift.argtypes = [C.c_float, C.c_int, C.c_int]
        L.orc_auto_b_shift.restype = C.c_int
        _lib = L
    return _lib


def b_shift(mode, inverted=False):
    return lib().orc_auto_b_shift(mode.band_width, mode.autodetect_shift, int(inverted))


def rx_run(mode, samples, literal=False, threshold=DEFAULT_THRESHOLD, inverted=False, find_frame=None, scans=False):
    """The rx loop with --auto-carrier.  `inverted` is the CLI's --inverted (it negates the band
    shift; the mode's own tones do not matter here).  Returns a dict like orc.rx_run's, plus
    "frame_band" and "report_band": the mark band of every frame and of every report, and
    "scan_margin": the smallest relative margin of a scan decision (see orc_auto_bands).
    find_frame: an orc.FIND_FRAME_FN-style Python search, called with ctx = the loop's orc_plan.
    scans: also return "scans", one dict per carrier scan (orc_auto_scan; outcome and cause by name)."""
    samples = np.ascontiguousarray(samples, np.float32)
    cfg = mode.rx_config()
    res, bands, log = orc.OrcRxResult(), Bands(), ScanLog()
    cb = orc.FIND_FRAME_FN(find_frame) if find_frame is not None else None
    rc = lib().orc_rx_run_auto_log(C.byref(cfg), orc.fptr(samples), samples.size, 0 if literal else 1,
                                   threshold, mode.autodetect_shift, int(inverted),
                                   C.cast(cb, C.c_void_p) if cb else None, C.byref(res), C.byref(bands),
                                   C.byref(log) if scans else None)
    if rc != 0:
        lib().orc_auto_scan_log_free(C.byref(log))
        raise ValueError("orc_rx_run_auto_log failed")
    out = {
        "frames": [(r.bits, orc.f32(r.confidence), orc.f32(r.amplitude), r.frame_start, r.acquired, r.pos)
                   for r in (res.frames[i] for i in range(res.nframes))],
        "reports": [(r.nframes_decoded, r.carrier_nsamples, orc.f32(r.confidence_total),
                     orc.f32(r.amplitude_total), r.after_frame)
                    for r in (res.reports[i] for i in range(res.nreports))],
        "frame_band": [bands.frame_band[i] for i in range(res.nframes)],
        "report_band": [bands.report_band[i] for i in range(res.nreports)],
        "scan_margin": float(bands.min_margin),
    }
    if scans:
        out["scans"] = [dict(pos=e.pos, nvalid=e.nvalid, window=e.window, band=e.band, outcome=OUTCOMES[e.outcome],
                             cause=CAUSES[e.cause], nframes=e.nframes, nreports=e.nreports)
                        for e in (log.scans[i] for i in range(log.nscans))]
        lib().orc_auto_scan_log_free(C.byref(log))
    lib().orc_rx_result_free(C.byref(res))
    lib().orc_auto_bands_free(C.byref(bands))
    return out


def carrier_line(mode, band):
    """The `### CARRIER` line of src/minimodem.c:1336-1347 for a session on mark band `band`."""
    hz = float(np.float32(np.float32(band) * mode.band_width))
    if mode.data_rate >= 100:
        return "### CARRIER %u @ %.1f Hz ###" % (int(np.float32(mode.data_rate + np.float32(0.5))), hz)
    return "### CARRIER %.2f @ %.1f Hz ###" % (float(mode.data_rate), hz)


def stat_lines(mode, res):
    """The CARRIER and NOCARRIER lines, in order, that the CLI prints to stderr for these records."""
    lines, ri = [], 0
    reps = res["reports"]
    for i, fr in enumerate(res["frames"]):
        while ri < len(reps) and reps[ri][4] <= i:
            lines.append(orc.report_line(mode, reps[ri]))
            ri += 1
        if fr[4]:
            lines.append(carrier_line(mode, res["frame_band"][i]))
    lines.extend(orc.report_line(mode, r) for r in reps[ri:])
    return lines


class AutoSearch(tie_screen.Search):
    """tie_screen's perturbed frame search on the tones the auto loop has at the moment of each call: the
    bands are read from the loop's orc_plan (ctx) and set on the screen's own plan."""

    def find_frame(self, ctx, *args):
        p = orc.OrcPlan.from_address(ctx)
        mine = self.plan.p
        if (mine.b_mark, mine.b_space) != (p.b_mark, p.b_space):
            orc.lib().orc_plan_free(C.byref(mine))      # the tone table follows the bands
            mine.b_mark, mine.b_space = p.b_mark, p.b_space
        return tie_screen.Search.find_frame(self, ctx, *args)


def record_key(res):
    return tie_screen.record_key(res) + [("band",) + tuple(res["frame_band"]),
                                         ("report",) + tuple(r[0] for r in res["reports"]) + tuple(res["report_band"])]


def calls(mode, x, inverted=False):
    """the auto oracle's search results, in order, as tie_screen.replay takes them"""
    s = AutoSearch(mode, 0.0, 0)
    rx_run(mode, x, inverted=inverted, find_frame=s.find_frame)
    return s.calls


def flipped(mode, x, tie, inverted=False):
    """tie_screen.flipped for the auto loop: its rx loop on x with one search result replaced (tie = (call
    index, "conf" or "ampl", value), as tie_screen.replay lists them), the search on the tones of the moment"""
    j, what, value = tie
    n = [0]

    def find_frame(ctx, samples, frame_nsamples, first, tmax, step, limit, expect, bits_out, ampl_out, start_out):
        c = orc.lib().orc_find_frame(C.cast(ctx, C.POINTER(orc.OrcPlan)), samples, frame_nsamples, first, tmax, step,
                                     limit, expect, bits_out, ampl_out, start_out)
        n[0] += 1
        if n[0] - 1 == j:
            if what == "conf":
                c = float(value)
            else:
                ampl_out[0] = float(value)
        return c
    return rx_run(mode, x, inverted=inverted, find_frame=find_frame)


def screen(mode, x, inverted=False, seeds=tie_screen.SEEDS):
    """(the FLAT auto oracle's result for x, robust?): robust when every scan decision keeps a relative
    margin of SCAN_TIE, tie_screen's perturbed searches (seeds runs) give the same records, bands and
    search margins, and every squelch, refine trigger or refine-keep inside tie_screen.replay's margins,
    decided the other way (flipped), gives them too."""
    want = rx_run(mode, x, inverted=inverted)
    if want["scan_margin"] < SCAN_TIE:
        return want, False
    key = record_key(want)
    for k in range(seeds):
        s = AutoSearch(mode, tie_screen.DELTA, 1 + k)
        res = rx_run(mode, x, inverted=inverted, find_frame=s.find_frame)
        if not s.margin_ok or record_key(res) != key:
            return want, False
    for tie in tie_screen.replay(mode, calls(mode, x, inverted), tie_screen.DELTA)[2]:
        if record_key(flipped(mode, x, tie, inverted)) != key:
            return want, False
    return want, True
