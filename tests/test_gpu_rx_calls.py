"""The ten batched rx entry points share one validation and launch path: one table over all of them.

- Refusals: a NULL engine, NULL or misaligned samples, a stride that does not fit the element size, NULL
  frames / states / auto states, max_frames 0, nsamples_all above the stride (no per-row lengths) or above
  2^32 - 4, 2^31 rows, and per kind: NULL tone_bands, 0 channels per row or more than 2^31 - 1 channels, an
  engine without auto-carrier.  Each returns -EINVAL, launches nothing and names the call's family first
  in fsk_b200_last_error().  Rows are never read: the refusals need no memory beyond a small buffer.
- nrows == 0 returns 0 before any other check, except the kind's own preconditions (auto-carrier set;
  an engine and tone_bands, channels_per_row != 0), which still return -EINVAL.
- One valid call per entry point launches and names its kernel family in last_kernel().

The CPU test runs the `gpu` tests of this file on the host SIMT emulation of the kernels (tests/emu)."""
import ctypes as C

import numpy as np
import pytest

import autoorc
import minimodem_b200 as mm
from gpudev import dev, sync, torch, upload

EINVAL = 22
STRIDE = 64
TOP = 1 << 32

# entry point -> (kind, bytes per sample, family named in its errors)
CALLS = {
    "rx_batch": ("fixed", 4, "rx_batch"),
    "rx_batch_s16": ("fixed", 2, "rx_batch_s16"),
    "rx_batch_auto": ("auto", 4, "rx_batch_auto"),
    "rx_batch_auto_s16": ("auto", 2, "rx_batch_auto"),
    "rx_batch_tones": ("tones", 4, "rx_batch_tones"),
    "rx_batch_tones_s16": ("tones", 2, "rx_batch_tones"),
    "rx_batch_channels": ("channels", 4, "rx_batch_tones"),
    "rx_batch_channels_s16": ("channels", 2, "rx_batch_tones"),
    "rx_batch_host": ("host", 4, "rx_batch_host"),
    "rx_batch_host_s16": ("host", 2, "rx_batch_host_s16"),
}
KERNEL = {"fixed": "k_rx<", "host": "k_rx<", "auto": "k_rx_auto<", "tones": "k_rx_tones<", "channels": "k_rx_tones<"}


# --------------------------------------------------------------------------
# CPU
# --------------------------------------------------------------------------
def test_rx_calls_on_the_emulated_kernels():
    """The `gpu` tests below on the host SIMT emulation of the kernels."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 900, module="test_gpu_rx_calls.py")
    assert " passed" in tail and "failed" not in tail


# --------------------------------------------------------------------------
# the table
# --------------------------------------------------------------------------
class Call:
    """One entry point with valid arguments for one row of STRIDE zeros (k = 2 channels for the channel
    calls); call(**overrides) replaces any of them."""

    def __init__(self, name):
        t = torch()
        self.name = name
        self.kind, self.elem, self.family = CALLS[name]
        self.host = self.kind == "host"
        self.k = 2 if self.kind == "channels" else 1
        self.eng = mm.RxEngine.for_mode("1200", 48000)
        self.plain = mm.RxEngine.for_mode("1200", 48000)            # never given auto-carrier
        if self.kind == "auto":
            self.eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
        dtype = np.float32 if self.elem == 4 else np.int16
        if self.host:
            self.keep = (np.zeros((1, STRIDE), dtype), np.zeros((1, 4), mm.FRAME_DTYPE), np.zeros(1, mm.STATE_DTYPE))
            x, fr, st = (C.c_void_p(a.ctypes.data) for a in self.keep)
            self.args = dict(e=self.eng._e, samples=x, nrows=1, stride=STRIDE, n_all=STRIDE, frames=fr,
                             max_frames=4, states=st)
            return
        n = self.k
        x = t.zeros((1, STRIDE), dtype=t.float32 if self.elem == 4 else t.int16, device=dev())
        fr = t.zeros((n, 4, 5), dtype=t.int32, device=dev())
        st = t.zeros((n, mm.STATE_WORDS), dtype=t.int32, device=dev())
        ast = t.zeros((n, mm.api.AUTO_STATE_BYTES), dtype=t.uint8, device=dev())
        each = upload(np.array([STRIDE], np.int32))
        tb = self.eng.tone_bands([1200.0, 1070.0][:n], [2200.0, 1270.0][:n], device=dev())
        self.keep = (x, fr, st, ast, each, tb)
        P = mm.api._ptr
        self.args = dict(e=self.eng._e, samples=P(x), nrows=1, stride=STRIDE, each=P(each), n_all=STRIDE,
                         frames=P(fr), max_frames=4, states=P(st), ast=P(ast), tb=P(tb), k=n,
                         stream=mm.api._stream_handle())

    def misaligned(self):
        return C.c_void_p(self.args["samples"].value + 4)

    def __call__(self, **overrides):
        a = dict(self.args, **overrides)
        fn = getattr(mm.api.lib(), "fsk_b200_" + self.name)
        if self.host:
            return fn(a["e"], a["samples"], a["nrows"], a["stride"], a["n_all"], a["frames"], a["max_frames"],
                      a["states"])
        head = (a["e"], a["samples"], a["nrows"], a["stride"], a["each"], a["n_all"])
        out = (a["frames"], a["max_frames"], a["states"])
        if self.kind == "fixed":
            return fn(*head, *out, a["stream"])
        if self.kind == "auto":
            return fn(*head, *out, a["ast"], None, a["stream"])
        if self.kind == "tones":
            return fn(*head, a["tb"], *out, a["stream"])
        return fn(*head, a["k"], a["tb"], *out, a["stream"])


def refusals(c):
    """(what, overrides) of every refusal that applies to the call"""
    cases = [("NULL engine", dict(e=None)),
             ("NULL samples", dict(samples=None)),
             ("stride not a multiple of 4", dict(stride=STRIDE + 2, n_all=8)),
             ("NULL frames", dict(frames=None)),
             ("NULL states", dict(states=None)),
             ("max_frames 0", dict(max_frames=0)),
             ("nsamples_all above the stride", dict(each=None, n_all=STRIDE + 4)),
             ("nsamples_all above 2^32 - 4", dict(stride=1 << 40, n_all=TOP - 3)),
             ("2^31 rows", dict(nrows=1 << 31))]
    if not c.host:
        cases.append(("misaligned samples", dict(samples=c.misaligned())))
    if c.elem == 2 and not c.host:
        cases.append(("stride not a multiple of 8", dict(stride=STRIDE + 4, n_all=8)))
    if c.kind == "auto":
        cases += [("NULL auto_states", dict(ast=None)), ("auto-carrier not set", dict(e=c.plain._e))]
    if c.kind in ("tones", "channels"):
        cases.append(("NULL tone_bands", dict(tb=None)))
    if c.kind == "channels":
        cases += [("0 channels per row", dict(k=0)), ("2^31 channels", dict(nrows=1 << 30))]
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CALLS))
def test_rx_call_refusals_launch_nothing(name):
    c = Call(name)
    for what, kw in refusals(c):
        before = mm.launch_count()
        assert c(**kw) == -EINVAL, (name, what)
        assert mm.launch_count() == before, (name, what)
        err = mm.api.lib().fsk_b200_last_error().decode()
        assert err.startswith(c.family + ":"), (name, what, err)
        if what == "nsamples_all above 2^32 - 4":
            assert "2^32 - 4" in err, (name, err)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CALLS))
def test_rx_call_with_no_rows(name):
    """nrows 0 returns 0 before the common checks (a NULL engine included); the kind's own preconditions
    come first"""
    c = Call(name)
    refused = []
    if c.kind == "auto":
        refused = [dict(e=None), dict(e=c.plain._e)]
    if c.kind in ("tones", "channels"):
        refused = [dict(e=None), dict(tb=None)] + ([dict(k=0)] if c.kind == "channels" else [])
    taken = [dict(), dict(samples=None, frames=None, states=None, max_frames=0, n_all=TOP - 1)]
    if c.kind in ("fixed", "host"):
        taken.append(dict(e=None))
    before = mm.launch_count()
    for kw in refused:
        assert c(nrows=0, **kw) == -EINVAL, (name, kw)
    for kw in taken:
        assert c(nrows=0, **kw) == 0, (name, kw)
    assert mm.launch_count() == before, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CALLS))
def test_rx_call_launches_its_kernel_family(name):
    c = Call(name)
    before = mm.launch_count()
    assert c() == 0, (name, mm.api.lib().fsk_b200_last_error().decode())
    sync()
    assert mm.launch_count() > before, name
    lk = c.eng.last_kernel()
    assert lk.startswith(KERNEL[c.kind]), (name, lk)
    assert lk.endswith(" channels=2") == (c.kind == "channels"), (name, lk)
