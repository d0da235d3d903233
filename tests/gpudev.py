"""Device plumbing the `gpu` test files share: the device (an H100, or the host SIMT emulation of the
kernels under FSK_B200_EMU=1, tests/emu), host rows and PCM, copies to and from the device, and the runner
that puts a test file's `gpu` tests on the emulated kernels."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def torch():
    return pytest.importorskip("torch")


def mm():
    import minimodem_b200
    return minimodem_b200


def emulated():
    import conftest
    return conftest.EMU_DEVICE is not None


def dev():
    import conftest
    if conftest.EMU_DEVICE is not None:         # FSK_B200_EMU=1: the kernels' source on the host emulator
        return conftest.EMU_DEVICE
    assert torch().cuda.is_available(), "GPU tests need a CUDA device"
    return torch().device("cuda:0")


def sync():
    if not emulated():
        torch().cuda.synchronize()


def upload(a):
    """a device copy (the emulated device shares host memory, so from_numpy alone would alias `a`)"""
    return torch().from_numpy(np.array(a, copy=True, order="C")).to(dev())


def rows(streams, dtype, align=4, n=None):
    """(buf, n): the streams zero-padded into rows of a stride that is a multiple of `align`, and n, the
    longest stream (or the n given)"""
    n = max(len(a) for a in streams) if n is None else n
    stride = (n + align - 1) & ~(align - 1)
    buf = np.zeros((len(streams), stride), dtype)
    for i, a in enumerate(streams):
        buf[i, :len(a)] = a
    return buf, n


def pcm(a):
    """int16 PCM of float samples, rounded in float64 (exact for float32 input, whose product with 32768 is)"""
    return np.clip(np.round(np.asarray(a).astype(np.float64) * 32768.0), -32768, 32767).astype(np.int16)


def widen(x):
    """what the kernels read from int16 rows: s16 / 32768, exactly"""
    return np.asarray(x, np.int16).astype(np.float32) * np.float32(1.0 / 32768.0)


def records(fr, st):
    """(records per channel as bytes, states as numpy) of a call's outputs"""
    fr, st = mm().frames_to_numpy(fr), mm().states_to_numpy(st)
    return [fr[c, :int(st["nframes"][c])].tobytes() for c in range(len(st))], st


def state_rows(st):
    return upload(st.view(np.int32).reshape(len(st), -1))


def bands_tensor(b):
    return upload(np.asarray(b, np.int64).astype(np.uint32).view(np.int32).reshape(-1, 2))


def run_emulated(select, async_mode, timeout, module="test_gpu_parity.py", extra_env=None):
    """the `gpu` tests of tests/<module> selected by -k `select`, on the host SIMT emulation of the kernels in
    a subprocess, cp.async copies landing `async_mode` ("eager" or "late"); returns the tail of its output"""
    env = dict(os.environ, FSK_B200_EMU="1", FSK_EMU_ASYNC=async_mode, **(extra_env or {}))
    env.pop("FSK_B200_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", module),
                        "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "-k", select],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout)
    tail = r.stdout.decode(errors="replace")[-3000:]
    assert r.returncode == 0, tail
    return tail
