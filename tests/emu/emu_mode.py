"""TEST INFRASTRUCTURE: switch the parity tests of tests/test_gpu_parity.py to the host SIMT
emulation of the kernels (tests/emu/cuda_runtime.h).  Active only when FSK_B200_EMU=1:

    FSK_B200_EMU=1 python -m pytest tests/test_gpu_parity.py -m gpu -k "..."

The product binding (minimodem_b200/api.py) is not changed for this: the emulation library is
selected through the binding's existing FSK_B200_LIB override, and the three things the tests
need from CUDA -- "this tensor is device memory", a stream handle, a device synchronize -- are
patched here, in the test process only."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libfsk_b200_emu.so")


def active():
    return os.environ.get("FSK_B200_EMU") == "1"


def build():
    subprocess.check_call(["make", "-s", "-C", HERE])
    return LIB


def activate():
    """Call before minimodem_b200 is imported.  FSK_EMU_LIB selects another emulation build
    (e.g. one made with `make OUT=... BUILD=... EXTRA=-DFSK_MULTI_MIN_N=64` to try a compile-time variant)."""
    global LIB
    if os.environ.get("FSK_EMU_LIB"):
        LIB = os.environ["FSK_EMU_LIB"]
    else:
        build()
    os.environ["FSK_B200_LIB"] = LIB
    import torch
    import minimodem_b200.api as api
    assert api.LIB_PATH == LIB, "minimodem_b200 was imported before the emulation was selected"
    api.ALLOW_NON_PRODUCT_LIBRARY = True      # the binding refuses the emulation build otherwise
    # host memory plays device memory
    torch.Tensor.is_cuda = property(lambda self: True)
    torch.cuda.synchronize = lambda *a, **k: None
    torch.cuda.is_available = lambda: True
    api._stream_handle = lambda stream=None: C.c_void_p(0)
    return torch.device("cpu")
