import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


# FSK_B200_EMU=1: run the "gpu" tests on the host SIMT emulation of the kernels (tests/emu)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_mode  # noqa: E402

EMU_DEVICE = emu_mode.activate() if emu_mode.active() else None


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref (the reference compiled in place)")


def pytest_collection_modifyitems(config, items):
    import orc
    if not orc.have_ref():
        # built from /root/reference when present (this container); prebuilt on the GPU box
        try:
            orc.build_ref()
        except Exception:
            pass
    if not orc.have_ref():
        skip = pytest.mark.skip(reason="oracle/_ref not built and /root/reference absent")
        for it in items:
            if "ref" in it.keywords:
                it.add_marker(skip)
