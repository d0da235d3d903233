"""The kernels' SOURCE on the host SIMT emulator (tests/emu): the parity tests that normally need
an H100 (tests/test_gpu_parity.py, marker `gpu`) run here on CPU cores against the emulation
build of the very same minimodem_b200/csrc/*.cu / *.cuh files.  It checks what an emulator can
check -- control flow, ring bookkeeping, lane exchanges, cp.async ordering (copies land as late
as the code's own waits allow, or at once), record and state formats, every decoder -- before
GPU minutes are spent; timing, the approximate sqrt/div units and the hardware itself are
checked only by the `gpu` run.  The emulation library is never loaded by the product."""
import os
import subprocess

import pytest

from gpudev import run_emulated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parity_suite_on_the_emulated_kernels_late_copies():
    """Everything but the large round-trip batches; cp.async copies land only at the waits."""
    tail = run_emulated("not roundtrip", "late", 1500)
    assert " passed" in tail and "failed" not in tail


def test_reference_vectors_on_the_emulated_kernels_eager_copies():
    """The reference vectors and the resume/ragged cases with copies landing at issue: a copy
    requested while its target is still being read would corrupt the window."""
    tail = run_emulated("reference_vectors or edge_cases or overflow or lane_split", "eager", 900)
    assert " passed" in tail and "failed" not in tail


def test_random_modes_and_option_vectors_on_the_emulated_kernels():
    """tests/emu_fuzz.py: 64 random framings / rates / bit orders: oracle TX -> emulated kernels -> records
    equal to the oracle's rx loop; and the second batch of reference-CLI option vectors (tests/refcases.py
    MORE).  Streams that keep losing and finding the carrier are in tests/test_gpu_carrier_sessions.py."""
    tail = run_emulated("random_mode or second_batch or batched_kernels_print", "late", 1200, module="emu_fuzz.py")
    assert "failed" not in tail and ("113 passed" in tail or "114 passed" in tail)     # one seed is ring-limited


def test_every_instantiation_on_the_emulated_kernels_with_perturbed_units():
    """tests/test_gpu_instantiations.py at the device's sizes (under a minute): every rx, find-frame and
    transmitter instance the launchers can dispatch (the TMA bulk fills excepted: not emulated), on random
    framings, with the approximate sqrt and divide perturbed by up to 64 ulp (FSK_EMU_ULP=64).  Every stream the near-tie
    screen calls robust must still give the oracle's records: the screen's margin covers arithmetic that
    differs from the oracle's, which is what makes the random cases exact on the GPU."""
    tail = run_emulated("instantiation or screen or odd_stride", "late", 900, module="test_gpu_instantiations.py",
                        extra_env={"FSK_EMU_ULP": "64"})
    assert " passed" in tail and "failed" not in tail


@pytest.mark.parametrize("async_mode", ["eager", "late"])
def test_launch_shapes_on_the_emulated_kernels(async_mode):
    """tests/test_gpu_launch_shapes.py: ring depths, warps per block and neighbours leave every record and
    state as it is (the TMA bulk fill excepted: not emulated).  With copies landing at issue, a look-ahead
    copy that overwrote a window still being read would show."""
    tail = run_emulated("", async_mode, 1800, module="test_gpu_launch_shapes.py")
    assert " passed" in tail and "failed" not in tail


@pytest.mark.parametrize("async_mode", ["eager", "late"])
def test_long_rows_on_the_emulated_kernels(async_mode):
    """tests/test_gpu_long_rows.py: a stream at the end of a row of up to 2^32 - 4 samples (a memfd aliased
    over the whole range) decodes as at the start of a small row, in every rx family (the TMA bulk fill
    excepted: not emulated); the row-limit refusals, the live push at the cap and the transmitter's bounds."""
    tail = run_emulated("", async_mode, 900, module="test_gpu_long_rows.py")
    assert " passed" in tail and "failed" not in tail


def test_the_emulator_itself():
    """tests/emu/selftest.cpp: hand-verifiable kernels.  Group-masked shuffles / votes with
    divergent trip counts, block barriers and dynamic shared memory give CUDA's results; cp.async
    data is invisible before the issuing thread's wait in `late` mode and visible at once in
    `eager` mode; a lane missing from a *_sync, a lane outside its own mask, a copy past the
    shared-memory allocation and a thread that exits with copies in flight are all reported."""
    emu = os.path.join(ROOT, "tests", "emu")
    subprocess.check_call(["make", "-s", "-C", emu, "selftest"])
    exe = os.path.join(emu, "build", "selftest")
    for case in ("groups", "block", "async"):
        for mode in ("late", "eager"):
            r = subprocess.run([exe, case], env=dict(os.environ, FSK_EMU_ASYNC=mode), stdout=subprocess.PIPE,
                               stderr=subprocess.STDOUT, timeout=120)
            assert r.returncode == 0 and b"ok" in r.stdout, (case, mode, r.stdout[-400:])
    for case, msg in (("deadlock", b"deadlock"), ("wrong_mask", b"mask does not name it"),
                      ("oob", b"outside the block's shared memory"), ("exit_in_flight", b"copies in flight")):
        r = subprocess.run([exe, case], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=120)
        assert r.returncode != 0 and msg in r.stdout, (case, r.returncode, r.stdout[-400:])
