"""The kernels' SOURCE on the host SIMT emulator (tests/emu): the parity tests that normally need
an H100 (tests/test_gpu_parity.py, marker `gpu`) run here on CPU cores against the emulation
build of the very same minimodem_b200/csrc/*.cu / *.cuh files.  It checks what an emulator can
check -- control flow, ring bookkeeping, lane exchanges, cp.async ordering (copies land as late
as the code's own waits allow, or at once), record and state formats, every decoder -- before
GPU minutes are spent; timing, the approximate sqrt/div units and the hardware itself are
checked only by the `gpu` run.  The emulation library is never loaded by the product."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_emulated(select, async_mode, timeout, module="test_gpu_parity.py"):
    env = dict(os.environ, FSK_B200_EMU="1", FSK_EMU_ASYNC=async_mode)
    env.pop("FSK_B200_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", module),
                        "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "-k", select],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout)
    tail = r.stdout.decode(errors="replace")[-3000:]
    assert r.returncode == 0, tail
    return tail


def test_parity_suite_on_the_emulated_kernels_late_copies():
    """Everything but the large round-trip batches; cp.async copies land only at the waits."""
    tail = run_emulated("not roundtrip", "late", 1500)
    assert " passed" in tail and "failed" not in tail


def test_reference_vectors_on_the_emulated_kernels_eager_copies():
    """The reference vectors and the resume/ragged cases with copies landing at issue: a copy
    requested while its target is still being read would corrupt the window."""
    tail = run_emulated("reference_vectors or edge_cases or overflow or lane_split", "eager", 900)
    assert " passed" in tail and "failed" not in tail


def test_random_modes_and_dropouts_on_the_emulated_kernels():
    """tests/emu_fuzz.py: 64 random framings / rates / bit orders, 24 streams that keep losing and
    finding the carrier (also decoded in 3-frame record buffers with resume): oracle TX -> emulated
    kernels -> records equal to the oracle's rx loop; and the second batch of reference-CLI option
    vectors (tests/refcases.py MORE)."""
    tail = run_emulated("random_mode or dropouts or second_batch or batched_kernels_print", "late", 1200,
                        module="emu_fuzz.py")
    assert "failed" not in tail and ("137 passed" in tail or "138 passed" in tail)     # one seed is ring-limited


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
