"""The drop-in boundary, end to end: the UNMODIFIED reference CLI -- its main(), rx loop, decoders
and its own src/fsk.h -- linked against this repository's library instead of src/fsk.c + FFTW
(oracle/Makefile: _ref/minimodem_dropin), run on the reference's own test invocations
(tests/*.test, tests/self-test; restated in tests/refcases.py, texts and results in tests/golden/).

Here (no GPU) the library behind the binary is the emulation build of the kernels' source
(tests/emu), put in front of the product library with LD_LIBRARY_PATH; on an H100 the same
binary runs on the product library in tests/test_gpu_parity.py::test_reference_cli_on_this_library."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import golden_util as gu      # noqa: E402
import orc                    # noqa: E402
import refcases               # noqa: E402
from make_golden import read_wav  # noqa: E402
from clicases import emulation_as_product, random_invocation  # noqa: E402

DROPIN = os.path.join(ROOT, "oracle", "_ref", "minimodem_dropin")


def _nocarrier_ampl(stderr):
    line = [ln for ln in stderr.decode(errors="replace").splitlines() if ln.startswith("### NOCARRIER")][0]
    return float(line.split("ampl=")[1].split()[0])


def _amplitude_ok(volume, rx_ampl):
    """tests/30-amplitude.test's rule: the rx amplitude within 0.01 of the tx volume ("E" counts as 0.0), or, for
    integer samples at a volume above 1.0 (clamped), between 1.00 and 1.02."""
    a = 0.0 if volume == "E" else float(volume)
    return (a - 0.01 < rx_ampl < a + 0.01) or (a > 1.0 and 1.00 < rx_ampl < 1.02)


@pytest.mark.ref
def test_reference_self_tests_pass_with_this_library_behind_the_reference_cli(tmp_path):
    """The runs of the reference's own test scripts (tests/*.test: every tests/self-test invocation, restated as
    data in tests/refcases.py with the texts in tests/golden/) through the drop-in binary, tx and rx, with the
    scripts' pass conditions: the decoded text equals what was sent (for Caller-ID, the message text the reference
    decoded, committed as its stdout), `confidence=inf ... (rate perfect)` for the -P runs, the rx amplitude
    against the tx volume for 30/31, and three identical tx runs for 16/17.  The tx audio must also be the audio
    the unmodified reference CLI produced (its hash is committed)."""
    if not os.path.exists(DROPIN):
        pytest.skip("oracle/_ref/minimodem_dropin not built")
    env = dict(os.environ, LD_LIBRARY_PATH=emulation_as_product())
    wav = str(tmp_path / "x.wav")
    failed = []
    for case in refcases.CASES:
        g = gu.load(case["name"])
        text = bytes(g["text"])
        subprocess.run([DROPIN, "--tx", "--file", wav] + list(case["tx"]), input=text, env=env, check=True)
        audio, rate, _ = read_wav(wav)
        if gu.sha(audio) != bytes(g["audio_sha256"]):
            failed.append((case["name"], "tx audio differs from the reference's"))
            continue
        r = subprocess.run([DROPIN, "--rx", "--file", wav] + list(case["rx"]), env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, timeout=900)
        want = bytes(g["stdout"]) if case["tx_ascii"] else text
        if r.returncode != 0 or r.stdout != want:
            failed.append((case["name"], r.returncode, r.stdout[:60], r.stderr[-200:]))
        elif case["perfect"] and not re.search(rb"confidence=inf .* \(rate perfect\)", r.stderr):
            failed.append((case["name"], "not perfect", r.stderr[-200:]))
        elif case["name"].startswith(("30-amplitude", "31-amplitude")) and not _amplitude_ok(
                case["name"].rsplit("-", 1)[1], _nocarrier_ampl(r.stderr)):
            failed.append((case["name"], "rx amplitude", r.stderr[-200:]))
    for extra in ([], ["--float-samples"]):                 # 16/17-verify-tx-consistent
        text = bytes(gu.load("01-self-test-1200")["text"])
        outs = []
        for i in range(3):
            w = str(tmp_path / ("tx%d.wav" % i))
            subprocess.run([DROPIN, "--tx", "--file", w, "1200"] + extra, input=text, env=env, check=True)
            outs.append(open(w, "rb").read())
        if not outs[0] == outs[1] == outs[2]:
            failed.append(("verify-tx-consistent", extra))
    assert len(refcases.CASES) == 44
    assert not failed, failed


@pytest.mark.ref
@pytest.mark.parametrize("seed", range(40))
def test_dropin_cli_equals_reference_cli_on_a_random_invocation(seed, tmp_path):
    """The reference's main() on this library (emulated kernels) against the reference's main() on its
    own src/fsk.c, for a random baud rate / sample rate / framing / bit order / tone pair: the same
    stdout, the same CARRIER / NOCARRIER lines (confidence to the parity tolerance)."""
    import numpy as np
    if not os.path.exists(DROPIN):
        pytest.skip("oracle/_ref/minimodem_dropin not built")
    rng = np.random.default_rng(9000 + seed)
    mode, kw, tx_args, rx_args, flt, vol = random_invocation(rng)
    text = bytes(rng.integers(32, 127, int(rng.integers(4, 30)), dtype=np.uint8)) + b"\n"
    wav = str(tmp_path / "x.wav")
    subprocess.run([orc.REF_CLI, "--tx", "--file", wav] + tx_args, input=text, check=True)
    ref = subprocess.run([orc.REF_CLI, "--rx", "--file", wav] + rx_args, stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, check=True)
    env = dict(os.environ, LD_LIBRARY_PATH=emulation_as_product())
    our = subprocess.run([DROPIN, "--rx", "--file", wav] + rx_args, env=env, stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, timeout=600)
    assert our.returncode == 0, our.stderr[-400:]
    assert our.stdout == ref.stdout, (rx_args, our.stdout[:40], ref.stdout[:40])
    a = [ln.split() for ln in our.stderr.decode().splitlines() if ln.startswith("###")]
    b = [ln.split() for ln in ref.stderr.decode().splitlines() if ln.startswith("###")]
    assert len(a) == len(b), (our.stderr, ref.stderr)
    for fa, fb in zip(a, b):
        if fa[1] == "NOCARRIER":
            assert fa[:3] == fb[:3] and fa[4:] == fb[4:], (fa, fb)
            assert gu.close(float(fa[3].split("=")[1]), float(fb[3].split("=")[1]), 2e-3, cond=gu.CONF_COND)
        else:
            assert fa == fb
