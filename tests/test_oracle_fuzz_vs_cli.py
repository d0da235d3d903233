"""Differential fuzz of the oracle against the UNMODIFIED reference CLI (oracle/_ref/minimodem_ref),
run here where /root/reference exists: random baud rates, sample rates, framings, bit orders, tone
pairs and payloads go through the reference's own transmitter and receiver; the oracle's
transmitter must produce the same samples, and the oracle's rx loop (LITERAL mode, the reference's
ring and all) the same text and the same stat lines.  The golden vectors pin fixed cases; this pins
the space between them."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_util as gu
import orc
from clicases import random_invocation

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden import read_wav  # noqa: E402

pytestmark = pytest.mark.ref


@pytest.mark.parametrize("seed", range(60))
def test_oracle_matches_the_reference_cli_on_a_random_invocation(seed, tmp_path):
    rng = np.random.default_rng(5000 + seed)
    mode, kw, tx_args, rx_args, flt, vol = random_invocation(rng)
    text = bytes(rng.integers(32, 127, int(rng.integers(4, 40)), dtype=np.uint8)) + b"\n"
    wav = str(tmp_path / "x.wav")
    subprocess.run([orc.REF_CLI, "--tx", "--file", wav] + tx_args, input=text, check=True)
    r = subprocess.run([orc.REF_CLI, "--rx", "--file", wav] + rx_args, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, check=True)
    audio, rate, is_float = read_wav(wav)
    m = orc.Mode(mode, **kw)
    # the transmitter restatement: same samples
    words = orc.ref_encode("ascii8", text) & ((1 << m.n_data_bits) - 1)
    mine = orc.tx_words(m, words, vol, 4096, flt)
    assert mine.size == audio.size, (tx_args, mine.size, audio.size)
    assert hashlib.sha256(mine.tobytes()).digest() == hashlib.sha256(audio.tobytes()).digest(), tx_args
    # the rx loop restatement, with the reference's ring: same text, same stat lines
    res = orc.rx_run(m, audio, literal=True)
    assert orc.ref_decode(m, res["frames"]) == r.stdout, (rx_args, r.stdout[:40])
    want = [ln.strip() for ln in r.stderr.decode().splitlines() if ln.startswith("### NOCARRIER")]
    got = [orc.report_line(m, rp) for rp in res["reports"]]
    assert len(got) == len(want), (rx_args, got, want)
    for a_line, b_line in zip(got, want):
        fa, fb = a_line.split(), b_line.split()
        assert fa[:3] == fb[:3] and fa[4:] == fb[4:], (a_line, b_line)
        assert gu.close(float(fa[3].split("=")[1]), float(fb[3].split("=")[1]), 2e-3, cond=gu.CONF_COND)
