"""Random modes through the emulated kernels (run by tests/test_emu_parity.py in a subprocess with
FSK_B200_EMU=1; the file name keeps pytest from collecting it on its own).

Framings, bit orders, rates and baud rates that no committed vector has: the oracle's transmitter
makes the stream, the oracle's rx loop says what the records must be, the kernels' source (on the
host SIMT emulator) has to produce them -- exact bits, frame starts and acquire flags, confidence
and amplitude to the parity tolerance.  This is a logic check of the kernels over geometry the
vectors do not reach (window counts from 7 to 44 bits, every lane split the launcher picks,
fractional samples per bit, long windows), run on the emulator.  Random framings reach the hardware
through tests/test_gpu_instantiations.py instead: there every stream first goes through a
deterministic near-tie screen (tests/tie_screen.py), so that a stream whose records a knife-edge
decision could flip under the device's approximate units is known in advance rather than being a
flaky case, and all other streams are compared exactly."""
import numpy as np
import pytest

import golden_util as gu
import minimodem_b200 as mm
import orc
import rxcases
from gpudev import upload
from rxcases import BAUDS, RATES, engine_for, rx_on_gpu
from rxfam import as_oracle_frames, compare_frames, compare_reports, reports_of

pytestmark = pytest.mark.gpu

def random_mode(rng):
    while True:
        baud = int(rng.choice(BAUDS))
        rate = int(rng.choice(RATES))
        spb = rate / baud
        if spb < 6 or spb > 700:
            continue
        kw = dict(sample_rate=rate)
        kw["n_data_bits"] = int(rng.choice([5, 6, 7, 8, 9, 12, 16, 24, 32]))
        kw["startbits"] = int(rng.choice([1, 1, 2, 3, 5]))
        kw["stopbits"] = float(rng.choice([1.0, 1.0, 1.5, 2.0, 3.0]))
        kw["msb_first"] = bool(rng.integers(0, 2))
        kw["invert_start_stop"] = bool(rng.integers(0, 2))
        kw["inverted"] = bool(rng.integers(0, 2))
        if kw["n_data_bits"] + kw["startbits"] + kw["stopbits"] + 1 > 48:
            continue
        try:
            m = orc.Mode(str(baud), **kw)
            m.derived()
            orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
        except Exception:
            continue
        if max(m.mark_f, m.space_f) >= rate / 2 - m.band_width:
            continue
        return str(baud), kw


@pytest.mark.parametrize("seed", range(64))
def test_random_mode_records_match_the_oracle(seed):
    rng = np.random.default_rng(1000 + seed)
    mode, kw = random_mode(rng)
    rx = orc.Mode(mode, **kw)
    nwords = int(rng.integers(6, 18))
    words = rng.integers(0, 1 << rx.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
    streams = []
    for s in range(3):
        a = orc.tx_words(rx, words, float(rng.uniform(0.3, 1.0)), 4096, True)
        lead = int(rng.integers(0, 3 * int(rx.derived().nsamples_per_bit) + 1))
        x = np.concatenate([np.zeros(lead, np.float32), a])
        x = (x + np.float32(0.01) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
    eng, _ = engine_for((mode, kw))
    recs, st = rx_on_gpu(eng, streams)
    decoded = 0
    for s, x in enumerate(streams):
        want = orc.rx_run(rx, x, literal=False)
        got = as_oracle_frames(recs[s])
        compare_frames(got, want["frames"], "%s %r stream %d" % (mode, kw, s))
        compare_reports(reports_of(recs[s], st[s]), want["reports"], "%s %r stream %d" % (mode, kw, s))
        decoded += len(got)
    assert decoded >= nwords, (mode, kw, decoded, nwords)


import refcases  # noqa: E402


@pytest.mark.parametrize("case", refcases.MORE, ids=[c["name"] for c in refcases.MORE])
def test_second_batch_of_option_vectors(case):
    """tests/refcases.py MORE: runs of the unmodified reference CLI that are on the CPU lists only;
    here the emulated kernels have to reproduce their records, decoded bytes and stat lines."""
    if case["ring_limited"]:
        # the kernels follow the flat semantic: all of the text, of which the reference printed the start
        g = gu.load(case["name"])
        _, rx = gu.modes(case)
        a = gu.audio(case, g)
        eng, _ = engine_for(case)
        (recs,), st = rx_on_gpu(eng, [a])
        got = as_oracle_frames(recs)
        compare_frames(got, orc.rx_run(rx, a, literal=False)["frames"], case["name"])
        out = orc.decode_records(rx, refcases.decoder_of(case, rx), orc.frame_records(got))
        assert out == bytes(g["text"]) and out.startswith(bytes(g["stdout"]))
        return
    rxcases.check_reference_vector(case)


@pytest.mark.parametrize("seed", range(40))
def test_batched_kernels_print_what_the_reference_cli_prints(seed, tmp_path):
    """Closing the loop without the oracle in between: a random invocation goes through the
    unmodified reference CLI (transmit, then receive), and the same audio through rx_batch +
    decode_batch on the emulated kernels; the text must be the CLI's stdout.  (Where the reference's
    sample ring makes it read stale samples -- slow modes, DESIGN.md 5 item 2 -- the oracle's two
    modes already differ and the case is skipped.)"""
    import os
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import read_wav
    from clicases import random_invocation
    if not orc.have_ref() or not os.path.exists(orc.REF_CLI):
        pytest.skip("needs the reference CLI (oracle/_ref)")
    rng = np.random.default_rng(12000 + seed)
    mode, kw, tx_args, rx_args, flt, vol = random_invocation(rng)
    text = bytes(rng.integers(32, 127, int(rng.integers(4, 30)), dtype=np.uint8)) + b"\n"
    wav = str(tmp_path / "x.wav")
    subprocess.run([orc.REF_CLI, "--tx", "--file", wav] + tx_args, input=text, check=True)
    ref = subprocess.run([orc.REF_CLI, "--rx", "--file", wav] + rx_args, stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, check=True)
    audio, rate, _ = read_wav(wav)
    m = orc.Mode(mode, **kw)
    lit = orc.rx_run(m, audio, literal=True)["frames"]
    flat = orc.rx_run(m, audio, literal=False)["frames"]
    if [f[:1] + f[3:5] for f in lit] != [f[:1] + f[3:5] for f in flat]:
        pytest.skip("the reference's ring changes this one")
    eng, _ = engine_for((mode, kw))
    n = audio.size
    buf = np.zeros((2, rxcases.pad4(n)), np.float32)
    buf[:, :n] = audio
    frames, states = eng.rx_batch(upload(buf), nsamples=n)
    out, cnt = eng.decode_batch(mm.decoder_for_mode(mode, m.n_data_bits), frames, states)
    o, c = out.cpu().numpy(), cnt.cpu().numpy()
    for s in range(2):
        assert bytes(o[s, :c[s]]) == ref.stdout, (rx_args, bytes(o[s, :c[s]])[:40], ref.stdout[:40])
