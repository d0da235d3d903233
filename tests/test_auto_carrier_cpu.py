"""--auto-carrier (-a): the oracle's rx loop with the carrier scan (oracle/auto_oracle.c) against the
UNMODIFIED reference CLI (oracle/_ref/minimodem_ref), on random invocations.  The audio puts one or two
transmissions on random tone pairs (offset from the band centres, or with the mode's own shift) behind
silent lead-ins as long as several sample rings, with noise below and above the detection threshold,
`--inverted`, a gap that makes the receiver drop the carrier and rescan, and mark tones so low that the
space band falls below band 1.  LITERAL mode (the reference's sample ring) must print what the CLI
prints: the decoded text, and every CARRIER line (with its frequency) and NOCARRIER line in order.
FLAT mode (the batched semantic: the whole stream searchable, the scan over the virtual ring count)
must agree with it wherever the ring does not limit the reference: at 400 baud and above.  Below,
the search that follows a scan reaches past the half ring the reference holds then."""
import struct
import subprocess

import numpy as np
import pytest

import autoorc
import golden_util as gu
import orc
import refcases

# (mode, sample rates): the three preset classes of src/minimodem.c:900-934
CLASSES = [("1200", (48000, 22050, 11025)), ("600", (48000, 8000)), ("300", (48000, 8000)),
           ("110", (8000,)), ("rtty", (8000,))]


def write_wav_float(path, audio, rate):
    """A mono IEEE-float WAV file, as `minimodem --tx --float-samples` writes one."""
    data = np.ascontiguousarray(audio, "<f4").tobytes()
    fmt = struct.pack("<HHIIHH", 3, 1, rate, rate * 4, 4, 32)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt)
        f.write(b"data" + struct.pack("<I", len(data)) + data)


def transmission(rng, mode, rate, bw, b_shift, inverted, low=False):
    """Audio of random data words (printable characters for 8-bit framings) on a random tone pair."""
    nb = int((rate + bw / 2) / bw) // 2 + 1
    if low:
        bm = int(rng.integers(1, max(2, -b_shift if b_shift < 0 else 2)))
    else:
        lo, hi = max(2, 2 - b_shift), min(nb - 3, nb - 3 - b_shift)
        bm = int(rng.integers(lo, max(lo + 1, hi)))
    mark = float(bm * bw + rng.uniform(-0.3, 0.3) * bw)
    if rng.random() < 0.7:
        space = mark + b_shift * bw
    else:
        m0 = orc.Mode(mode, sample_rate=rate)
        space = mark - m0.autodetect_shift
    space = min(max(space, bw), rate / 2 - bw)
    m = orc.Mode(mode, sample_rate=rate, mark=mark, space=space, inverted=inverted)
    lo, hi = (33, 127) if m.n_data_bits >= 7 else (0, 1 << m.n_data_bits)
    words = rng.integers(lo, hi, int(rng.integers(4, 24)), dtype=np.uint64).astype(np.uint32)
    return orc.tx_words(m, words)


def ring_limited(m):
    """True when a search right after a scan that emptied the ring reads past the half ring the
    reference then holds (fsk_oracle.c's touch_max): the reference reads stale ring content there,
    the batched receiver the stream itself (DESIGN.md section 5)."""
    d = m.derived()
    touch = int(d.nsamples_per_bit + d.nsamples_overscan) + 2 + d.expect_nsamples + int(d.nsamples_per_bit) + 2
    return touch > d.samplebuf_size // 2


def random_case(seed, classes=CLASSES):
    rng = np.random.default_rng(7000 + seed)
    mode, rates = classes[int(rng.integers(len(classes)))]
    rate = int(rng.choice(rates))
    inverted = rng.random() < 0.25
    m = orc.Mode(mode, sample_rate=rate)
    bw = float(m.band_width)
    b_shift = autoorc.b_shift(m, inverted)
    S = int(m.derived().samplebuf_size)
    lead = int(rng.choice([0, S // 3, S + int(rng.integers(1, S)), 3 * S]))
    parts = [np.zeros(lead, np.float32)]
    parts.append(transmission(rng, mode, rate, bw, b_shift, inverted, low=rng.random() < 0.15))
    if rng.random() < 0.5:           # a gap, then a second transmission on other tones
        gap = int(rng.uniform(30, 80) * float(m.derived().nsamples_per_bit))
        parts.append(np.zeros(gap, np.float32))
        parts.append(transmission(rng, mode, rate, bw, b_shift, inverted))
    parts.append(np.zeros(int(rng.integers(0, S)), np.float32))
    audio = np.concatenate(parts)
    sigma = float(rng.choice([0.0, 0.0, 3e-4, 0.03]))   # below and above the 0.001 threshold
    if sigma:
        audio = (audio + rng.normal(0, sigma, audio.size)).astype(np.float32)
    rx_args = [mode, "--samplerate", str(rate), "-a"] + (["--inverted"] if inverted else [])
    return orc.Mode(mode, sample_rate=rate, inverted=inverted), audio, rate, rx_args, inverted


def compare_lines(got, want, ctx):
    assert [g.split()[1] for g in got] == [w.split()[1] for w in want], (ctx, got, want)
    for a_line, b_line in zip(got, want):
        if a_line.startswith("### CARRIER"):
            assert a_line == b_line, (ctx, a_line, b_line)
            continue
        fa, fb = a_line.split(), b_line.split()
        assert fa[:3] == fb[:3] and fa[4:] == fb[4:], (ctx, a_line, b_line)
        assert gu.close(float(fa[3].split("=")[1]), float(fb[3].split("=")[1]), 2e-3, cond=gu.CONF_COND)


@pytest.mark.ref
@pytest.mark.parametrize("seed", range(60))
def test_auto_oracle_matches_the_reference_cli(seed, tmp_path):
    m, audio, rate, rx_args, inverted = random_case(seed)
    wav = str(tmp_path / "x.wav")
    write_wav_float(wav, audio, rate)
    r = subprocess.run([orc.REF_CLI, "--rx", "--file", wav] + rx_args, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, check=True)
    res = autoorc.rx_run(m, audio, literal=True, inverted=inverted)
    assert orc.ref_decode(m, res["frames"]) == r.stdout, (rx_args, r.stdout[:60])
    want = [ln.strip() for ln in r.stderr.decode().splitlines() if ln.startswith("### ")]
    compare_lines(autoorc.stat_lines(m, res), want, rx_args)


@pytest.mark.parametrize("seed", range(60))
def test_flat_auto_oracle_matches_literal(seed):
    m, audio, rate, rx_args, inverted = random_case(seed, CLASSES[:2])
    assert not ring_limited(m)
    lit = autoorc.rx_run(m, audio, literal=True, inverted=inverted)
    flat = autoorc.rx_run(m, audio, literal=False, inverted=inverted)
    assert flat["frames"] == lit["frames"], rx_args
    assert flat["reports"] == lit["reports"] and flat["frame_band"] == lit["frame_band"], rx_args
    assert flat["report_band"] == lit["report_band"], rx_args


def test_the_cases_cover_every_path():
    """The seeds reach a decode, a rescan after a drop onto another band, a lead-in longer than the
    ring, and --inverted."""
    seen = set()
    for seed in range(60):
        m, audio, rate, rx_args, inverted = random_case(seed)
        res = autoorc.rx_run(m, audio, literal=False, inverted=inverted)
        if res["frames"]:
            seen.add("decode")
        if len(set(res["report_band"])) > 1:
            seen.add("rescan onto another band")
        if inverted and res["frames"]:
            seen.add("inverted")
        if res["frames"] and res["frames"][0][5] > m.derived().samplebuf_size:
            seen.add("long lead-in")
    assert seen == {"decode", "rescan onto another band", "inverted", "long lead-in"}, seen


def test_an_out_of_range_space_band_is_rejected():
    """A Bell103 mark tone in band 2 has its space band (b_shift -4) below band 1: the scan finds the
    carrier every time and rejects it, so nothing decodes; the same text 1 kHz higher decodes."""
    m = orc.Mode("300", sample_rate=8000)
    assert autoorc.b_shift(m) == -4
    out = []
    for mark in (100.0, 1100.0):
        tx = orc.Mode("300", sample_rate=8000, mark=mark, space=mark - 200)
        words = np.frombuffer(b"HELLO", np.uint8).astype(np.uint32)
        a = np.concatenate([np.zeros(500, np.float32), orc.tx_words(tx, words), np.zeros(500, np.float32)])
        out.append(autoorc.rx_run(m, a)["frames"])
    assert out[0] == [] and len(out[1]) >= 5


@pytest.mark.ref
@pytest.mark.parametrize("name", ["cli-auto-carrier", "cli-auto-carrier-rtty"])
def test_auto_oracle_reproduces_the_cli_auto_carrier_vectors(name):
    """The reference CLI's own --auto-carrier runs, committed under tests/golden: both oracle modes
    print its stdout and its stat lines."""
    case = refcases.BY_NAME[name]
    g = gu.load(name)
    _, rx = gu.modes(case)
    a = gu.audio(case, g)
    want = [ln.strip() for ln in bytes(g["stderr"]).decode().splitlines() if ln.startswith("### ")]
    for literal in (True, False):
        res = autoorc.rx_run(rx, a, literal=literal)
        assert orc.ref_decode(rx, res["frames"]) == bytes(g["stdout"]), (name, literal)
        compare_lines(autoorc.stat_lines(rx, res), want, (name, literal))


def test_gpu_auto_carrier_file_on_the_emulated_kernels():
    """tests/test_gpu_auto_carrier.py on the host SIMT emulation of the kernels (tests/emu), with the
    emulated sqrt moved by up to 64 ulp."""
    from gpudev import run_emulated
    tail = run_emulated("not live_stream", "late", 1800, module="test_gpu_auto_carrier.py",
                        extra_env={"FSK_EMU_ULP": "64"})
    assert " passed" in tail and "failed" not in tail


def test_the_auto_screen_replays_the_oracle_exactly():
    """autoorc.AutoSearch (tests/tie_screen.py's search on the tones of the moment) with no perturbation
    is the auto oracle's own search: same records, reports and bands, bit for bit."""
    for seed in range(12):
        m, audio, rate, rx_args, inverted = random_case(seed)
        want = autoorc.rx_run(m, audio, inverted=inverted)
        s = autoorc.AutoSearch(m, 0.0, 0)
        got = autoorc.rx_run(m, audio, inverted=inverted, find_frame=s.find_frame)
        for k in ("frames", "reports", "frame_band", "report_band"):
            assert got[k] == want[k], (rx_args, k)
