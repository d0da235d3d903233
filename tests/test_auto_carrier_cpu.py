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
import rxcases

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
    """(oracle mode, audio, rate, CLI arguments, inverted) of a random invocation"""
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


# the carrier-session streams of the auto call (tests/test_gpu_carrier_sessions.py): every AUTO_COMBOS preset,
# and --inverted at 1200 baud
SESSIONS = ["session:%s@%d" % w for w in sorted(set(rxcases.COVER.values()))] + ["session:1200@48000:inverted"]


def session_preset(name):
    """(mode, rate, inverted) of a SESSIONS name"""
    mode, rest = name.split(":")[1].split("@")
    return mode, int(rest), name.endswith(":inverted")


def session_streams(name):
    """(mode, audio, rate, rx_args, inverted) of every stream of a carrier-session case"""
    import rxfam
    mode, rate, inv = session_preset(name)
    c = rxcases.session_case(dict(rxfam.FAMILIES["auto"], inverted=bool(inv)), (mode, rate))
    rx_args = [mode, "--samplerate", str(rate), "-a"] + (["--inverted"] if inv else [])
    return [(orc.Mode(mode, sample_rate=rate, inverted=bool(inv)), x, rate, rx_args, bool(inv)) for x in c.rows]


def inputs(seed, classes=CLASSES):
    return [random_case(seed, classes)] if isinstance(seed, int) else session_streams(seed)


@pytest.mark.ref
@pytest.mark.parametrize("seed", list(range(60)) + SESSIONS)
def test_auto_oracle_matches_the_reference_cli(seed, tmp_path):
    """LITERAL prints what the CLI prints, on the random cases and the carrier-session streams"""
    for m, audio, rate, rx_args, inverted in inputs(seed):
        wav = str(tmp_path / "x.wav")
        write_wav_float(wav, audio, rate)
        r = subprocess.run([orc.REF_CLI, "--rx", "--file", wav] + rx_args, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, check=True)
        res = autoorc.rx_run(m, audio, literal=True, inverted=inverted)
        assert orc.ref_decode(m, res["frames"]) == r.stdout, (seed, rx_args, r.stdout[:60])
        want = [ln.strip() for ln in r.stderr.decode().splitlines() if ln.startswith("### ")]
        compare_lines(autoorc.stat_lines(m, res), want, (seed, rx_args))


@pytest.mark.parametrize("seed", list(range(60)) + [s for s in SESSIONS if not ring_limited(
    orc.Mode(session_preset(s)[0], sample_rate=session_preset(s)[1]))])
def test_flat_auto_oracle_matches_literal(seed):
    for m, audio, rate, rx_args, inverted in inputs(seed, CLASSES[:2]):
        assert not ring_limited(m)
        lit = autoorc.rx_run(m, audio, literal=True, inverted=inverted)
        flat = autoorc.rx_run(m, audio, literal=False, inverted=inverted)
        assert flat["frames"] == lit["frames"], (seed, rx_args)
        assert flat["reports"] == lit["reports"] and flat["frame_band"] == lit["frame_band"], (seed, rx_args)
        assert flat["report_band"] == lit["report_band"], (seed, rx_args)


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


def test_the_auto_replay_reproduces_the_oracle_exactly():
    """tie_screen.replay over the auto oracle's search calls (autoorc.calls) restates its frames and reports
    bit for bit, on every random case (the carrier-session streams: test_every_case_reaches_every_loop_event)."""
    import tie_screen
    for seed in range(60):
        m, audio, rate, rx_args, inverted = random_case(seed)
        want = autoorc.rx_run(m, audio, inverted=inverted)
        frames, reports, ties = tie_screen.replay(m, autoorc.calls(m, audio, inverted))
        assert frames == [f[:5] for f in want["frames"]] and reports == want["reports"] and not ties, rx_args


def _auto_fade(r):
    """1200 baud under auto-carrier: a burst at 0.8, then with no gap one at 0.8 r, sigma = 1e-4; the scan takes
    bands 5 and 9 (test_gpu_auto_carrier's test_a_stream_on_the_configured_tones_gives_the_fixed_tone_records),
    so up to a drop the loop is the fixed-tone loop on 1000 / 1800 Hz"""
    m = orc.Mode("1200")
    rng = np.random.default_rng(5)
    a = orc.tx_words(m, rng.integers(0, 256, 6).astype(np.uint32), 0.8, 4096, True)
    b = orc.tx_words(m, rng.integers(0, 256, 6).astype(np.uint32), 1.0, 4096, True)
    bg = (1e-4 * rng.standard_normal(a.size + b.size)).astype(np.float32)
    return m, orc.Mode("1200", mark=1000.0, space=1800.0), a.size, \
        (np.concatenate([a, np.float32(0.8 * r) * b]) + bg).astype(np.float32)


def _auto_squelch_ratio(r):
    """amplitude / (0.25 track_amplitude) - 1 at the first search that reaches into the fade"""
    m, fixed, at, x = _auto_fade(r)
    res = orc.rx_run(fixed, x, literal=False, want_calls=True)
    j = next(i for i, cl in enumerate(res["calls"]) if cl[8] > 0 and cl[10] + cl[9] >= at)
    track = np.float32(0)
    for f in res["frames"]:
        if f[5] + f[3] >= res["calls"][j][10]:
            break
        track = np.float32((track + f[2]) / np.float32(2))
    return float(res["calls"][j][8]) / float(np.float32(0.25) * track) - 1


@pytest.mark.parametrize("eps", [-1e-5, -1e-6, -1e-7, 1e-7, 1e-6, 1e-5])
def test_the_auto_screen_flags_a_squelch_tie(eps):
    """A fade under auto-carrier tuned (secant on its amplitude ratio) so that the squelch `amplitude <
    track_amplitude * 0.25` sits within eps of a tie: autoorc.screen flags it (the replay's margin, decided
    the other way by autoorc.flipped); a fade clear of the tie stays robust."""
    r0, r1 = 0.25, 0.26
    g0, g1 = _auto_squelch_ratio(r0) - eps, _auto_squelch_ratio(r1) - eps
    for _ in range(30):
        if abs(g1) < abs(eps) / 2 + 6e-8 or g1 == g0:
            break
        r0, r1, g0 = r1, r1 - g1 * (r1 - r0) / (g1 - g0), g1
        g1 = _auto_squelch_ratio(r1) - eps
    assert abs(g1) < abs(eps) / 2 + 6e-8, (eps, r1, g1)
    m, fixed, at, x = _auto_fade(r1)
    auto = autoorc.rx_run(m, x)
    k = sum(1 for f in auto["frames"] if f[5] + f[3] < at)
    assert k >= 5 and auto["frames"][:k] == orc.rx_run(fixed, x, literal=False)["frames"][:k]
    assert set(auto["frame_band"]) == {5}
    _, robust = autoorc.screen(m, x)
    assert not robust, (eps, r1)
    _, robust = autoorc.screen(m, _auto_fade(0.3)[3])
    assert robust
