"""The reference's own test vectors (tests/*.test under /root/reference), restated
as data: for each run of tests/self-test, the text file, the tx/rx command
lines, and the equivalent oracle Mode / tx options.  tests/golden/make_golden.py
runs the unmodified reference CLI on these and commits what it observed;
the parity tests replay them.

Each case: name, text (file under reference tests/ or literal bytes), tx args,
rx args, mode kwargs for tx and rx (they differ in 21-rate-slop), tx options.
"""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)


def _case(name, text, tx, rx=None, mode="1200", mkw=None, rx_mode=None, rx_mkw=None,
          amplitude=1.0, lut=4096, float_samples=False, rxnoise=0.0, rx_one=False,
          perfect=False, tx_ascii=False, bins=False, audio=False, ring_limited=False):
    """ring_limited: the reference stops early on this input because of how it sizes and refills its
    sample ring (DESIGN.md 5, item 2); only the oracle's LITERAL mode reproduces that, the batched
    (flat) semantic decodes the whole stream and the reference's output is a prefix of it."""
    return dict(ring_limited=ring_limited, name=name, text=text, tx=tx, rx=rx if rx is not None else tx, mode=mode,
                mkw=mkw or {}, rx_mode=rx_mode or mode, rx_mkw=rx_mkw if rx_mkw is not None else (mkw or {}),
                amplitude=amplitude, lut=lut, float_samples=float_samples, rxnoise=rxnoise,
                rx_one=rx_one, perfect=perfect, tx_ascii=tx_ascii, bins=bins, audio=audio)


ASCII = "testdata-ascii.txt"
PERFECT = dict(sample_rate=24000, mark=1200, space=2400)
PERFECT_ARGS = ["1200", "--samplerate", "24000", "-M", "1200", "-S", "2400"]

CASES = [
    _case("01-self-test-1200", ASCII, ["1200"], bins=True),
    _case("02-self-test-300", ASCII, ["300"], mode="300", bins=True),
    _case("03-self-test-rtty", "testdata-baudot.txt", ["rtty"], mode="rtty", bins=True),
    _case("04-self-test-0.5", b"KAMAL\n", ["0.5"], mode="0.5"),
    _case("05-self-test-12000", ASCII, ["12000"], mode="12000", bins=True),
    _case("06-self-test-float-samples", ASCII, ["--float-samples", "12000"], mode="12000",
          float_samples=True),
    _case("07-self-test-no-lut", ASCII, ["1200", "--lut=0"], lut=0),
    _case("08-self-test-lut16", ASCII, ["1200", "--lut=16"], lut=16),
    _case("09-self-test-lut16-float", ASCII, ["1200", "--lut=16", "--float-samples"], lut=16,
          float_samples=True),
    _case("10-verify-perfect", ASCII, PERFECT_ARGS, mkw=PERFECT, perfect=True, bins=True),
    _case("11-verify-perfect-nolut", ASCII, PERFECT_ARGS + ["--lut=0"], mkw=PERFECT, lut=0, perfect=True),
    _case("12-verify-perfect-lut16", ASCII, PERFECT_ARGS + ["--lut=16"], mkw=PERFECT, lut=16, perfect=True),
    _case("13-verify-perfect-nolut-float", ASCII, PERFECT_ARGS + ["--lut=0", "--float-samples"],
          mkw=PERFECT, lut=0, float_samples=True, perfect=True),
    _case("14-verify-perfect-lut16-float", ASCII, PERFECT_ARGS + ["--lut=16", "--float-samples"],
          mkw=PERFECT, lut=16, float_samples=True, perfect=True),
    _case("15-verify-perfect-float", ASCII, PERFECT_ARGS + ["--float-samples"], mkw=PERFECT,
          float_samples=True, perfect=True),
]
for _adj in (-8, -1, 0, 1, 8):
    CASES.append(_case("21-rate-slop-%d" % (300 + _adj), ASCII, [str(300 + _adj)], rx=["300"],
                       mode=str(300 + _adj), rx_mode="300", bins=(_adj == 8)))
for _flt in (False, True):
    for _a in ("3.50", "1.00", "0.30", "0.01", "E"):
        amp = FLT_EPSILON if _a == "E" else float(np.float32(float(_a)))
        args = ["--volume", _a, "1200"] + (["--float"] if _flt else [])
        CASES.append(_case("%s-%s" % ("31-amplitude-float" if _flt else "30-amplitude", _a), ASCII,
                           args, rx=["1200"] + (["--float"] if _flt else []), amplitude=amp,
                           float_samples=_flt))
for _pure in (False, True):
    for _n in ("0.00", "0.05", "0.10", "0.50"):
        flags = ["1200"] + (["-M", "1200", "-S", "2400"] if _pure else [])
        mkw = dict(mark=1200, space=2400) if _pure else {}
        CASES.append(_case("%s-%s" % ("41-noise-purefreqs" if _pure else "40-noise", _n), ASCII,
                           flags + ["--volume", "0.5"], rx=flags + ["--Xrxnoise", _n, "--rx-one"],
                           mkw=mkw, amplitude=0.5, rxnoise=float(np.float32(float(_n))), rx_one=True,
                           bins=(_n == "0.10" and not _pure)))
CASES += [
    _case("60-multibyte", "testdata-multibyte.txt", ["1200"]),
    _case("70-callerid-mdmf", "testdata-callerid-mdmf.bytes", ["1200", "--ascii"], rx=["callerid"],
          rx_mode="callerid", tx_ascii=True),
    _case("71-callerid-sdmf", "testdata-callerid-sdmf.bytes", ["1200", "--ascii"], rx=["callerid"],
          rx_mode="callerid", tx_ascii=True),
    _case("80-SAME", ASCII, ["SAME"], mode="same", bins=True),
    _case("81-ascii7", ASCII, ["-7", "1200"], mkw=dict(n_data_bits=7)),
    _case("81-tdd", "testdata-baudot.txt", ["tdd"], mode="tdd"),
]

# small extra vectors (short payloads) whose AUDIO is committed too, so that the
# kernels can be checked against the real reference without regenerating audio
SMALL = [
    _case("small-1200", b"Hello, B200!\n", ["1200"], audio=True, bins=True),
    _case("small-300", b"Bell103 ok\n", ["300"], mode="300", audio=True, bins=True),
    _case("small-rtty", b"RYRY CQ DE B200\n", ["rtty", "--samplerate", "8000"], mode="rtty",
          mkw=dict(sample_rate=8000), audio=True, bins=True),
    _case("small-same", b"ZCZC-WXR-TOR\n", ["same"], mode="same", audio=True, bins=True),
    _case("small-1200-float-noise", b"noisy frame test\n", ["1200", "--float-samples", "--volume", "0.5"],
          rx=["1200", "--Xrxnoise", "0.10"], amplitude=0.5, float_samples=True, rxnoise=float(np.float32(0.10)),
          audio=True, bins=True),
]

ALL = CASES + SMALL

# Option combinations none of the reference's own tests use (framing, bit order, tone
# inversion, sync byte, odd sample rates, thresholds): short payloads, audio committed.
# Minted like the others from the unmodified reference CLI; on the CPU and the GPU lists.
_OPT_TEXT = b"Options: B200 {~}\n"
OPTIONS = [
    _case("opt-2start-2stop", _OPT_TEXT, ["1200", "--startbits", "2", "--stopbits", "2.0"],
          mkw=dict(startbits=2, stopbits=2.0), audio=True),
    _case("opt-stop-1.5", _OPT_TEXT, ["1200", "--stopbits", "1.5"], mkw=dict(stopbits=1.5), audio=True),
    _case("opt-msb-first", _OPT_TEXT, ["1200", "--msb-first"], mkw=dict(msb_first=True), audio=True),
    _case("opt-7bit-msb-first", _OPT_TEXT, ["-7", "1200", "--msb-first"],
          mkw=dict(n_data_bits=7, msb_first=True), audio=True),
    _case("opt-invert-start-stop", _OPT_TEXT, ["1200", "--invert-start-stop"],
          mkw=dict(invert_start_stop=True), audio=True),
    _case("opt-inverted", _OPT_TEXT, ["1200", "--inverted"], mkw=dict(inverted=True), audio=True),
    _case("opt-sync-byte-600", _OPT_TEXT, ["600", "--sync-byte", "0x7E"], mode="600",
          mkw=dict(sync_byte=0x7E), audio=True),
    _case("opt-2400-44100", _OPT_TEXT, ["2400", "--samplerate", "44100"], mode="2400",
          mkw=dict(sample_rate=44100), audio=True),
    _case("opt-600-22050", _OPT_TEXT, ["600", "--samplerate", "22050"], mode="600",
          mkw=dict(sample_rate=22050), audio=True),
    _case("opt-300-bandwidth-25", _OPT_TEXT, ["300", "-b", "25"], mode="300", mkw=dict(bandwidth=25.0),
          audio=True),
    _case("opt-110-baudot", b"RYRY 5-BIT AT 110\n", ["110", "-5"], mode="110", mkw=dict(baudot=True),
          audio=True),
    _case("opt-thresholds", _OPT_TEXT, ["1200"], rx=["1200", "-c", "3.0", "-l", "4.0"],
          rx_mkw=dict(confidence=3.0, limit=4.0), audio=True),
    _case("opt-binary-output", _OPT_TEXT, ["1200"], rx=["1200", "--binary-output"], audio=True),
    _case("opt-rtty-binary-output", b"RYRY\n", ["rtty", "--samplerate", "8000"],
          rx=["rtty", "--samplerate", "8000", "--binary-output"], mode="rtty", mkw=dict(sample_rate=8000),
          audio=True),
    _case("opt-mark-space", _OPT_TEXT, ["1200", "-M", "1500", "-S", "2100"], mkw=dict(mark=1500, space=2100),
          audio=True),
]



def decoder_of(case, rx_mode):
    """The databits decoder the reference's main() ends up with for this rx invocation
    (src/minimodem.c:552-892): --binary-output overrides the mode's."""
    return "binary" if "--binary-output" in case["rx"] else rx_mode.decoder


# A second batch of option runs: they pin the oracle on the CPU and the emulated kernels
# (tests/emu_fuzz.py); not on the GPU list (that one is long enough).
MORE = [
    _case("more-v21", _OPT_TEXT, ["V.21"], mode="V.21", audio=True),
    _case("more-6bit-3start", _OPT_TEXT, ["1200", "--startbits", "3", "--stopbits", "1.0"],
          mkw=dict(n_data_bits=8, startbits=3, stopbits=1.0), audio=True),
    _case("more-12000-96000", _OPT_TEXT, ["12000", "--samplerate", "96000"], mode="12000",
          mkw=dict(sample_rate=96000), audio=True),
    _case("more-1200-11025", _OPT_TEXT, ["1200", "--samplerate", "11025"], mkw=dict(sample_rate=11025), audio=True),
    _case("more-1200-bw100", _OPT_TEXT, ["1200", "-b", "100"], mkw=dict(bandwidth=100.0), audio=True),
    _case("more-tdd-inverted", b"TDD INVERTED 123\n", ["tdd", "--inverted"], mode="tdd", mkw=dict(inverted=True),
          audio=True),
    _case("more-same-msb", b"ZCZC-MSB-FIRST\n", ["same", "--msb-first"], mode="same", mkw=dict(msb_first=True),
          audio=True),
    # 8 data + 1 start + 3 stop bits: the advance after a frame exceeds the half-filled sample ring and
    # the reference's loop ends after the first frame (src/minimodem.c:1150-1152)
    _case("more-150-stop3", _OPT_TEXT, ["150", "--stopbits", "3.0", "--samplerate", "16000"], mode="150",
          mkw=dict(sample_rate=16000, stopbits=3.0), audio=True, ring_limited=True),
    _case("more-volume-E", _OPT_TEXT, ["1200", "--volume", "E"], amplitude=FLT_EPSILON, audio=True),
    _case("more-quiet-noise", _OPT_TEXT, ["1200", "--float-samples", "--volume", "0.05"],
          rx=["1200", "--Xrxnoise", "0.02"], amplitude=0.05, float_samples=True, rxnoise=float(np.float32(0.02)),
          audio=True),
]

EVERY = ALL + OPTIONS

# Runs that only the whole CLI can make (the oracle's rx loop has no --auto-carrier): they pin the
# drop-in binary (the reference's main() on this library), tests/test_gpu_parity.py
# test_reference_cli_on_this_library and tests/test_dropin_cli.py.
CLI_ONLY = [
    _case("cli-auto-carrier", b"auto carrier probe 0123456789\n", ["1200", "-M", "1600", "-S", "2600"],
          rx=["1200", "--auto-carrier"], audio=True),
    _case("cli-auto-carrier-rtty", b"RYRY AUTO\n", ["rtty", "--samplerate", "8000", "-M", "1000", "-S", "830"],
          rx=["rtty", "--samplerate", "8000", "--auto-carrier"], mode="rtty", mkw=dict(sample_rate=8000), audio=True),
]

BY_NAME = {c["name"]: c for c in EVERY + CLI_ONLY + MORE}
