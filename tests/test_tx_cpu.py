"""The transmitter's CPU side: the product's encoders (host build of fsk_b200_decode_core.h) against the
reference's databits_encode_ascii8 / baudot_encode, the oracle's restatement of fsk_transmit_stdin over
text against the audio the reference CLI wrote, the row bound of fsk_b200_tx_max_samples, the C ABI's
struct layout, and the GPU tests of the transmitter on the host emulation of its kernel."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import golden_util as gu
import orc
import refcases
import txorc
from gpudev import run_emulated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = refcases.EVERY + refcases.MORE


def tx_kind(case, tx):
    return "ascii8" if case["tx_ascii"] or tx.decoder != "baudot" else "baudot"


# ---- encoders ------------------------------------------------------------------------------------
@pytest.mark.ref
@pytest.mark.parametrize("kind", ["ascii8", "baudot"])
@pytest.mark.parametrize("charset", [0, 1, 2])
def test_encoder_every_byte_from_each_charset(kind, charset):
    """All 256 byte values, each from a fresh encoder in charset 0 (unknown), 1 (LTRS) or 2 (FIGS)."""
    texts = [bytes([b]) for b in range(256)]
    want = txorc.ref_encode_fresh(kind, texts, charset)
    for b, w in zip(range(256), want):
        st = txorc.Encoder(txorc.KINDS[kind], charset)
        got = txorc.encode(kind, bytes([b]), st)
        assert np.array_equal(got, w), (kind, charset, hex(b), got, w)


@pytest.mark.ref
@pytest.mark.parametrize("kind", ["ascii8", "baudot"])
def test_encoder_random_strings_carry_the_charset(kind):
    rng = np.random.default_rng(17)
    texts = []
    for i in range(2000):
        n = int(rng.integers(0, 40))
        # printable text with figures and shift-provoking characters, and a share of arbitrary bytes
        pool = rng.integers(0, 256, n) if i % 4 == 0 else rng.integers(32, 127, n)
        texts.append(bytes(int(x) for x in pool))
    want = txorc.ref_encode_fresh(kind, texts)
    for t, w in zip(texts, want):
        assert np.array_equal(txorc.encode(kind, t), w), (kind, t)


def test_encoder_matches_the_golden_words():
    """The words the reference's encoder produced for each golden vector (stored with it)."""
    for case in CASES:
        g = gu.load(case["name"])
        tx, _ = gu.modes(case)
        assert np.array_equal(txorc.encode(tx_kind(case, tx), bytes(g["text"])), g["words"]), case["name"]


# ---- the oracle's transmitter over text -------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_tx_events_reproduce_the_reference_audio(case):
    g = gu.load(case["name"])
    tx, _ = gu.modes(case)
    a = txorc.tx_events(tx, list(bytes(g["text"])), tx_kind(case, tx), case["amplitude"], case["lut"],
                        case["float_samples"])
    assert a.size == int(g["audio_len"][0])
    assert gu.sha(a) == bytes(g["audio_sha256"])


def test_tx_events_idle_semantics():
    """An idle timeout before the first byte and between bytes: the idle tone, then the preamble again
    but no leader (src/minimodem.c:207-237); idle at the end keeps the trailer."""
    m = orc.Mode("same")
    text = list(b"AB")
    plain = txorc.tx_events(m, text, "ascii8")
    bit = int(np.float32(np.float32(48000) / m.data_rate) + np.float32(0.5))
    frame = 8 * bit
    idle = 48000 // 25
    with_idle = txorc.tx_events(m, [text[0], txorc.IDLE, text[1], txorc.IDLE], "ascii8")
    # leader 0 (no start bits); preamble 16 frames + A; idle; preamble again + B; idle; trailer 2 bits
    assert with_idle.size == (16 + 1) * frame + idle + (16 + 1) * frame + idle + 2 * bit
    assert plain.size == (16 + 2) * frame + 2 * bit


# ---- the row bound --------------------------------------------------------------------------------------
def _emu_lib():
    emu = os.path.join(ROOT, "tests", "emu")
    subprocess.check_call(["make", "-s", "-C", emu])
    L = C.CDLL(os.path.join(emu, "libfsk_b200_emu.so"))
    import minimodem_b200.api as api
    L.fsk_b200_rx_config_for_mode.argtypes = [C.c_char_p, C.c_float, C.c_void_p, C.c_void_p]
    L.fsk_b200_tx_config_from_rx.argtypes = [C.c_void_p, C.c_void_p]
    L.fsk_b200_tx_engine_new.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.fsk_b200_tx_engine_new.restype = C.c_void_p
    L.fsk_b200_tx_engine_destroy.argtypes = [C.c_void_p]
    L.fsk_b200_tx_max_samples.argtypes = [C.c_void_p, C.c_uint32, C.c_uint]
    L.fsk_b200_tx_max_samples.restype = C.c_uint64
    L.fsk_b200_encoder_for_mode.argtypes = [C.c_char_p, C.c_uint]
    return L, api


@pytest.mark.parametrize("mode,kw", [("1200", {}), ("rtty", dict(sample_rate=8000)), ("tdd", {}), ("same", {}),
                                     ("300", dict(startbits=2, stopbits=3.0))])
def test_max_samples_bounds_every_row(mode, kw):
    """fsk_b200_tx_max_samples (host code, reached through the emulation build, which needs no GPU)
    against the oracle's length of random texts: a bound, exact for ascii8."""
    L, api = _emu_lib()
    ov = api.RxConfig()
    ov.nstartbits, ov.nstopbits = kw.get("startbits", -1), kw.get("stopbits", -1.0)
    rx = api.RxConfig()
    assert L.fsk_b200_rx_config_for_mode(mode.encode(), kw.get("sample_rate", 48000), C.byref(ov), C.byref(rx)) == 0
    tc = api.TxConfig()
    assert L.fsk_b200_tx_config_from_rx(C.byref(rx), C.byref(tc)) == 0
    kind = L.fsk_b200_encoder_for_mode(mode.encode(), rx.n_data_bits)
    te = L.fsk_b200_tx_engine_new(C.byref(tc), C.byref(api.TxSignal(1.0, 4096, 1)), kind)
    assert te
    m = orc.Mode(mode, **kw)
    rng = np.random.default_rng(5)
    name = "baudot" if kind == 1 else "ascii8"
    for _ in range(60):
        n = int(rng.integers(1, 50))
        text = list(rng.integers(32, 127, n))
        for flags, events in ((2, text), (3, text), (3, [])):
            got = txorc.tx_events(m, events, name)
            bound = int(L.fsk_b200_tx_max_samples(te, len(events), flags))
            assert got.size <= bound
            if name == "ascii8" and events and flags == 2:
                assert got.size == bound, (mode, n, flags, got.size, bound)
    L.fsk_b200_tx_engine_destroy(te)


# ---- ABI layout -----------------------------------------------------------------------------------------
def test_struct_layout_matches_the_header(tmp_path):
    import minimodem_b200.api as api
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stdio.h>
#include <stddef.h>
#include "fsk_b200.h"
#define F(T, f) printf("%s.%s %zu\\n", #T, #f, offsetof(T, f));
int main(void) {
    printf("fsk_b200_tx_signal %zu\\n", sizeof(fsk_b200_tx_signal));
    printf("fsk_b200_tx_state %zu\\n", sizeof(fsk_b200_tx_state));
    printf("fsk_b200_tx_config %zu\\n", sizeof(fsk_b200_tx_config));
    F(fsk_b200_tx_signal, amplitude) F(fsk_b200_tx_signal, sin_table_len) F(fsk_b200_tx_signal, float_samples)
    F(fsk_b200_tx_state, cphase) F(fsk_b200_tx_state, baudot_charset) F(fsk_b200_tx_state, transmitting)
    F(fsk_b200_tx_state, reserved)
    return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    lines = dict(ln.rsplit(" ", 1) for ln in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(lines["fsk_b200_tx_state"]) == api.TX_STATE_BYTES == C.sizeof(api.TxState) == 16
    assert int(lines["fsk_b200_tx_signal"]) == C.sizeof(api.TxSignal)
    assert int(lines["fsk_b200_tx_config"]) == C.sizeof(api.TxConfig)
    for cls, name in ((api.TxSignal, "fsk_b200_tx_signal"), (api.TxState, "fsk_b200_tx_state")):
        for f, _ in cls._fields_:
            assert int(lines["%s.%s" % (name, f)]) == getattr(cls, f).offset, (name, f)


# ---- the GPU tests on the emulated kernel --------------------------------------------------------------------
def test_tx_gpu_tests_on_the_emulated_kernel():
    """tests/test_tx_gpu.py (marker gpu) against the emulation build of the same kernel source, at the
    reduced sizes that file picks under the emulator."""
    tail = run_emulated("", "late", 1500, module="test_tx_gpu.py")
    assert " passed" in tail and "failed" not in tail
