"""TEST INFRASTRUCTURE for the transmitter: ctypes bindings of oracle/tx_oracle.c -- orc_tx_events (the
reference's fsk_transmit_stdin over bytes and idle timeouts, on fsk_oracle.c's tone generator) and
orc_encode_byte (the host build of the product's encoders, minimodem_b200/csrc/fsk_b200_decode_core.h)
-- and the reference's own encoders run from a fresh process state.  The library is compiled on first
use into a temporary directory, so the tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

import orc

IDLE = -1                       # ORC_TX_IDLE: one select() timeout of the reference's input loop
KINDS = {"ascii8": 0, "baudot": 1}


class Encoder(C.Structure):
    """orc_encoder of oracle/tx_oracle.c: the kind and the charset carried between calls."""
    _fields_ = [("kind", C.c_int), ("charset", C.c_uint32)]


SOURCES = [os.path.join(orc.ORACLE_DIR, f) for f in ("tx_oracle.c", "fsk_oracle.c", "fsk_oracle.h")] + [
    os.path.join(orc.ROOT, "minimodem_b200", "csrc", "fsk_b200_decode_core.h"), os.path.join(orc.ROOT, "include", "fsk_b200.h")]
_lib = None


def build():
    """Compile oracle/tx_oracle.c (gcc, as oracle/Makefile compiles the oracle) into a temporary
    directory, named after a hash of its sources."""
    h = hashlib.sha256()
    for f in SOURCES:
        with open(f, "rb") as fh:
            h.update(fh.read())
    out = os.path.join(tempfile.gettempdir(), "fsk_tx_oracle_%d_%s.so" % (os.getuid(), h.hexdigest()[:16]))
    if not os.path.exists(out):
        tmp = out + ".%d" % os.getpid()
        subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-Wno-unused-function", "-fPIC", "-ffp-contract=off",
                               "-I", os.path.join(orc.ROOT, "include"), "-shared", "-o", tmp,
                               os.path.join(orc.ORACLE_DIR, "tx_oracle.c"), "-lm", "-lpthread"])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_tx_events.argtypes = [C.POINTER(orc.OrcTxConfig), C.POINTER(C.c_int), C.c_size_t, C.c_void_p,
                                    C.c_void_p, C.POINTER(C.c_float), C.c_size_t]
        L.orc_tx_events.restype = C.c_size_t
        L.orc_encode_byte.argtypes = [C.c_void_p, C.c_ubyte, C.POINTER(C.c_uint)]
        L.orc_encode_byte.restype = C.c_uint
        _lib = L
    return _lib


def encode(kind, data, state=None):
    """bytes -> data words through the product's encoder (host build); `state` (Encoder) carries the
    Baudot charset from call to call."""
    st = state if state is not None else Encoder(KINDS.get(kind, kind), 0)
    w = (C.c_uint * 2)()
    out = []
    for b in bytes(data):
        n = lib().orc_encode_byte(C.addressof(st), b, w)
        out.extend(w[i] for i in range(n))
    return np.array(out, np.uint32)


def bound(mode, events):
    """Samples orc_tx_events can produce at most for these events."""
    bit = int(np.float32(np.float32(mode.sample_rate) / mode.data_rate) + np.float32(0.5))
    frame = (mode.n_data_bits + 3 + 3) * bit
    nbytes = sum(1 for e in events if e != IDLE)
    nidle = len(events) - nbytes
    return (nbytes * (2 + 16 + 2) + 8) * frame + nidle * (mode.sample_rate // 25 + 1)


def tx_events(mode, events, kind, amplitude=1.0, lut=4096, float_samples=False, state=None):
    """The reference transmitter over `events` (byte values and IDLE), then end of input: float32
    samples (int16 output scaled by 1/32768, as the reference's rx reads it back)."""
    cfg = mode.tx_config(amplitude, lut, float_samples)
    ev = np.ascontiguousarray(events, np.int32)
    cap = bound(mode, events)
    out = np.zeros(cap, np.float32)
    st = state if state is not None else Encoder(KINDS.get(kind, kind), 0)
    fn = C.cast(lib().orc_encode_byte, C.c_void_p)
    n = lib().orc_tx_events(C.byref(cfg), ev.ctypes.data_as(C.POINTER(C.c_int)), ev.size, fn,
                            C.addressof(st), out.ctypes.data_as(C.POINTER(C.c_float)), cap)
    assert n <= cap, (n, cap)
    return out[:n]


_FRESH = r"""
import ctypes as C, os, sys
L = C.CDLL(sys.argv[1])
for name in ("databits_encode_ascii8", "baudot_encode"):
    getattr(L, name).argtypes = [C.POINTER(C.c_uint), C.c_char]
L.baudot_reset.argtypes = []
enc = L.baudot_encode if sys.argv[2] == "baudot" else L.databits_encode_ascii8
start = int(sys.argv[3])
out = sys.stdout
for line in sys.stdin:
    data = bytes.fromhex(line.strip())
    r, w = os.pipe()
    pid = os.fork()
    if pid == 0:                                  # a fresh copy of the process: baudot_charset as at start
        os.close(r)
        if start:
            L.baudot_reset()                      # charset 1 (LTRS)
        buf = (C.c_uint * 2)()
        if start == 2:
            L.baudot_encode(buf, C.c_char(b"1"))  # a figure: charset 2 (FIGS)
        words = []
        for ch in data:
            n = enc(buf, C.c_char(bytes([ch])))
            words.extend(buf[i] for i in range(n))
        os.write(w, (" ".join(str(x) for x in words) + "\n").encode())
        os._exit(0)
    os.close(w)
    got = b""
    while True:
        b = os.read(r, 65536)
        if not b:
            break
        got += b
    os.close(r)
    os.waitpid(pid, 0)
    out.write(got.decode())
out.flush()
"""


def ref_encode_fresh(kind, texts, charset=0):
    """The reference's own encoder (oracle/_ref/libfsk_ref.so) on each text, every one from a fresh
    process state with baudot_charset = `charset` (0 as at program start; 1 and 2 reached with
    baudot_reset and a figure).  The reference keeps the charset in a static variable, so each text
    runs in a forked child.  Returns a list of uint32 word arrays."""
    inp = "".join(bytes(t).hex() + "\n" for t in texts)
    r = subprocess.run([sys.executable, "-c", _FRESH, orc.LIBREF, kind, str(charset)], input=inp.encode(),
                       stdout=subprocess.PIPE, check=True, env=dict(os.environ, PYTHONPATH=""))
    lines = r.stdout.decode().split("\n")[:len(texts)]
    return [np.array([int(x) for x in ln.split()], np.uint32) for ln in lines]
