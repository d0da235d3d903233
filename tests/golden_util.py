"""Helpers shared by the parity tests: load tests/golden/*.npz, regenerate the
audio of a reference test vector with the oracle's TX restatement."""
import hashlib
import os

import numpy as np

import orc
import refcases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def modes(case):
    tx = orc.Mode(case["mode"], **case["mkw"])
    rx = orc.Mode(case["rx_mode"], **case["rx_mkw"])
    return tx, rx


def audio(case, g=None):
    """The float32 samples the reference rx saw for this case."""
    g = g if g is not None else load(case["name"])
    if "audio_f32" in g.files:
        return g["audio_f32"]
    if "audio_s16" in g.files:
        return g["audio_s16"].astype(np.float32) * np.float32(1.0 / 32768.0)
    tx, _ = modes(case)
    return orc.tx_words(tx, g["words"], case["amplitude"], case["lut"], case["float_samples"])


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).digest()


def stat_lines(g):
    err = bytes(g["stderr"]).decode(errors="replace")
    return [ln.strip() for ln in err.splitlines() if ln.startswith("### NOCARRIER")]


def close(a, b, rel=1e-4, cond=0.0):
    """confidence/amplitude comparison: inf and nan are classes that must match.

    `cond` widens the tolerance for ill-conditioned confidences: confidence =
    snr*(1-divergence) with snr = sum(sig)/sum(noise) (src/fsk.c:292,336), so a
    perturbation dn of the off-tone magnitudes (relative to the signal) moves it
    by a relative dn*confidence.  Two correct float FFTs already differ by
    dn ~ 1e-7..1e-6, hence rel + cond*|confidence|."""
    a, b = float(a), float(b)
    if np.isinf(a) or np.isinf(b) or np.isnan(a) or np.isnan(b):
        return (np.isinf(a) and np.isinf(b) and (a > 0) == (b > 0)) or (np.isnan(a) and np.isnan(b))
    m = max(abs(a), abs(b))
    return abs(a - b) <= (rel + cond * m) * m + 1e-30


CONF_COND = 5e-7     # see close(): noise-bin error budget relative to the signal
