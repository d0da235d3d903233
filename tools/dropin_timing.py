"""tools/dropin_timing.py (run on the GPU box): wall time of the unmodified reference CLI on its own src/fsk.c
(oracle/_ref/minimodem_ref) against the same main() linked to libfsk_b200.so (oracle/_ref/minimodem_dropin) on
the tests/01-self-test-1200 audio (200 160 samples).  The drop-in serves every fsk_find_frame call with two
synchronous copies and a one-stream launch: it is a correctness shim, and this is what it costs."""
import os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_util as gu, refcases, orc
from clicases import write_wav
case = refcases.BY_NAME["01-self-test-1200"]
g = gu.load(case["name"]); a = gu.audio(case, g)
d = tempfile.mkdtemp(); wav = os.path.join(d, "x.wav")
write_wav(wav, a, int(g["audio_len"][1]), bool(g["audio_len"][2]))
out = {}
for name in ("minimodem_ref", "minimodem_dropin"):
    exe = os.path.join(os.path.dirname(orc.LIBREF), name)
    ts = []
    for i in range(4):
        t = time.perf_counter()
        r = subprocess.run([exe, "--rx", "--file", wav] + list(case["rx"]), stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        ts.append(time.perf_counter() - t)
        assert r.returncode == 0 and r.stdout == bytes(g["stdout"]), (name, r.stderr[-300:])
    out[name] = min(ts[1:])
print("samples %d: reference CLI %.1f ms, drop-in CLI on libfsk_b200.so %.1f ms (process start and CUDA context included)" % (
    a.size, out["minimodem_ref"] * 1e3, out["minimodem_dropin"] * 1e3))
