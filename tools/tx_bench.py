#!/usr/bin/env python
"""Transmitter throughput on the GPU: kernel time of fsk_b200_tx_text_batch (text -> samples) and of
fsk_b200_tx_batch (pre-encoded words -> samples), by CUDA events over warmed, repeated launches.

    python tools/tx_bench.py                                  # this tree's library
    python tools/tx_bench.py --compare OTHER/libfsk_b200.so   # plus OTHER's fsk_b200_tx_batch, alternating

Workloads: 65 536 Bell202 streams of 480 characters (about 192 000 samples each, the rx headline's
stream length), float32 and int16, --lut=4096; RTTY at 8 kHz; and fsk_b200_tx_batch on the Bell202
words.  The kernel writes 4 (float) or 2 (int16) bytes of HBM per sample and reads next to nothing,
so the bound that applies is HBM write bandwidth: the share printed is bytes written / kernel time
over the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(torch, fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return min(ms), sum(ms) / len(ms)


def rates(samples, bytes_per_sample, ms):
    return {"ms": round(ms, 3), "samples_per_s": samples / (ms * 1e-3),
            "bytes_written_per_s": samples * bytes_per_sample / (ms * 1e-3),
            "write_bound_share_of_3.35TBps": samples * bytes_per_sample / (ms * 1e-3) / HBM_BYTES_PER_S}


def words_for(torch, streams, chars, dev):
    g = torch.Generator(device="cpu").manual_seed(7)
    return torch.randint(32, 127, (streams, chars), generator=g, dtype=torch.int32).to(dev)


def child_tx_batch(a):
    """fsk_b200_tx_batch of the library at a.lib (any version of it), through its C ABI only."""
    import torch
    import minimodem_b200 as mm            # TxConfig and the sine table; the call below goes to a.lib
    L = C.CDLL(a.lib)
    L.fsk_b200_tx_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32, C.c_void_p]
    dev = torch.device("cuda:0")
    cfg = mm.TxConfig(48000.0, 1200.0, 1200.0, 2200.0, 8, 1.0, 1.0, 0, 0, 0, 0, 2, 2)
    words = words_for(torch, a.streams, a.chars, dev)
    n = (2 + 2 + 10 * a.chars) * 40
    stride = (n + 3) & ~3
    out = torch.empty((a.streams, stride), dtype=torch.float32, device=dev)
    table = torch.from_numpy(mm.sin_table(4096, 1.0)).to(dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        rc = L.fsk_b200_tx_batch(C.byref(cfg), C.c_void_p(table.data_ptr()), 4096, C.c_void_p(words.data_ptr()),
                                 a.chars, None, C.c_void_p(out.data_ptr()), a.streams, stride, n, st)
        assert rc == 0, rc
    best, mean = timed(torch, run, a.warmup, a.reps)
    rows = out[:: max(1, a.streams // 64)].cpu().numpy()
    r = rates(a.streams * n, 4, best)
    r.update(mean_ms=round(mean, 3), lib=a.lib, check=hashlib.sha256(rows.tobytes()).hexdigest()[:16])
    print(json.dumps(r))


def text_workload(torch, mm, mode, rate, streams, chars, float_samples, warmup, reps):
    dev = torch.device("cuda:0")
    te = mm.TxEngine.for_mode(mode, rate, float_samples=float_samples)
    text = words_for(torch, streams, chars, dev).to(torch.uint8)
    lens = torch.full((streams,), chars, dtype=torch.int32, device=dev)
    states = te.new_states(streams, dev)
    stride = (te.max_samples(chars, mm.TX_FINAL) + 7) & ~7
    out = torch.empty((streams, stride), dtype=torch.float32 if float_samples else torch.int16, device=dev)
    cnt = torch.empty((streams,), dtype=torch.int32, device=dev)

    def run():
        states.zero_()
        te.text_batch(text, lens, states, mm.TX_FINAL, out=out, out_len=cnt)
    best, mean = timed(torch, run, warmup, reps)
    samples = int(cnt.sum().item())
    r = rates(samples, 4 if float_samples else 2, best)
    r.update(mean_ms=round(mean, 3), streams=streams, chars=chars, samples_per_stream=samples // streams)
    del out
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--chars", type=int, default=480)
    ap.add_argument("--rtty-chars", type=int, default=160)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--compare", default="", help="another build of libfsk_b200.so: its fsk_b200_tx_batch too")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the tx_batch comparison")
    ap.add_argument("--child-tx-batch", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--lib", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child_tx_batch:
        return child_tx_batch(a)
    import torch
    import minimodem_b200 as mm
    assert torch.cuda.is_available(), "tx_bench.py needs a CUDA device"
    res = {"card": card(), "library": mm.version()}
    res["bell202_float"] = text_workload(torch, mm, "1200", 48000, a.streams, a.chars, True, a.warmup, a.reps)
    res["bell202_int16"] = text_workload(torch, mm, "1200", 48000, a.streams, a.chars, False, a.warmup, a.reps)
    res["rtty8k_int16"] = text_workload(torch, mm, "rtty", 8000, a.streams, a.rtty_chars, False, a.warmup, a.reps)
    libs = [("this", mm.LIB_PATH)] + ([("compare", os.path.abspath(a.compare))] if a.compare else [])
    runs = {k: [] for k, _ in libs}
    for _ in range(a.rounds):
        for k, path in libs:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child-tx-batch", "--lib", path,
                                "--streams", str(a.streams), "--chars", str(a.chars), "--warmup", str(a.warmup),
                                "--reps", str(a.reps)], stdout=subprocess.PIPE, text=True, check=True)
            runs[k].append(json.loads(p.stdout.strip().splitlines()[-1]))
    res["tx_batch"] = runs
    if a.compare:
        res["tx_batch_same_output"] = len({r["check"] for v in runs.values() for r in v}) == 1
    res["bound"] = "HBM writes (4 or 2 bytes per sample, nothing read per sample)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
