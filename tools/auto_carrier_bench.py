#!/usr/bin/env python
"""--auto-carrier on the GPU: kernel time of fsk_b200_rx_batch_auto against fsk_b200_rx_batch on the same
streams, by CUDA events over warmed launches (the two alternate).

    python tools/auto_carrier_bench.py [--streams 65536] [--nsamples 192000] [--reps 3]

Workloads, all Bell202 at 48 kHz with the rx headline's stream length (192 000 samples of transmission
per stream, from fsk_b200_tx_batch on the preset tones):
  preset   the transmission alone: the scan finds the carrier in its first window;
  silence  behind 1 s of zeros: the scan visits every window of the lead-in;
  noise    behind 1 s of low noise (sigma 1e-4, band magnitudes ~3e-5, below the 0.001 threshold): the same
           scan, on non-zero samples.
The scan evaluates every band of every window (120 bands x 40 samples per 40-sample window), so the last
two show what a silent or quiet lead-in costs.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--nsamples", type=int, default=192000)
    ap.add_argument("--lead", type=int, default=48000, help="lead-in samples (1 s at 48 kHz)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch
    import minimodem_b200 as mm
    assert torch.cuda.is_available(), "auto_carrier_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    cfg = mm.rx_config_for_mode("1200", 48000)
    eng = mm.RxEngine.for_mode("1200", 48000)
    eng.set_auto_carrier(0.001)
    tcfg = mm.tx_config_from(cfg)
    S, n, lead = a.streams, a.nsamples, a.lead
    bit = 40
    nwords = max(1, (n - (tcfg.leader_bits + tcfg.trailer_bits) * bit) // (10 * bit))
    gen = torch.Generator(device="cpu").manual_seed(20261016)
    words = torch.randint(32, 127, (S, nwords), generator=gen, dtype=torch.int32).to(dev)
    stride = (n + lead + 3) & ~3
    x = torch.empty((S, stride), dtype=torch.float32, device=dev)
    max_frames = eng.max_frames(n + lead)
    frames = torch.empty((S, max_frames, 5), dtype=torch.int32, device=dev)
    states = torch.zeros((S, mm.STATE_WORDS), dtype=torch.int32, device=dev)
    auto = torch.zeros((S, mm.AUTO_STATE_BYTES), dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms

    out = {"tool": "auto_carrier_bench", "card": card(), "streams": S, "nsamples": n, "lead": lead, "results": {}}
    for name in ("preset", "silence", "noise"):
        lead_in = torch.full((S,), 0 if name == "preset" else lead, dtype=torch.int32, device=dev)
        total = n + (0 if name == "preset" else lead)
        mm.tx_batch(tcfg, words, total, lead_in=lead_in, out=x, stride=stride)
        if name == "noise":
            g = torch.Generator(device=dev).manual_seed(5)
            rows = max(1, (256 << 20) // (lead * 4))
            for s0 in range(0, S, rows):
                x[s0:s0 + rows, :lead] += 1e-4 * torch.randn((min(rows, S - s0), lead), generator=g, device=dev)
        torch.cuda.synchronize()

        def fixed():
            states.zero_()
            eng.rx_batch(x, nsamples=total, max_frames=max_frames, frames=frames, states=states)

        def scan():
            states.zero_()
            auto.zero_()
            eng.rx_batch_auto(x, nsamples=total, max_frames=max_frames, frames=frames, states=states,
                              auto_states=auto)
        r = {}
        for label, fn in (("rx_batch", fixed), ("rx_batch_auto", scan)):
            ms = timed(fn)
            st = mm.states_to_numpy(states)
            r[label] = {"ms_min": round(min(ms), 3), "ms_mean": round(sum(ms) / len(ms), 3),
                        "records": int(st["nframes"].sum()), "kernel": eng.last_kernel()}
        r["auto_over_fixed"] = round(r["rx_batch_auto"]["ms_min"] / r["rx_batch"]["ms_min"], 3)
        out["results"][name] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
