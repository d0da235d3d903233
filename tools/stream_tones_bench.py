#!/usr/bin/env python
"""-M / -S per stream on the GPU: kernel time of fsk_b200_rx_batch_tones against fsk_b200_rx_batch on the
same streams, by CUDA events, best of --reps warmed launches.

    python tools/stream_tones_bench.py [--streams 65536] [--nsamples 192000] [--reps 5]

Workloads, each 65 536 streams of 192 000 samples from fsk_b200_tx_batch:
  bell202  "1200" at 48 kHz; second pair 1300/2100 Hz;
  bell103  "300" at 48 kHz; originate 1270/1070 Hz, second pair the answer channel 2225/2025 Hz;
  rtty     "rtty" at 8 kHz; second pair 2125/2295 Hz.
Per workload:
  rx_batch                the fixed-tone call with the kernel it picks by default;
  rx_batch_per_candidate  the same on an engine made with FSK_B200_MULTI=0 FSK_B200_PREFIX=0, which runs the
                          per-candidate kernel the tone calls use;
  tones_preset            rx_batch_tones, every stream on the preset pair;
  tones_mix               rx_batch_tones, the first half of the streams on the preset pair, the second half on
                          the second pair (its rows transmitted on that pair).
The records and states of tones_preset must equal those of rx_batch_per_candidate bit for bit; the run
checks that and reports it.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("bell202", "1200", 48000, (1300.0, 2100.0)),
             ("bell103", "300", 48000, (2225.0, 2025.0)),
             ("rtty", "rtty", 8000, (2125.0, 2295.0))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--nsamples", type=int, default=192000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    a = ap.parse_args()

    import torch
    import minimodem_b200 as mm
    assert torch.cuda.is_available(), "stream_tones_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    S, n = a.streams, a.nsamples
    half = S // 2
    stride = (n + 3) & ~3

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

    out = {"tool": "stream_tones_bench", "card": card(), "streams": S, "nsamples": n, "reps": a.reps, "results": {}}
    x = torch.empty((S, stride), dtype=torch.float32, device=dev)
    for name, mode, rate, second in WORKLOADS:
        if a.only and name not in a.only.split(","):
            continue
        cfg = mm.rx_config_for_mode(mode, rate)
        cfg2 = mm.rx_config_for_mode(mode, rate, f_mark=second[0], f_space=second[1])
        eng = mm.RxEngine.for_mode(mode, rate)
        os.environ["FSK_B200_MULTI"], os.environ["FSK_B200_PREFIX"] = "0", "0"
        per_cand = mm.RxEngine.for_mode(mode, rate)
        del os.environ["FSK_B200_MULTI"], os.environ["FSK_B200_PREFIX"]
        p = eng.params
        preset = eng.tone_bands(float(p.f_mark), float(p.f_space), device=dev).expand(S, 2).contiguous()
        mix = eng.tone_bands([float(p.f_mark)] * half + [second[0]] * (S - half),
                             [float(p.f_space)] * half + [second[1]] * (S - half), device=dev)
        tcfg, tcfg2 = mm.tx_config_from(cfg), mm.tx_config_from(cfg2)
        bit = int(rate / float(cfg.data_rate))
        nwords = max(1, (n - (tcfg.leader_bits + tcfg.trailer_bits) * bit) // (int(tcfg.n_data_bits + 3) * bit))
        gen = torch.Generator(device="cpu").manual_seed(20261016)
        words = torch.randint(0, 1 << int(tcfg.n_data_bits), (S, nwords), generator=gen, dtype=torch.int32).to(dev)
        max_frames = eng.max_frames(n)
        frames = torch.zeros((S, max_frames, 5), dtype=torch.int32, device=dev)
        states = torch.zeros((S, mm.STATE_WORDS), dtype=torch.int32, device=dev)
        r = {"second_pair": list(second), "bands_preset": [int(p.b_mark), int(p.b_space)],
             "bands_second": mix[-1].tolist()}

        def run(label, fn, rows):
            def once():
                states.zero_()
                fn()
            ms = timed(once)
            st = mm.states_to_numpy(states)
            k = (per_cand if label == "rx_batch_per_candidate" else eng).last_kernel()
            r[label] = {"ms_min": round(min(ms), 3), "ms_mean": round(sum(ms) / len(ms), 3),
                        "msamples_per_s": round(S * n / (min(ms) * 1e3), 1), "records": int(st["nframes"].sum()),
                        "rows": rows, "kernel": k}

        mm.tx_batch(tcfg, words, n, out=x, stride=stride)
        torch.cuda.synchronize()
        run("rx_batch", lambda: eng.rx_batch(x, nsamples=n, max_frames=max_frames, frames=frames, states=states),
            "preset")
        frames.zero_()
        run("rx_batch_per_candidate", lambda: per_cand.rx_batch(x, nsamples=n, max_frames=max_frames, frames=frames,
                                                                  states=states), "preset")
        ref_frames, ref_states = frames.clone(), states.clone()
        frames.zero_()
        run("tones_preset", lambda: eng.rx_batch_tones(x, preset, nsamples=n, max_frames=max_frames, frames=frames,
                                                        states=states), "preset")
        r["tones_preset_equals_per_candidate"] = bool(torch.equal(frames, ref_frames) and torch.equal(states, ref_states))
        del ref_frames, ref_states
        mm.tx_batch(tcfg2, words[half:], n, out=x[half:], stride=stride)
        torch.cuda.synchronize()
        run("tones_mix", lambda: eng.rx_batch_tones(x, mix, nsamples=n, max_frames=max_frames, frames=frames,
                                                     states=states), "half preset, half second pair")
        r["tones_preset_over_rx_batch"] = round(r["tones_preset"]["ms_min"] / r["rx_batch"]["ms_min"], 3)
        r["tones_preset_over_per_candidate"] = round(r["tones_preset"]["ms_min"] / r["rx_batch_per_candidate"]["ms_min"], 3)
        out["results"][name] = r
        del frames, states
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
