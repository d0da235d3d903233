#!/usr/bin/env python
"""The live receiver on 16-bit PCM, on the GPU: device time per feed of LiveReceiver for three ways of feeding
int16 audio, alternated in one run.

    python tools/live_pcm16_bench.py [--streams 65536] [--rounds 3] [--feeds 200] [--warmup 10]

Workloads (int16 audio from the device transmitter, one stream per row behind a random lead-in, cycled over a
block of --block chunks):
  bell202-20ms / bell202-100ms   "1200" at 48 kHz, chunks of 960 / 4 800 samples;
  rtty-20ms / rtty-100ms         "rtty" at 8 kHz, chunks of 160 / 800 samples.
Arms, each a LiveReceiver of its own over the same chunks, alternated in rounds of --feeds feeds:
  f32         float32 rows fed float32 chunks (the chunk widened before the timed window: a float source);
  widen+f32   what an int16 source does without pcm16: fsk_b200_s16_to_f32 on each chunk, then the float feed;
  pcm16       LiveReceiver(pcm16=True): int16 rows, the int16 push and the _s16 rx call.
Per arm: the device time of a feed (CUDA events around it, then a synchronise), the bytes of its rows, and a
check that the three arms' text and counts are equal feed by feed.  Prints one JSON line with the card's name,
power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "bell202-20ms": ("1200", 48000, 960),
    "bell202-100ms": ("1200", 48000, 4800),
    "rtty-20ms": ("rtty", 8000, 160),
    "rtty-100ms": ("rtty", 8000, 800),
}
ARMS = ("f32", "widen+f32", "pcm16")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--feeds", type=int, default=200, help="feeds of each arm per round")
    ap.add_argument("--warmup", type=int, default=10, help="feeds of each arm before the first round, not timed")
    ap.add_argument("--block", type=int, default=16, help="chunks of transmitted audio, cycled")
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    a = ap.parse_args()

    import torch
    import minimodem_b200 as mm
    from minimodem_b200.serving import LiveReceiver
    assert torch.cuda.is_available(), "live_pcm16_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    S = a.streams
    gen = torch.Generator(device="cpu").manual_seed(20261017)

    def transmit(mode, rate, n):
        """S rows of n int16 samples: random printable text after a random lead-in, the transmitter's default"""
        cfg = mm.rx_config_for_mode(mode, rate)
        te = mm.TxEngine.for_mode(mode, rate)
        text_len = int(n / rate * cfg.data_rate / 8) + 8
        text = torch.randint(32, 127, (S, text_len), generator=gen, dtype=torch.uint8).to(dev)
        lens = torch.full((S,), text_len, dtype=torch.int32, device=dev)
        lead = torch.randint(0, n // 8, (S,), generator=gen, dtype=torch.int32).to(dev)
        tones = te.tone_pairs([cfg.f_mark] * S, [cfg.f_space] * S, device=dev)
        rows, _ = te.text_channels(text, lens, tones, 1, n, lead_in=lead)
        assert rows.dtype == torch.int16
        return rows

    def digest(out):
        text, cnt = out
        w = int(cnt.max().item()) if cnt.numel() else 0
        keep = torch.arange(w, device=dev)[None, :] < cnt[:, None]
        t = torch.where(keep, text[:, :w].to(torch.int64), 0)
        pos = torch.arange(1, w + 1, device=dev, dtype=torch.int64)[None, :]
        return (int(cnt.sum().item()), int((t * pos).sum().item()), int(t.sum(dim=1).mul(
            torch.arange(1, S + 1, device=dev, dtype=torch.int64)).sum().item()))

    def workload(name):
        mode, rate, c = WORKLOADS[name]
        audio = transmit(mode, rate, a.block * c)
        rx = {arm: LiveReceiver(mode, rate, S, max_chunk=c, device=dev, pcm16=(arm == "pcm16")) for arm in ARMS}
        assert rx["pcm16"].rows.dtype == torch.int16, "the int16 rows are not in use for %s" % name
        wide = torch.empty((S, c), dtype=torch.float32, device=dev)
        ms = {arm: [] for arm in ARMS}
        dig = {arm: [] for arm in ARMS}
        nxt = {arm: 0 for arm in ARMS}

        def feed(arm, timed):
            i = nxt[arm] % a.block
            nxt[arm] += 1
            chunk = audio[:, i * c:(i + 1) * c].contiguous()
            if arm == "f32":
                mm.s16_to_f32(chunk, out=wide)                 # a float source: not part of the feed
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if arm == "f32":
                out = rx[arm].feed(wide)
            elif arm == "widen+f32":
                out = rx[arm].feed(mm.s16_to_f32(chunk, out=wide))
            else:
                out = rx[arm].feed(chunk)
            e1.record()
            e1.synchronize()
            if timed:
                ms[arm].append(e0.elapsed_time(e1))
            dig[arm].append(digest(out))

        for arm in ARMS:
            for _ in range(a.warmup):
                feed(arm, False)
        for _ in range(a.rounds):
            for arm in ARMS:
                for _ in range(a.feeds):
                    feed(arm, True)
        res = {"mode": mode, "sample_rate": rate, "chunk_samples": c, "streams": S,
               "feeds_timed_per_arm": a.rounds * a.feeds, "stride": {arm: rx[arm].stride for arm in ARMS}}
        for arm in ARMS:
            v = sorted(ms[arm])
            r = rx[arm].rows
            res[arm] = {"ms_per_feed_mean": round(sum(v) / len(v), 4), "ms_per_feed_median": round(v[len(v) // 2], 4),
                        "ms_per_feed_min": round(v[0], 4), "timed_s": round(sum(v) / 1000, 3),
                        "row_bytes": r.numel() * r.element_size(), "row_dtype": str(r.dtype).replace("torch.", ""),
                        "rx_kernel": rx[arm].engine.last_kernel().split(" ")[0]}
        res["text_bytes"] = sum(d[0] for d in dig["pcm16"])
        res["text_and_counts_equal"] = dig["f32"] == dig["widen+f32"] == dig["pcm16"]
        res["pcm16_over_widen+f32"] = round(res["pcm16"]["ms_per_feed_mean"] / res["widen+f32"]["ms_per_feed_mean"], 3)
        res["pcm16_over_f32"] = round(res["pcm16"]["ms_per_feed_mean"] / res["f32"]["ms_per_feed_mean"], 3)
        del rx, audio, wide
        torch.cuda.empty_cache()
        return res

    out = {"tool": "live_pcm16_bench", "card": card(), "results": {}}
    for name in WORKLOADS:
        if not a.only or name in a.only.split(","):
            out["results"][name] = workload(name)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
