#!/usr/bin/env python
"""Live streams that end and start on their own, on the GPU: LiveReceiver fed 2 000-sample chunks, with calls
ending and starting between feeds, time per feed (push, rx and decode) by CUDA events.

    python tools/stream_lifetimes_bench.py [--rows 16384] [--feeds 48] [--churn 0.01]

Workloads (rows from the device transmitter, float32, each channel behind a random lead-in):
  bell202   "1200" at 48 kHz, one stream per row (fsk_b200_tx_text_channels with k = 1);
  duplex    Bell103 "300" at 48 kHz, originate (1270/1070 Hz) and answer (2225/2025 Hz) summed into each row
            (fsk_b200_tx_text_channels with k = 2), decoded with tones= and channels_per_row=2.
Arms, each a whole run over the same feeds:
  steady     no churn: LiveReceiver.feed(chunk);
  events     per feed, --churn of the rows end (their chunk is the stream's last) and --churn of the rows that
             ended earlier open again: LiveReceiver.feed(chunk, opened=, ended=), one push, one rx, one decode;
  workaround the same churn without the events: the opened rows' fill, states and decoder states zeroed with
             indexed torch stores, the feed, then per ending row a one-row rx at holdback 0 (rows[r:r+1]) and a
             one-row decode, the engine's holdback toggled around them; a row that ended gets no samples after.
The texts of the events and workaround arms must be equal feed by feed; the run reports that per workload.
Prints one JSON line with the card's name, power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ORIGINATE, ANSWER = (1270.0, 1070.0), (2225.0, 2025.0)
CHUNK = 2000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--feeds", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=4, help="feeds of each arm not timed")
    ap.add_argument("--churn", type=float, default=0.01)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    a = ap.parse_args()

    import numpy as np
    import torch
    import minimodem_b200 as mm
    from minimodem_b200.serving import LiveReceiver
    assert torch.cuda.is_available(), "stream_lifetimes_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    S, n = a.rows, a.feeds * CHUNK
    gen = torch.Generator(device="cpu").manual_seed(20261017)

    def transmit(mode, pairs, k, text_len):
        """S rows of n samples, k channels each on `pairs` (one per channel of a row), random printable text"""
        te = mm.TxEngine.for_mode(mode, 48000, float_samples=True)
        text = torch.randint(32, 127, (S * k, text_len), generator=gen, dtype=torch.uint8).to(dev)
        lens = torch.randint(text_len // 2, text_len + 1, (S * k,), generator=gen, dtype=torch.int32).to(dev)
        lead = torch.randint(0, 4 * CHUNK, (S * k,), generator=gen, dtype=torch.int32).to(dev)
        tones = te.tone_pairs([p[0] for p in pairs] * S, [p[1] for p in pairs] * S, device=dev)
        rows, _ = te.text_channels(text, lens, tones, k, n, lead_in=lead)
        return rows.mul_(0.5 / k)

    def churn_plan(seed):
        """per feed: (ending rows, opening rows); a row opens again only after it has ended"""
        rng = np.random.default_rng(seed)
        live, gone, plan = np.ones(S, bool), [], []
        m = max(1, int(round(a.churn * S)))
        for f in range(a.feeds):
            opening = np.array(sorted(rng.choice(gone, min(m, len(gone)), replace=False)), np.int64) if gone else \
                np.zeros(0, np.int64)
            live[opening] = True
            gone = sorted(set(gone) - set(opening.tolist()))
            ending = np.array(sorted(rng.choice(np.nonzero(live)[0], m, replace=False)), np.int64)
            live[ending] = False
            gone = sorted(set(gone) | set(ending.tolist()))
            plan.append((ending, opening))
        return plan

    def run(label, lines, mode, k, kw, plan):
        rx = LiveReceiver(mode, 48000, S, max_chunk=CHUNK, device=dev, **kw)
        eng = rx.engine
        ms, outs = [], []
        gone = torch.zeros((S,), dtype=torch.bool, device=dev)
        full = torch.full((S,), CHUNK, dtype=torch.int32, device=dev)
        for f in range(a.feeds):
            chunk = lines[:, f * CHUNK:(f + 1) * CHUNK].contiguous()
            ending, opening = plan[f] if plan else (None, None)
            if plan:
                end_t, open_t = torch.from_numpy(ending).to(dev), torch.from_numpy(opening).to(dev)
                ended = torch.zeros((S,), dtype=torch.bool, device=dev).index_fill_(0, end_t, True)
                opened = torch.zeros((S,), dtype=torch.bool, device=dev).index_fill_(0, open_t, True)
                ch_open = (open_t[:, None] * k + torch.arange(k, device=dev)).reshape(-1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            extra = []
            if label == "steady":
                o, cnt = rx.feed(chunk)
            elif label == "events":
                o, cnt = rx.feed(chunk, opened=opened, ended=ended)
            else:
                rx.fill.index_fill_(0, open_t, 0)
                rx.states.index_fill_(0, ch_open, 0)
                rx.dstates.index_fill_(0, ch_open, 0)
                gone.index_fill_(0, open_t, False)
                o, cnt = rx.feed(chunk, torch.where(gone, 0, full))
                for r in ending.tolist():
                    c0, c1 = r * k, (r + 1) * k
                    rx.states[c0:c1, 2] = 0                      # StreamState.nframes: the records were decoded
                    rx.states[c0:c1, 7] = 0                      # StreamState.done: held back, not ended
                    eng.set_holdback(0)
                    if k > 1:
                        fr, _ = eng.rx_batch_tones(rx.rows[r:r + 1], rx.tones[c0:c1], nsamples=rx.stride,
                                                   nsamples_each=rx.fill[r:r + 1], max_frames=rx.max_frames,
                                                   states=rx.states[c0:c1], channels_per_row=k)
                    else:
                        fr, _ = eng.rx_batch(rx.rows[r:r + 1], nsamples=rx.stride, nsamples_each=rx.fill[r:r + 1],
                                             max_frames=rx.max_frames, states=rx.states[c0:c1])
                    eng.set_holdback(rx.window)
                    extra.append((r, eng.decode_batch(rx.kind, fr, rx.states[c0:c1], dstates=rx.dstates[c0:c1],
                                                      out_stride=rx.row_bytes)))
                gone.index_fill_(0, end_t, True)
            e1.record()
            e1.synchronize()
            if f >= a.warmup:
                ms.append(e0.elapsed_time(e1))
            if label != "steady":
                o, cnt = o.clone(), cnt.clone()
                for r, (xo, xc) in extra:                        # the end of a row's text, after the feed's
                    for j in range(k):
                        c, at, m = r * k + j, int(cnt[r * k + j]), int(xc[j])
                        o[c, at:at + m] = xo[j, :m]
                        cnt[c] += m
                w = int(cnt.max().item()) if cnt.numel() else 0
                outs.append((o[:, :w].cpu(), cnt.cpu()))
        res = {"ms_per_feed_mean": round(sum(ms) / len(ms), 3), "ms_per_feed_min": round(min(ms), 3),
               "text_bytes": int(sum(int(c.sum()) for _, c in outs)) if outs else None,
               "dropped_last_feed": int(rx.dropped.sum().item())}
        del rx
        torch.cuda.empty_cache()
        return res, outs

    def workload(mode, pairs, k, text_len, kw):
        lines = transmit(mode, pairs, k, text_len)
        torch.cuda.synchronize()
        plan = churn_plan(len(mode) + k)
        res = {"rows": S, "channels_per_row": k, "chunk": CHUNK, "feeds": a.feeds, "feeds_timed": a.feeds - a.warmup,
               "rows_ending_per_feed": len(plan[0][0]), "rows_opening_per_feed_max": int(max(len(p[1]) for p in plan))}
        res["steady"], _ = run("steady", lines, mode, k, kw, None)
        res["events"], te = run("events", lines, mode, k, kw, plan)
        res["workaround"], tw = run("workaround", lines, mode, k, kw, plan)

        def same(x, y):
            (ox, cx), (oy, cy) = x, y
            if not torch.equal(cx, cy):
                return False
            w = min(ox.shape[1], oy.shape[1])
            keep = torch.arange(w)[None, :] < cx[:, None]
            return bool(torch.equal(ox[:, :w][keep], oy[:, :w][keep]))
        res["events_text_equals_workaround"] = all(same(x, y) for x, y in zip(te, tw))
        res["events_over_steady"] = round(res["events"]["ms_per_feed_mean"] / res["steady"]["ms_per_feed_mean"], 3)
        res["events_over_workaround"] = round(res["events"]["ms_per_feed_mean"] / res["workaround"]["ms_per_feed_mean"], 3)
        del lines
        torch.cuda.empty_cache()
        return res

    want = lambda name: not a.only or name in a.only.split(",")
    out = {"tool": "stream_lifetimes_bench", "card": card(), "churn": a.churn, "results": {}}
    if want("bell202"):
        out["results"]["bell202"] = workload("1200", [(1200.0, 2200.0)], 1, 240, {})
    if want("duplex"):
        eng = mm.RxEngine.for_mode("300", 48000)
        bands = eng.tone_bands([ORIGINATE[0], ANSWER[0]] * S, [ORIGINATE[1], ANSWER[1]] * S, device=dev)
        out["results"]["duplex"] = workload("300", [ORIGINATE, ANSWER], 2, 60, dict(tones=bands, channels_per_row=2))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
