#!/usr/bin/env python
"""Tone-pair channels over shared rows on the GPU: fsk_b200_rx_batch_channels on the lines against
fsk_b200_rx_batch_tones on the lines materialized k times, kernel time by CUDA events, best of --reps warmed
launches, plus the sample memory each arm holds.

    python tools/channels_bench.py [--reps 5] [--only duplex,passband,live]

Workloads (rows from fsk_b200_tx_batch with random data words, summed on the device):
  duplex    Bell103 "300" at 48 kHz, 16 384 lines x 192 000 samples; each line is an originate transmission
            (1270/1070 Hz) plus an answer transmission (2225/2025 Hz) behind a random lead-in; k = 2.
  passband  RTTY at 8 kHz, 4 096 lines x 192 000 samples; line r holds 6 RTTY signals (5 for odd r) with
            marks 400 Hz apart, each behind its own random lead-in; k = 6, the sixth channel of a 5-signal line
            disabled (a band >= nbands).
Arms:
  tones_copied  rx_batch_tones on the lines repeated k times (row r*k + j = line r), one pair per row;
  channels      rx_batch_tones(..., channels_per_row=k) on the lines.
The records and states of the two arms must be equal byte for byte; the run reports that per workload.
  live      the duplex lines through LiveReceiver(channels_per_row=2) against LiveReceiver(tones=...) on the
            copied rows, 2 000-sample chunks; time per feed (push, rx and decode) by CUDA events over the
            feeds after the first --live-warmup; the copied arm's chunks are repeated before the clock starts.
Prints one JSON line with the card's name, power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ORIGINATE, ANSWER = (1270.0, 1070.0), (2225.0, 2025.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--nsamples", type=int, default=192000)
    ap.add_argument("--duplex-lines", type=int, default=16384)
    ap.add_argument("--passband-lines", type=int, default=4096)
    ap.add_argument("--live-feeds", type=int, default=24)
    ap.add_argument("--live-warmup", type=int, default=4)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    a = ap.parse_args()

    import torch
    import minimodem_b200 as mm
    assert torch.cuda.is_available(), "channels_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    n = a.nsamples
    stride = (n + 3) & ~3
    gen = torch.Generator(device="cpu").manual_seed(20261016)
    want = lambda name: not a.only or name in a.only.split(",")

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

    def transmit(mode, rate, pair, nlines, max_lead, scale):
        """nlines rows of random words on `pair`, each behind a random lead-in of up to max_lead samples"""
        cfg = mm.rx_config_for_mode(mode, rate, f_mark=pair[0], f_space=pair[1])
        tcfg = mm.tx_config_from(cfg)
        bit = int(rate / float(cfg.data_rate))
        nwords = max(1, (n - max_lead - (tcfg.leader_bits + tcfg.trailer_bits) * bit) // (int(tcfg.n_data_bits + 3) * bit))
        words = torch.randint(0, 1 << int(tcfg.n_data_bits), (nlines, nwords), generator=gen, dtype=torch.int32).to(dev)
        lead = torch.randint(0, max_lead + 1, (nlines,), generator=gen, dtype=torch.int32).to(dev)
        return mm.tx_batch(tcfg, words, n, lead_in=lead, stride=stride).mul_(scale)

    def compare(eng, x, bands, k, max_frames):
        """(result dict, channel frames, channel states) of the two arms on lines x with k channels each"""
        S = x.shape[0]
        res = {"lines": S, "channels_per_row": k, "channels": S * k}
        frames = torch.zeros((S * k, max_frames, 5), dtype=torch.int32, device=dev)
        states = torch.zeros((S * k, mm.STATE_WORDS), dtype=torch.int32, device=dev)

        def arm(label, rows, fn):
            def once():
                states.zero_()
                fn()
            frames.zero_()
            ms = timed(once)
            st = mm.states_to_numpy(states)
            res[label] = {"ms_min": round(min(ms), 3), "ms_mean": round(sum(ms) / len(ms), 3),
                          "sample_bytes": rows.numel() * rows.element_size(), "records": int(st["nframes"].sum()),
                          "kernel": eng.last_kernel()}

        arm("channels", x, lambda: eng.rx_batch_tones(x, bands, nsamples=n, max_frames=max_frames, frames=frames,
                                                      states=states, channels_per_row=k))
        ch_frames, ch_states = frames.clone(), states.clone()
        copied = x.repeat_interleave(k, dim=0)
        arm("tones_copied", copied, lambda: eng.rx_batch_tones(copied, bands, nsamples=n, max_frames=max_frames,
                                                               frames=frames, states=states))
        res["records_and_states_equal"] = bool(torch.equal(frames, ch_frames) and torch.equal(states, ch_states))
        res["channels_over_tones_copied"] = round(res["channels"]["ms_min"] / res["tones_copied"]["ms_min"], 3)
        del copied, frames, states
        torch.cuda.empty_cache()
        return res

    out = {"tool": "channels_bench", "card": card(), "nsamples": n, "reps": a.reps, "results": {}}
    lines = None
    if want("duplex") or want("live"):
        S = a.duplex_lines
        lines = transmit("300", 48000, ORIGINATE, S, 0, 0.5)
        lines.add_(transmit("300", 48000, ANSWER, S, 48000, 0.4))
        torch.cuda.synchronize()
        eng = mm.RxEngine.for_mode("300", 48000)
        bands = eng.tone_bands([ORIGINATE[0], ANSWER[0]] * S, [ORIGINATE[1], ANSWER[1]] * S, device=dev)
        if want("duplex"):
            out["results"]["duplex"] = compare(eng, lines, bands, 2, eng.max_frames(n))

    if want("live"):
        out["results"]["live"] = live(a, mm, torch, dev, lines)
    del lines
    torch.cuda.empty_cache()

    if want("passband"):
        S, k = a.passband_lines, 6
        eng = mm.RxEngine.for_mode("rtty", 8000)
        p = eng.params
        shift = float(p.f_space) - float(p.f_mark)
        marks = [600.0 + 400.0 * i for i in range(k)]
        x = torch.zeros((S, stride), dtype=torch.float32, device=dev)
        five = (torch.arange(S, device=dev) % 2 == 1)
        for i, m in enumerate(marks):
            sig = transmit("rtty", 8000, (m, m + shift), S, 8000, 0.25)
            if i == k - 1:
                sig[five] = 0.0
            x.add_(sig)
            del sig
        torch.cuda.synchronize()
        b = eng.tone_bands(marks * S, [m + shift for m in marks] * S, device=dev).view(S, k, 2)
        b[five, k - 1] = int(p.nbands)                           # the padding channel of a 5-signal line
        r = compare(eng, x, b.view(S * k, 2).contiguous(), k, eng.max_frames(n))
        r["signals_per_line"] = "6 (even lines), 5 (odd lines, sixth channel disabled)"
        out["results"]["passband"] = r
        del x
        torch.cuda.empty_cache()
    print(json.dumps(out))


def live(a, mm, torch, dev, lines):
    """LiveReceiver with channels against LiveReceiver(tones=...) on copied rows, same 2 000-sample chunks"""
    from minimodem_b200.serving import LiveReceiver
    S, k, chunk = lines.shape[0], 2, 2000
    eng = mm.RxEngine.for_mode("300", 48000)
    bands = eng.tone_bands([ORIGINATE[0], ANSWER[0]] * S, [ORIGINATE[1], ANSWER[1]] * S, device=dev)
    nfeeds = min(a.live_feeds, lines.shape[1] // chunk)
    res = {"lines": S, "channels_per_row": k, "chunk": chunk, "feeds_timed": nfeeds - a.live_warmup}
    texts = {}
    for label, nrows, kw in (("channels", S, dict(channels_per_row=k)), ("tones_copied", S * k, {})):
        lr = LiveReceiver("300", 48000, nrows, max_chunk=chunk, device=dev, tones=bands, **kw)
        ms, got = [], []
        for f in range(nfeeds):
            c = lines[:, f * chunk:(f + 1) * chunk]
            c = (c.repeat_interleave(k, dim=0) if label == "tones_copied" else c).contiguous()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            o, cnt = lr.feed(c)
            e1.record()
            e1.synchronize()
            if f >= a.live_warmup:
                ms.append(e0.elapsed_time(e1))
            got.append((o.cpu(), cnt.cpu()))
        texts[label] = got
        res[label] = {"ms_per_feed_min": round(min(ms), 3), "ms_per_feed_mean": round(sum(ms) / len(ms), 3),
                      "row_bytes": lr.rows.numel() * lr.rows.element_size(),
                      "dropped": int(lr.dropped.sum().item())}
        del lr
        torch.cuda.empty_cache()
    res["text_equal"] = all(torch.equal(oa, ob) and torch.equal(ca, cb)
                            for (oa, ca), (ob, cb) in zip(texts["channels"], texts["tones_copied"]))
    res["channels_over_tones_copied"] = round(res["channels"]["ms_per_feed_mean"] / res["tones_copied"]["ms_per_feed_mean"], 3)
    return res


if __name__ == "__main__":
    main()
