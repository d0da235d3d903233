#!/usr/bin/env python
"""The transmitter's tone pair per stream and its tone-pair channels summed into shared rows, on the GPU.
Kernel times by CUDA events, best of `--reps` warmed launches; one JSON line with the card's name, power limit
and max SM clock.

    python tools/tx_channels_bench.py

- tones: 65 536 Bell202 streams of 480 characters (about 192 000 samples each), float32 and int16,
  --lut=4096: text_batch (the fixed pair); text_batch_tones with the engine's own pair on every stream (rows,
  counts and states must equal text_batch's byte for byte); text_batch_tones with every second stream on
  1300/2100 Hz.
- duplex: Bell103 at 48 kHz, 192 000 samples per line, originate (1270/1070) + answer (2225/2025) behind random
  lead-ins, k = 2.  (a) 16 384 lines: text_channels against two text_batch_tones row sets placed at their
  lead-ins and added with torch; the rows must be equal; time and peak device memory of both.  (b) 65 536
  lines as float32, text_channels alone (the other arm does not fit), fed to rx_batch_tones(channels_per_row=2):
  whether every channel decodes to the text sent.
- passband: RTTY at 8 kHz, 4 096 lines x 6 channels 400 Hz apart, int16, the sixth disabled on odd lines;
  the first rows checked against the saturated int32 sum of their channels sent one per row."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tx_bench import card, rates, timed, words_for  # noqa: E402


def tones_workload(torch, mm, streams, chars, float_samples, warmup, reps):
    dev = torch.device("cuda:0")
    te = mm.TxEngine.for_mode("1200", 48000, float_samples=float_samples)
    text = words_for(torch, streams, chars, dev).to(torch.uint8)
    lens = torch.full((streams,), chars, dtype=torch.int32, device=dev)
    stride = (te.max_samples(chars, mm.TX_FINAL) + 7) & ~7
    dt = torch.float32 if float_samples else torch.int16
    own = te.tone_pairs(te.cfg.f_mark, te.cfg.f_space, device=dev).expand(streams, 2).contiguous()
    half = own.clone()
    half[1::2] = te.tone_pairs(1300.0, 2100.0, device=dev)
    res = {}
    # one row buffer for all arms (a float32 set is 50 GB at the default size)
    out = torch.empty((streams, stride), dtype=dt, device=dev)
    states = te.new_states(streams, dev)
    cnt = torch.empty((streams,), dtype=torch.int32, device=dev)
    for arm, tones in (("own_pair", own), ("half_moved", half), ("text_batch", None)):
        def run():
            states.zero_()
            te.text_batch(text, lens, states, mm.TX_FINAL, out=out, out_len=cnt, tones=tones)
        best, mean = timed(torch, run, warmup, reps)
        samples = int(cnt.sum().item())
        r = rates(samples, 4 if float_samples else 2, best)
        r.update(mean_ms=round(mean, 3), samples_per_stream=samples // streams)
        res[arm] = r
    # the text_batch arm ran last: the own-pair call must give its rows, counts and states, compared in slices
    n = int(cnt.max().item())
    equal, step = int(cnt.min().item()) == n, 4096                 # every row has the same length here
    for i in range(0, streams, step):
        j = min(i + step, streams)
        st = te.new_states(j - i, dev)
        o, c = te.text_batch(text[i:j], lens[i:j], st, mm.TX_FINAL, out=torch.empty((j - i, stride), dtype=dt, device=dev),
                             tones=own[i:j])
        equal &= bool(torch.equal(o[:, :n], out[i:j, :n]) and torch.equal(c, cnt[i:j]) and torch.equal(st, states[i:j]))
    res["own_pair_equal"] = equal
    res["own_pair_over_text_batch"] = round(res["own_pair"]["ms"] / res["text_batch"]["ms"], 4)
    res["half_moved_over_text_batch"] = round(res["half_moved"]["ms"] / res["text_batch"]["ms"], 4)
    del out
    torch.cuda.empty_cache()
    return res


def place(torch, audio, cnt, lead, nout):
    """rows [n, nout]: audio[s, :cnt[s]] placed at lead[s], zero elsewhere, cut at nout (in slices of rows)"""
    n = audio.shape[0]
    out = torch.zeros((n, nout), dtype=audio.dtype, device=audio.device)
    pos = torch.arange(nout, device=audio.device)
    for i in range(0, n, 1024):
        j = min(i + 1024, n)
        idx = pos[None, :] - lead[i:j, None].long()
        ok = (idx >= 0) & (idx < cnt[i:j, None].long())
        out[i:j] = torch.where(ok, audio[i:j].gather(1, idx.clamp(0, audio.shape[1] - 1)),
                               torch.zeros((), dtype=audio.dtype, device=audio.device))
    return out


def duplex_inputs(torch, mm, te, lines, chars, nout, seed):
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(seed)
    text = torch.randint(32, 127, (lines * 2, chars), generator=g, dtype=torch.uint8).to(dev)
    lens = torch.full((lines * 2,), chars, dtype=torch.int32, device=dev)
    lead = torch.randint(0, nout - te.max_samples(chars, mm.TX_FINAL), (lines * 2,), generator=g,
                         dtype=torch.int32).to(dev)
    tones = te.tone_pairs([1270.0, 2225.0] * lines, [1070.0, 2025.0] * lines, device=dev)
    return text, lens, lead, tones


def peak(torch, fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    r = fn()
    torch.cuda.synchronize()
    return r, torch.cuda.max_memory_allocated() - base


def duplex_a(torch, mm, lines, chars, nout, warmup, reps):
    """text_channels against two text_batch_tones row sets placed at their lead-ins and added with torch"""
    te = mm.TxEngine.for_mode("300", 48000, float_samples=True)
    text, lens, lead, tones = duplex_inputs(torch, mm, te, lines, chars, nout, 11)
    dev = text.device
    stride = (nout + 7) & ~7
    rows = torch.empty((lines, stride), dtype=torch.float32, device=dev)
    cnt = torch.empty((lines * 2,), dtype=torch.int32, device=dev)
    res = {"lines": lines, "nsamples": nout}
    ms, _ = timed(torch, lambda: te.text_channels(text, lens, tones, 2, nout, lead_in=lead, out=rows, out_len=cnt),
                  warmup, reps)
    _, mem = peak(torch, lambda: te.text_channels(text, lens, tones, 2, nout, lead_in=lead))
    res["text_channels"] = {"ms": round(ms, 3), "peak_bytes": mem}
    ostride = (te.max_samples(chars, mm.TX_FINAL) + 7) & ~7

    def two_sets():
        out = []
        for d in (0, 1):
            a, c = te.text_batch(text[d::2].contiguous(), lens[d::2].contiguous(), te.new_states(lines, dev),
                                 mm.TX_FINAL, out=torch.empty((lines, ostride), dtype=torch.float32, device=dev),
                                 tones=tones[d::2].contiguous())
            out.append(place(torch, a, c, lead[d::2].contiguous(), nout))
            del a
        return out[0] + out[1]
    ms2, _ = timed(torch, two_sets, 1, 3)
    want, mem2 = peak(torch, two_sets)
    res["two_row_sets_plus_add"] = {"ms": round(ms2, 3), "peak_bytes": mem2}
    res["rows_equal"] = bool(torch.equal(rows[:, :nout], want))
    res["out_len_equal"] = bool(torch.equal(cnt.long(), (lead.long() + te.max_samples(chars, mm.TX_FINAL))))
    del rows, want
    torch.cuda.empty_cache()
    return res


def duplex_b(torch, mm, lines, chars, nout, warmup, reps):
    """text_channels alone, float32, decoded by rx_batch_tones(channels_per_row=2)"""
    te = mm.TxEngine.for_mode("300", 48000, float_samples=True)
    text, lens, lead, tones = duplex_inputs(torch, mm, te, lines, chars, nout, 12)
    dev = text.device
    rows = torch.empty((lines, nout), dtype=torch.float32, device=dev)
    cnt = torch.empty((lines * 2,), dtype=torch.int32, device=dev)
    ms, _ = timed(torch, lambda: te.text_channels(text, lens, tones, 2, nout, lead_in=lead, out=rows, out_len=cnt),
                  warmup, reps)
    res = {"lines": lines, "nsamples": nout, "text_channels": {"ms": round(ms, 3)},
           "rows_bytes": rows.numel() * 4, "peak_bytes_allocated": torch.cuda.max_memory_allocated()}
    rx = mm.RxEngine.for_mode("300", 48000)
    bands = rx.tone_bands([1270.0, 2225.0] * lines, [1070.0, 2025.0] * lines, device=dev)
    exact = whole = total = 0
    for i in range(0, lines, 16384):                               # records for 16 384 lines at a time
        j = min(i + 16384, lines)
        frames, states = rx.rx_batch_tones(rows[i:j], bands[2 * i:2 * j].contiguous(), channels_per_row=2)
        got, n = rx.decode_batch(mm.decoder_for_mode("300", rx.params.n_data_bits), frames, states)
        g, c, t = got.cpu().numpy(), n.cpu().numpy(), text[2 * i:2 * j].cpu().numpy()
        for ch in range(t.shape[0]):
            d = g[ch, :c[ch]].tobytes()
            exact += d == t[ch].tobytes()
            whole += t[ch].tobytes() in d
        total += t.shape[0]
        del frames, states, got
    res["channels"] = total
    res["decoded_exact"] = exact          # the decoded text is the text sent
    res["decoded_whole"] = whole          # the text sent is there whole, with bytes of the other direction around it
    del rows
    torch.cuda.empty_cache()
    return res


def passband(torch, mm, lines, chars, nout, warmup, reps, check_rows=256):
    """RTTY at 8 kHz, 6 channels 400 Hz apart, int16, the sixth disabled on odd lines"""
    dev = torch.device("cuda:0")
    k = 6
    te = mm.TxEngine.for_mode("rtty", 8000, amplitude=1.0 / k)
    g = torch.Generator(device="cpu").manual_seed(13)
    text = torch.randint(65, 91, (lines * k, chars), generator=g, dtype=torch.uint8).to(dev)
    lens = torch.full((lines * k,), chars, dtype=torch.int32, device=dev)
    marks = [800.0 + 400 * j for j in range(k)] * lines
    spaces = [800.0 + 400 * j - 170.0 for j in range(k)] * lines
    for r in range(1, lines, 2):
        spaces[r * k + k - 1] = float("nan")
    tones = torch.tensor([marks, spaces], dtype=torch.float32).t().contiguous().to(dev)
    rows = torch.empty((lines, (nout + 7) & ~7), dtype=torch.int16, device=dev)
    cnt = torch.empty((lines * k,), dtype=torch.int32, device=dev)
    ms, _ = timed(torch, lambda: te.text_channels(text, lens, tones, k, nout, out=rows, out_len=cnt), warmup, reps)
    # the first rows against the saturated int32 sum of their channels sent one per row
    n = check_rows * k
    a, c = te.text_batch(text[:n], lens[:n], te.new_states(n, dev), mm.TX_FINAL, tones=tones[:n])
    ch = place(torch, a, c, torch.zeros((n,), dtype=torch.int32, device=dev), nout).int()
    want = ch.view(check_rows, k, nout).sum(dim=1).clamp(-32768, 32767).short()
    return {"lines": lines, "channels": k, "nsamples": nout, "text_channels": {"ms": round(ms, 3)},
            "rows_bytes": rows.numel() * 2, "checked_rows": check_rows,
            "rows_equal": bool(torch.equal(rows[:check_rows, :nout], want)),
            "disabled_out_len_zero": bool((cnt.view(lines, k)[1::2, k - 1] == 0).all().item())}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--chars", type=int, default=480)
    ap.add_argument("--duplex-lines", type=int, default=16384)
    ap.add_argument("--duplex-big-lines", type=int, default=65536)
    ap.add_argument("--duplex-chars", type=int, default=100)
    ap.add_argument("--passband-lines", type=int, default=4096)
    ap.add_argument("--passband-chars", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import minimodem_b200 as mm
    assert torch.cuda.is_available(), "tx_channels_bench.py needs a CUDA device"
    res = {"card": card(), "library": mm.version(), "streams": a.streams, "chars": a.chars}
    res["bell202_float"] = tones_workload(torch, mm, a.streams, a.chars, True, a.warmup, a.reps)
    res["bell202_int16"] = tones_workload(torch, mm, a.streams, a.chars, False, a.warmup, a.reps)
    res["duplex_a"] = duplex_a(torch, mm, a.duplex_lines, a.duplex_chars, 192000, a.warmup, a.reps)
    res["duplex_b"] = duplex_b(torch, mm, a.duplex_big_lines, a.duplex_chars, 192000, a.warmup, a.reps)
    res["passband"] = passband(torch, mm, a.passband_lines, a.passband_chars, 64000, a.warmup, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
