"""Tone-pair channels over shared rows: fsk_b200_rx_batch_channels / _s16 and fsk_b200_stream_push_channels.

A channel is a (row, tone pair) combination; every row carries k channels and channel c = r*k + j reads row
r.  Channel (r, j) must give what the reference CLI gives on row r with its pair, which is what
fsk_b200_rx_batch_tones gives on a copy of the row: the channel call is pinned bit for bit against the
tone call over rows materialized k times, and against the screened FLAT oracle on a full-duplex Bell103 line
and an RTTY passband.  The push is pinned to a numpy model of its rule.

The CPU test runs the `gpu` tests of this file on the host SIMT emulation of the kernels (tests/emu)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from gpudev import bands_tensor, dev, mm, pcm, records, rows, state_rows, sync, torch, upload
from rxcases import (ANSWER, COVER, KEYS, ORIGINATE, channel_rows, check_channels_against_oracle, duplex_case,
                     on_pair, push_model, random_states, run_channels, transmission)

EINVAL = 22
f32 = np.float32


def test_gpu_channels_file_on_the_emulated_kernels():
    """The `gpu` tests below on the host SIMT emulation of the kernels: copies landing late, the
    approximate units moved by up to 64 ulp."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 2400, module="test_gpu_channels.py",
                        extra_env={"FSK_EMU_ULP": "64"})
    assert " passed" in tail and "failed" not in tail


def test_live_receiver_channels_need_tones():
    from minimodem_b200.serving import LiveReceiver
    with pytest.raises(ValueError, match="needs tones"):
        LiveReceiver("300", 48000, 2, channels_per_row=2)


# --------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------


def nbands_of(mode, rate):
    return int(mm().RxEngine.for_mode(mode, rate).params.nbands)


# --------------------------------------------------------------------------
# 1. bit identity with copied rows
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_channels_equal_the_tone_call_on_copied_rows(key):
    """Every AUTO_COMBOS shape, k in {1, 2, 3, 5}: rx_batch_channels(rows, k, P) gives the records and states
    of rx_batch_tones(rows repeated k times, P) byte for byte, on the same kernel instance; float32 and int16
    rows, per-row lengths and nsamples_all."""
    mode, rate = COVER[key]
    G, W, L = key
    eng = mm().RxEngine.for_mode(mode, rate)
    for k in (1, 2, 3, 5):
        streams, lens, b = channel_rows(mode, rate, 2, k, zlib.crc32(repr((key, k)).encode()))
        bands = bands_tensor(b)
        variants = [(np.float32, True), (np.int16, False)] if k % 2 else [(np.int16, True), (np.float32, False)]
        for dtype, per_row in variants:
            buf, n = rows([pcm(a) for a in streams] if dtype == np.int16 else streams, dtype,
                          8 if dtype == np.int16 else 4)
            nall = n if per_row else int(lens.min())
            rep, lrep = np.repeat(buf, k, axis=0), np.repeat(lens, k)
            fa, sa = run_channels(eng, buf, nall, lens, bands, k, per_row=per_row)
            ka = eng.last_kernel()
            fb, sb = eng.rx_batch_tones(upload(rep), bands, nsamples=nall, nsamples_each=upload(lrep) if per_row else None)
            sync()
            kb = eng.last_kernel()
            what = (key, k, dtype.__name__, per_row)
            assert kb.startswith("k_rx_tones<G=%d,W=%d,L=%d,mode=0(per-candidate)" % (G, W, L)), (what, kb)
            assert ka == kb + (" channels=%d" % k if k > 1 else ""), (what, ka, kb)
            ra, sa = records(fa, sa)
            rb, sb = records(fb, sb)
            assert sa.tobytes() == sb.tobytes(), what
            assert ra == rb, what
            assert (sa["done"] == 1).sum() >= len(streams) and sa["nframes"].sum() >= 2, what
            off = b.reshape(-1, 2).max(axis=1) >= eng.params.nbands
            assert (sa["nframes"][off] == 0).all() and (sa["pos"][off] == 0).all(), what


# --------------------------------------------------------------------------
# 2. and 3. the oracle: a full-duplex line and a passband
# --------------------------------------------------------------------------


@pytest.mark.gpu
def test_full_duplex_bell103_lines_against_the_oracle():
    """Bell103 lines carrying originate and answer summed, at different offsets and amplitudes, k = 2: the
    originate channel and the answer channel of each line give the oracle's records on their pair."""
    rng = np.random.default_rng(2225)
    mo, ma = on_pair("300", 48000, *ORIGINATE), on_pair("300", 48000, *ANSWER)
    lines = []
    for _ in range(3):
        a = transmission(rng, mo, int(rng.integers(4, 7)), float(rng.uniform(0.2, 0.8)))
        b = transmission(rng, ma, int(rng.integers(4, 7)), float(rng.uniform(0.2, 0.8)))
        oa, ob = (int(v) for v in rng.integers(0, 3000, 2))
        x = np.zeros(max(oa + a.size, ob + b.size) + int(rng.integers(0, 1500)), np.float32)
        x[oa:oa + a.size] += a
        x[ob:ob + b.size] += b
        lines.append((x + f32(1e-3) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32))
    eng = mm().RxEngine.for_mode("300", 48000)
    texts = check_channels_against_oracle(eng, "300", 48000, lines, [[ORIGINATE, ANSWER]] * 3, 2, "duplex")
    assert all(len(t) >= 3 for t in texts)
    for r in range(3):
        assert texts[2 * r] != texts[2 * r + 1]


@pytest.mark.gpu
def test_rtty_passband_against_the_oracle():
    """RTTY at 8 kHz, several signals about 400 Hz apart on one row, one channel per signal plus one on an
    empty pair: every channel gives the oracle's records on its row and pair; the empty one gives no frame."""
    rng = np.random.default_rng(45)
    lines, pairs = [], []
    for nsig in (3, 2):
        x, ps = np.zeros(0, np.float32), []
        for i in range(nsig):
            mark = 700.0 + 400.0 * i + float(rng.uniform(-20, 20))
            ps.append((mark + 170.0, mark))
            m = on_pair("rtty", 8000, *ps[-1])
            a = transmission(rng, m, int(rng.integers(4, 7)), float(rng.uniform(0.2, 0.6)))
            a = np.concatenate([np.zeros(int(rng.integers(0, 1500)), np.float32), a])
            y = np.zeros(max(x.size, a.size), np.float32)
            y[:x.size] += x
            y[:a.size] += a
            x = y
        ps.append((2900.0, 2730.0))                                 # nothing is sent there
        pairs.append(ps + [ps[-1]] * (4 - len(ps)))
        lines.append((x + f32(1e-3) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32))
    eng = mm().RxEngine.for_mode("rtty", 8000)
    texts = check_channels_against_oracle(eng, "rtty", 8000, lines, pairs, 4, "passband")
    assert all(len(texts[c]) >= 1 for c in (0, 1, 2, 4, 5)), texts
    assert texts[3] == b"" and texts[6] == b"" and texts[7] == b""


# --------------------------------------------------------------------------
# 4. disabled channels, 5. output overflow
# --------------------------------------------------------------------------
def duplex_rows():
    """Three Bell103 lines of rxcases.duplex_case: both directions summed, originate only, answer only"""
    streams, _, _ = duplex_case()
    return [streams[6], streams[0], streams[1]]


@pytest.mark.gpu
def test_a_disabled_channel_is_skipped_and_leaves_its_row_alone():
    """A channel with a band >= nbands gets no records and keeps its state byte for byte; the other channels
    of its row give what they give with that channel enabled."""
    t = torch()
    lines = duplex_rows()
    eng = mm().RxEngine.for_mode("300", 48000)
    nb = int(eng.params.nbands)
    k = 3
    good = eng.tone_bands([ORIGINATE[0], ANSWER[0], ORIGINATE[0]] * 3, [ORIGINATE[1], ANSWER[1], ORIGINATE[1]] * 3,
                          device=dev())
    buf, n = rows(lines, np.float32, 4)
    lens = np.array([a.size for a in lines], np.int32)
    fa, sa = run_channels(eng, buf, n, lens, good, k)
    ra, sa = records(fa, sa)
    for c in (1, 3, 8):
        for bad in ([nb, 5], [5, nb], [0xFFFFFFFF, 0xFFFFFFFF]):
            bands = good.clone()
            bands[c] = t.tensor(np.array(bad, np.uint32).view(np.int32)).to(bands.device)
            st0 = np.zeros(9, mm().STATE_DTYPE)
            st0["pos"][c], st0["carrier"][c], st0["track_amplitude"][c], st0["nframes"][c] = 1234, 1, 0.5, 2
            frames = t.full((9, eng.max_frames(n), 5), 0x5A5A5A5A, dtype=t.int32).to(dev())
            fb, sb = eng.rx_batch_tones(upload(buf), bands, nsamples=n, nsamples_each=upload(lens), frames=frames,
                                        states=state_rows(st0), channels_per_row=k)
            sync()
            assert (frames.cpu().numpy()[c] == 0x5A5A5A5A).all(), (c, bad)
            rb, sb = records(fb, sb)
            assert sb[c].tobytes() == st0[c].tobytes(), (c, bad)
            for o in range(9):
                if o != c:
                    assert sb[o].tobytes() == sa[o].tobytes() and rb[o] == ra[o], (c, bad, o)


@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
def test_channel_output_overflow_resumes_to_the_records_of_one_pass(src):
    """Every call stops after 3 records per channel and the next resumes from the saved states: the records
    and final states of one pass."""
    lines = duplex_rows()
    eng = mm().RxEngine.for_mode("300", 48000)
    k = 2
    bands = eng.tone_bands([ORIGINATE[0], ANSWER[0]] * 3, [ORIGINATE[1], ANSWER[1]] * 3, device=dev())
    buf, n = rows([pcm(a) for a in lines], np.int16, 8) if src == "s16" else rows(lines, np.float32, 4)
    lens = np.array([a.size for a in lines], np.int32)
    whole, sw = records(*run_channels(eng, buf, n, lens, bands, k))
    whole = [[w[i:i + 20] for i in range(0, len(w), 20)] for w in whole]
    states = torch().zeros((6, mm().STATE_WORDS), dtype=torch().int32).to(dev())
    got = [[] for _ in range(6)]
    for call in range(10000):
        frames, states = run_channels(eng, buf, n, lens, bands, k, states=states, max_frames=3)
        recs, st = records(frames, states)
        for c in range(6):
            got[c] += [recs[c][i:i + 20] for i in range(0, len(recs[c]), 20)]
        if (st["done"] == 1).all():
            break
        st["nframes"][:] = 0
        states = state_rows(st)
    assert call >= 2 and got == whole
    st["nframes"] = sw["nframes"]
    assert st.tobytes() == sw.tobytes()


# --------------------------------------------------------------------------
# 6. the push against a numpy model
# --------------------------------------------------------------------------


@pytest.mark.gpu
def test_push_follows_the_channel_rule():
    """fsk_b200_stream_push_channels against a numpy model: k = 1, 3 and 40 (more than a warp), disabled
    channels, a row with no active channel, positions beyond fill, chunks that do not fit (counted in
    dropped); with k = 1 and no bands it equals fsk_b200_stream_push."""
    t = torch()
    rng = np.random.default_rng(31)
    stride, nrows, nb = 512, 7, 40
    for k in (1, 3, 40):
        for with_bands in (False, True):
            fill = rng.integers(0, stride + 1, nrows).astype(np.int32)
            fill[0] = stride                                      # a full row: the chunk cannot fit
            rows0 = rng.standard_normal((nrows, stride)).astype(np.float32)
            st0 = random_states(rng, nrows * k, fill, k)
            st0["pos"][0] = 0                                    # row 0 keeps all of its samples
            bands = None
            if with_bands:
                bands = rng.integers(0, nb, (nrows * k, 2)).astype(np.uint32)
                off = rng.random(nrows * k) < 0.4
                bands[off, int(rng.integers(2))] = nb + rng.integers(0, 3, int(off.sum())).astype(np.uint32)
                bands[0] = (1, 2)
                bands[2 * k:3 * k, 0] = nb                       # row 2: no active channel
            chunk = rng.standard_normal((nrows, 300)).astype(np.float32)
            clen = rng.integers(0, 301, nrows).astype(np.int32)
            clen[0] = 300
            want = push_model(rows0, fill.astype(np.int64), st0, k, bands, nb, chunk, clen)
            R, F, S, D = upload(rows0), upload(fill), state_rows(st0), upload(np.full(nrows, -1, np.int32))
            bt = upload(bands.view(np.int32)) if bands is not None else None
            mm().stream_push(R, F, S, upload(chunk), upload(clen), dropped=D, channels_per_row=k, tone_bands=bt, nbands=nb)
            sync()
            what = (k, with_bands)
            assert (R.cpu().numpy() == want[0]).all(), what
            assert (F.cpu().numpy() == want[1]).all(), what
            got = np.frombuffer(S.cpu().numpy().tobytes(), mm().STATE_DTYPE)
            assert got.tobytes() == want[2].tobytes(), what
            assert (D.cpu().numpy() == want[3]).all() and want[3][0] > 0, what
            if with_bands:
                assert want[1][2] == min(int(clen[2]), stride)  # row 2 kept nothing
            if k == 1 and not with_bands:
                R2, F2, S2, D2 = upload(rows0), upload(fill), state_rows(st0), upload(np.full(nrows, -1, np.int32))
                ch2, cl2 = upload(chunk), upload(clen)
                p = lambda x: C.c_void_p(x.data_ptr())
                assert mm().lib().fsk_b200_stream_push(p(R2), nrows, stride, p(F2), p(S2), p(ch2), 300, p(cl2), 0,
                                                       p(D2), None) == 0
                sync()
                for a, b in ((R, R2), (F, F2), (S, S2), (D, D2)):
                    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


# --------------------------------------------------------------------------
# 7. live
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_live_receiver_with_channels_does_not_depend_on_the_cut():
    """LiveReceiver(channels_per_row=3) on duplex lines, each row with an originate, an answer and a disabled
    channel, fed random per-row cuts at two chunk sizes: the text per channel of one whole-row channel call,
    nothing dropped, and no row grows past window + frame + chunk (the disabled channel does not pin it)."""
    from minimodem_b200.serving import LiveReceiver
    lines = duplex_rows()
    eng = mm().RxEngine.for_mode("300", 48000)
    nb = int(eng.params.nbands)
    k, nrows = 3, len(lines)
    b = np.array([list(mm().tone_bands(eng.params, *ORIGINATE)), list(mm().tone_bands(eng.params, *ANSWER)),
                  [nb, 3]] * nrows, np.uint32)
    bands = bands_tensor(b)
    buf, n = rows(lines, np.float32, 4)
    lens = np.array([a.size for a in lines], np.int64)
    frames, states = run_channels(eng, buf, n, lens.astype(np.int32), bands, k)
    out, cnt = eng.decode_batch(mm().DECODE_ASCII, frames, states)
    sync()
    whole = [out.cpu().numpy()[c, :int(cnt.cpu().numpy()[c])].tobytes() for c in range(nrows * k)]
    # row 0 carries both directions, row 1 originate only, row 2 answer only
    assert all(len(whole[c]) >= 5 for c in (0, 1, 3, 7)) and whole[2] == whole[5] == whole[8] == b""
    rng = np.random.default_rng(11)
    t = torch()
    for max_chunk in (701, 5000):
        lr = LiveReceiver("300", 48000, nrows, max_chunk=max_chunk, device=dev(), tones=bands, channels_per_row=k)
        bound = lr.window + lr.engine.params.frame_nsamples + max_chunk
        fed = np.zeros(nrows, np.int64)
        texts = [b""] * (nrows * k)

        def take(res):
            o, c = res
            o, c = o.cpu().numpy(), c.cpu().numpy()
            assert o.shape[0] == nrows * k
            assert (lr.dropped.cpu().numpy() == 0).all() and (lr.fill.cpu().numpy() <= bound).all()
            return [texts[s] + o[s, :c[s]].tobytes() for s in range(nrows * k)]
        while (fed < lens).any():
            m = np.minimum(rng.integers(1, max_chunk + 1, nrows), lens - fed)
            chunk = np.zeros((nrows, max_chunk), np.float32)
            for r in range(nrows):
                chunk[r, :m[r]] = buf[r, fed[r]:fed[r] + m[r]]
            texts = take(lr.feed(upload(chunk), upload(m.astype(np.int32))))
            fed += m
        texts = take(lr.finish())
        assert texts == whole, max_chunk


# --------------------------------------------------------------------------
# 8. refusals
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_channel_refusals_launch_nothing():
    """-EINVAL for channels_per_row 0, more than 2^31 - 1 channels, a NULL tone_bands, a misaligned row and
    nsamples_all beyond the stride; -ENOTSUP for 0.5 baud; nothing launched."""
    t = torch()
    L = mm().lib()
    x = t.zeros((2, 4096), dtype=t.float32).to(dev())
    fr = t.zeros((4, 16, 5), dtype=t.int32).to(dev())
    st = t.zeros((4, mm().STATE_WORDS), dtype=t.int32).to(dev())
    fill = t.zeros((2,), dtype=t.int32).to(dev())
    p = lambda a: C.c_void_p(a.data_ptr())
    slow = mm().RxEngine.for_mode("0.5", 48000)
    eng = mm().RxEngine.for_mode("1200", 48000)
    bands = eng.tone_bands([1200.0] * 4, [2200.0] * 4, device=dev())
    sbands = slow.tone_bands([1000.0] * 4, [1200.0] * 4, device=dev())
    n0 = mm().launch_count()
    with pytest.raises(RuntimeError, match="-95"):
        slow.rx_batch_tones(x, sbands, nsamples=4096, channels_per_row=2)
    for fn in (L.fsk_b200_rx_batch_channels, L.fsk_b200_rx_batch_channels_s16):
        call = lambda ptr, nrows, stride, nall, k, b: fn(eng._e, ptr, nrows, stride, None, nall, k, b, p(fr), 16,
                                                         p(st), None)
        assert call(p(x), 2, 4096, 4096, 0, p(bands)) == -EINVAL
        assert call(p(x), 2, 4096, 4096, 1 << 30, p(bands)) == -EINVAL
        assert call(p(x), 1 << 31, 4096, 4096, 1, p(bands)) == -EINVAL
        assert call(p(x), 2, 4096, 4096, 2, None) == -EINVAL
        assert call(p(x), 2, 4096, 4097, 2, p(bands)) == -EINVAL
        assert call(C.c_void_p(x.data_ptr() + 4), 2, 4096, 4096, 2, p(bands)) == -EINVAL
        assert call(p(x), 2, 4094, 4094, 2, p(bands)) == -EINVAL
    push = L.fsk_b200_stream_push_channels
    assert push(p(x), 2, 4096, p(fill), 0, None, 0, p(st), p(x), 4096, None, 0, None, None) == -EINVAL
    assert push(p(x), 2, 4096, p(fill), 1 << 30, None, 0, p(st), p(x), 4096, None, 0, None, None) == -EINVAL
    assert push(p(x), 2, 4096, None, 2, None, 0, p(st), p(x), 4096, None, 0, None, None) == -EINVAL
    assert mm().launch_count() == n0
