"""Tone-pair channels summed into shared rows (fsk_b200_tx_text_channels, TxEngine.text_channels): every row
against the sum of its channels sent one per row by fsk_b200_tx_text_batch_tones (pinned to the oracle and to
fixed-pair engines by tests/test_gpu_tx_tones.py), lead-ins placed and rows cut to nsamples_out: float32 added
left to right, int16 summed in int32 and saturated.  All 8 mixing instances by construction (int16 / float32,
16-byte and scalar stores, table in shared memory, in global memory, none), k in {1, 2, 3, 6}, disabled
channels first, middle and last; mixed Bell103 duplex lines and an RTTY passband back through
rx_batch_tones(channels_per_row=k) and LiveReceiver; refusals that launch nothing.

Under FSK_B200_EMU=1 (tests/emu) the gpu tests run on the host emulation of the kernel at reduced sizes."""
import ctypes as C

import numpy as np
import pytest

import minimodem_b200 as mm
import orc
from gpudev import dev, emulated, sync, upload
import txorc

torch = pytest.importorskip("torch")


def text_rows(texts):
    stride = max(max((len(t) for t in texts), default=0), 1)
    buf = np.zeros((len(texts), stride), np.uint8)
    for i, t in enumerate(texts):
        buf[i, :len(t)] = np.frombuffer(bytes(t), np.uint8)
    return upload(buf), torch.tensor([len(t) for t in texts], dtype=torch.int32).to(dev())


def expected(te, text, lens, tones, lead, k, nout):
    """(rows [nrows, nout], out_len [nrows*k]) from the tone call, one channel per row"""
    n = text.shape[0]
    a, c = te.text_batch(text, lens, te.new_states(n, dev()), mm.TX_FINAL, tones=tones)
    sync()
    a, c = a.cpu().numpy(), c.cpu().numpy().astype(np.int64)
    chans = np.zeros((n, nout), np.float32 if a.dtype == np.float32 else np.int64)
    for ch in range(n):
        lo = min(int(lead[ch]), nout)
        m = max(0, min(int(c[ch]), nout - lo))
        chans[ch, lo:lo + m] = a[ch, :m]
    nrows = n // k
    if a.dtype == np.float32:
        rows = chans[0::k].copy()
        for j in range(1, k):
            rows = (rows + chans[j::k]).astype(np.float32)              # IEEE float32, left to right
    else:
        rows = np.clip(chans.reshape(nrows, k, nout).sum(axis=1), -32768, 32767).astype(np.int16)
    valid = np.isfinite(tones.cpu().numpy()).all(axis=1) & (tones.cpu().numpy() > 0).all(axis=1)
    out_len = np.where(valid, c + lead, 0)
    return rows, out_len


# ---- 4. mixing, exact --------------------------------------------------------------------------------------------
SHAPES = [(fmt, align, lut) for fmt in ("f32", "s16") for align in ("aligned", "odd-stride") for lut in (0, 4096, 65536)]
BAD = [np.nan, np.inf, 0.0, -300.0]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,align,lut", SHAPES, ids=["%s-%s-lut%d" % s for s in SHAPES])
def test_rows_are_the_sum_of_their_channels(fmt, align, lut):
    """k in {1, 2, 3, 6}: random lead-ins (some past the row), texts that run past nsamples_out and texts that
    stop short, empty texts, disabled channels in first, middle and last position.  Each row equals the sum of
    its channels (== for float32, so signed zeros are equal); out_len per channel; the samples past
    nsamples_out keep their sentinel."""
    float_samples = fmt == "f32"
    rng = np.random.default_rng(300 + SHAPES.index((fmt, align, lut)))
    mode, kw = [("300", {}), ("1200", {}), ("rtty", dict(sample_rate=8000))][SHAPES.index((fmt, align, lut)) % 3]
    rate = kw.get("sample_rate", 48000)
    vol = 1.0 if fmt == "s16" else float(rng.choice([0.3, 1.0]))
    te = mm.TxEngine.for_mode(mode, rate, amplitude=vol, lut=lut, float_samples=float_samples)
    for k in (1, 2, 3, 6):
        nrows = 4 if emulated() else 24
        n = nrows * k
        maxlen = 3 if emulated() else 12
        texts = [bytes(int(x) for x in rng.integers(32, 127, 0 if ch % 5 == 3 else int(rng.integers(1, maxlen + 1))))
                 for ch in range(n)]
        text, lens = text_rows(texts)
        marks = rng.integers(400, rate // 2 - 200, n).astype(np.float32)
        spaces = rng.integers(400, rate // 2 - 200, n).astype(np.float32)
        for r in range(nrows):                          # disabled: first, middle, last, none
            pos = [0, k // 2, k - 1, None][r % 4]
            if pos is not None and k > 1 or (k == 1 and r % 4 == 0):
                spaces[r * k + pos] = BAD[r % len(BAD)]
        tones = upload(np.stack([marks, spaces], axis=1))
        full = te.max_samples(maxlen, mm.TX_FINAL)
        nout = int(rng.integers(full // 3, full + 1)) | (1 if align == "odd-stride" else 0)
        lead = rng.integers(0, nout // 2, n).astype(np.int32)
        lead[rng.integers(0, n, max(1, n // 8))] = nout + 5      # a channel wholly past its row
        stride = nout + 3 if align == "odd-stride" else ((nout + 7) & ~7) + 8
        if align == "odd-stride" and stride % 2 == 0:
            stride += 1
        sentinel = -5.5 if float_samples else -555
        out = torch.full((nrows, stride), sentinel, dtype=torch.float32 if float_samples else torch.int16, device=dev())
        assert (out.data_ptr() % 16 == 0 and stride * out.element_size() % 16 == 0) == (align == "aligned")
        lead_t = upload(lead)
        _, cnt = te.text_channels(text, lens, tones, k, nout, lead_in=lead_t, out=out)
        sync()
        want, want_len = expected(te, text, lens, tones, lead, k, nout)
        got = out.cpu().numpy()
        assert np.array_equal(cnt.cpu().numpy(), want_len), (k, cnt.cpu().numpy(), want_len)
        for r in range(nrows):
            assert (got[r, :nout] == want[r]).all(), (fmt, align, lut, k, r)
            assert (got[r, nout:] == sentinel).all(), (k, r, "wrote past nsamples_out")


@pytest.mark.gpu
def test_int16_rows_saturate_the_exact_sum():
    """Six channels of the same text, pair and lead-in at full volume: the int32 sum is six times the signal,
    saturated; with one of them inverted the sum stays in range and is exact (a saturating running sum
    would not be)."""
    te = mm.TxEngine.for_mode("1200", 48000, amplitude=1.0, lut=4096, float_samples=False)
    k, nrows = 6, 2
    texts = [b"SATURATE"] * (k * nrows)
    text, lens = text_rows(texts)
    pairs = np.tile(np.array([[1200.0, 2200.0]], np.float32), (k * nrows, 1))
    pairs[k + 2] = [2200.0, 1200.0]                     # row 1: one channel with the tones swapped
    tones = upload(pairs)
    nout = te.max_samples(len(texts[0]), mm.TX_FINAL)
    lead = np.zeros(k * nrows, np.int32)
    rows, _ = te.text_channels(text, lens, tones, k, nout)
    sync()
    want, _ = expected(te, text, lens, tones, lead, k, nout)
    got = rows.cpu().numpy()[:, :nout]
    assert np.array_equal(got, want)
    assert (got[0] == 32767).any() and (got[0] == -32768).any()


@pytest.mark.gpu
def test_one_channel_is_the_tone_call():
    """k = 1 and no lead-ins: each row is text_batch_tones with FSK_B200_TX_FINAL on a fresh state, padded
    with zeros to nsamples_out (and cut there)."""
    rng = np.random.default_rng(5)
    te = mm.TxEngine.for_mode("300", 48000, float_samples=True)
    n = 4 if emulated() else 64
    texts = [bytes(int(x) for x in rng.integers(32, 127, int(rng.integers(0, 6)))) for _ in range(n)]
    text, lens = text_rows(texts)
    tones = te.tone_pairs(rng.integers(500, 3000, n), rng.integers(500, 3000, n), device=dev())
    a, c = te.text_batch(text, lens, te.new_states(n, dev()), mm.TX_FINAL, tones=tones)
    nout = int(te.max_samples(text.shape[1], mm.TX_FINAL) * 3 // 4)
    rows, cnt = te.text_channels(text, lens, tones, 1, nout)
    sync()
    a, c, rows = a.cpu().numpy(), c.cpu().numpy(), rows.cpu().numpy()
    assert np.array_equal(cnt.cpu().numpy(), c)
    for s in range(n):
        want = np.zeros(nout, np.float32)
        m = min(int(c[s]), nout)
        want[:m] = a[s, :m]
        assert np.array_equal(rows[s, :nout].view(np.int32), want.view(np.int32)), s


# ---- 5. loopback ----------------------------------------------------------------------------------------------
def baudot_text(t):
    w = txorc.encode("baudot", t)
    return orc.decode_words("baudot", 5, w, resets=[1] + [0] * (len(w) - 1))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("case", ["bell103-duplex", "rtty-passband"])
def test_mixed_rows_decode_back(case, fmt):
    """Bell103 originate (1270/1070) + answer (2225/2025) behind random lead-ins, k = 2, and six RTTY signals
    400 Hz apart at 8 kHz, k = 6 (the last one disabled on odd rows): rx_batch_tones(channels_per_row=k) and
    decode_batch give back the text sent, whole, on at least 90 % of the channels, and
    LiveReceiver(tones=..., channels_per_row=k) fed the rows in chunks decodes exactly what the batch call does.  A disabled channel
    decodes nothing."""
    rng = np.random.default_rng(17 if case == "bell103-duplex" else 19)
    if case == "bell103-duplex":
        mode, rate, k = "300", 48000, 2
        marks, spaces = [1270.0, 2225.0], [1070.0, 2025.0]
    else:
        mode, rate, k = "rtty", 8000, 6
        marks = [800.0 + 400 * j for j in range(k)]
        spaces = [m - 170.0 for m in marks]
    nrows = 2 if emulated() else 48
    n = nrows * k
    te = mm.TxEngine.for_mode(mode, rate, amplitude=1.0 / k, float_samples=fmt == "f32")
    nchar = 5 if emulated() else 24
    texts = [bytes(int(x) for x in rng.integers(65, 91, int(rng.integers(1, nchar + 1)))) for _ in range(n)]
    text, lens = text_rows(texts)
    m = np.tile(np.array(marks, np.float32), nrows)
    s = np.tile(np.array(spaces, np.float32), nrows)
    if case == "rtty-passband":
        s[[r * k + k - 1 for r in range(1, nrows, 2)]] = np.nan
    tones = upload(np.stack([m, s], axis=1))
    lead = upload(rng.integers(0, rate // 4, n).astype(np.int32))
    nout = te.max_samples(text.shape[1], mm.TX_FINAL) + rate // 4 + rate // 2
    rows, _ = te.text_channels(text, lens, tones, k, nout, lead_in=lead)
    rx = mm.RxEngine.for_mode(mode, rate)
    disabled = ~np.isfinite(s)
    bands = rx.tone_bands(m, np.where(disabled, m + 170.0, s), device=dev())
    bands[upload(disabled)] = rx.params.nbands      # disabled on the receive side too
    kind = mm.decoder_for_mode(mode, rx.params.n_data_bits)
    frames, states = rx.rx_batch_tones(rows, bands, channels_per_row=k)
    out, cnt = rx.decode_batch(kind, frames, states)
    sync()
    wants = [b"" if disabled[c] else (baudot_text(t) if mode == "rtty" else t) for c, t in enumerate(texts)]
    got = [bytes(out[c, :int(cnt[c])].cpu().numpy()) for c in range(n)]
    # The mix itself is pinned sample for sample above; this is the receiver on what it makes.  Where the
    # signals overlap, the receiver can take bytes out of another signal around a channel's own transmission,
    # and the odd character in a crowded passband (as the reference CLI does on the same row); the text sent
    # must come back whole on nearly every channel, and a disabled channel decodes nothing.
    whole = sum(1 for c in range(n) if wants[c] and wants[c] in got[c])
    enabled = sum(1 for c in range(n) if wants[c])
    assert whole >= 0.9 * enabled, (case, fmt, whole, enabled)
    assert all(not got[c] for c in range(n) if disabled[c])
    if fmt == "f32":
        live = mm.LiveReceiver(mode, rate, nstreams=nrows, max_chunk=rate // 3, device=dev(), tones=bands,
                               channels_per_row=k)
        parts = [[] for _ in range(n)]
        pos = 0
        while pos < nout:
            w = min(int(rng.integers(rate // 10, rate // 3)), nout - pos)
            t, c = live.feed(rows[:, pos:pos + w].contiguous())
            for ch in range(n):
                parts[ch].append(bytes(t[ch, :int(c[ch])].cpu().numpy()))
            pos += w
        t, c = live.finish()
        for ch in range(n):
            parts[ch].append(bytes(t[ch, :int(c[ch])].cpu().numpy()))
        assert [b"".join(p) for p in parts] == got


# ---- 6. refusals ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_launch_nothing():
    te = mm.TxEngine.for_mode("1200", 48000)
    L = mm.lib()
    nrows, k, stride = 2, 2, 4
    text = torch.zeros((nrows * k, stride), dtype=torch.uint8, device=dev())
    lens = torch.zeros((nrows * k,), dtype=torch.int32, device=dev())
    tones = te.tone_pairs(1300.0, 2100.0, device=dev()).expand(nrows * k, 2).contiguous()
    nout = 1000
    out = torch.zeros((nrows, nout), dtype=torch.int16, device=dev())
    cnt = torch.zeros((nrows * k,), dtype=torch.int32, device=dev())
    p = lambda t: C.c_void_p(t.data_ptr())
    call = L.fsk_b200_tx_text_channels

    def args(**kw):
        a = dict(te=te._te, text=p(text), nrows=nrows, k=k, stride=stride, lens=p(lens), tones=p(tones), lead=None,
                 out=p(out), out_stride=nout, nout=nout, cnt=p(cnt), stream=None)
        a.update(kw)
        return list(a.values())
    before = mm.launch_count()
    for name in ("te", "text", "lens", "tones", "out", "cnt"):
        assert call(*args(**{name: None})) == -22, name
    assert call(*args(k=0)) == -22
    assert call(*args(nrows=(1 << 30), k=2)) == -22                # 2^31 channels
    assert call(*args(nrows=1, k=0xffffffff)) == -22
    assert call(*args(nout=nout + 1)) == -22
    assert call(*args(stride=1 << 32)) == -22
    assert mm.launch_count() == before
    assert call(*args()) == 0
    sync()
    assert mm.launch_count() == before + 1


# ---- CPU: the gpu tests above on the emulated kernel -------------------------------------------------------------
def test_tx_channels_gpu_tests_on_the_emulated_kernel():
    """This file's gpu tests against the emulation build of the same kernel source, at reduced sizes."""
    from gpudev import run_emulated
    tail = run_emulated("", "late", 1500, module="test_gpu_tx_channels.py")
    assert " passed" in tail and "failed" not in tail
