"""The batched transmitter on the device (fsk_b200_tx_text_batch, TxEngine, LiveTransmitter): text in,
the reference's `--tx` audio out, against the audio the reference CLI wrote (golden vectors) and the
oracle's restatement of its transmit loop (tests/txorc.py), and back through the receiver.

Under FSK_B200_EMU=1 (tests/emu) the same tests run on the host emulation of the kernel at reduced
sizes."""
import ctypes as C

import numpy as np
import pytest

import golden_util as gu
import minimodem_b200 as mm
import orc
import refcases
import txorc

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def dev():
    import conftest
    if conftest.EMU_DEVICE is not None:
        return conftest.EMU_DEVICE
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def emulated():
    import conftest
    return conftest.EMU_DEVICE is not None


def sync():
    if not emulated():
        torch.cuda.synchronize()


OVERRIDE_NAMES = dict(mark="f_mark", space="f_space", bandwidth="band_width", startbits="nstartbits",
                      stopbits="nstopbits", confidence="confidence_threshold", limit="confidence_search_limit")


def tx_engine(mode, kw, amplitude=1.0, lut=4096, float_samples=False, ascii=False):
    """TxEngine for orc.Mode(mode, **kw) through the library's presets (rx_config_for_mode ->
    tx_config_from_rx), its config checked against the oracle's restatement of main()."""
    ov = {OVERRIDE_NAMES.get(k, k): v for k, v in kw.items() if k not in ("sample_rate", "baudot")}
    if kw.get("baudot"):
        ov["n_data_bits"] = 5
    rx = mm.rx_config_for_mode(mode, kw.get("sample_rate", 48000), **ov)
    cfg = mm.tx_config_from(rx)
    m = orc.Mode(mode, **kw)
    want = m.tx_config(amplitude, lut, float_samples)
    for f in ("sample_rate", "data_rate", "f_mark", "f_space", "n_data_bits", "nstartbits", "nstopbits",
              "invert_start_stop", "msb_first", "do_tx_sync_bytes", "sync_byte", "leader_bits", "trailer_bits"):
        if f != "sync_byte" or want.do_tx_sync_bytes:
            assert getattr(cfg, f) == getattr(want, f), (mode, f, getattr(cfg, f), getattr(want, f))
    kind = mm.ENCODE_ASCII8 if ascii else mm.encoder_for_mode(mode, rx.n_data_bits)
    return mm.TxEngine(cfg, kind, amplitude, lut, float_samples), m, ("baudot" if kind == mm.ENCODE_BAUDOT else "ascii8")


def as_f32(x):
    """device rows -> float32 numpy, int16 read back as the reference's rx reads it (x / 32768)"""
    a = x.cpu().numpy()
    return a.astype(np.float32) * np.float32(1.0 / 32768.0) if a.dtype == np.int16 else a


def run_rows(te, texts, flags=mm.TX_FINAL, states=None, text_stride=None):
    n = len(texts)
    stride = max(text_stride or 0, max((len(t) for t in texts), default=0), 1)
    buf = np.zeros((n, stride), np.uint8)
    for i, t in enumerate(texts):
        buf[i, :len(t)] = np.frombuffer(bytes(t), np.uint8)
    lens = torch.tensor([len(t) for t in texts], dtype=torch.int32).to(dev())
    if states is None:
        states = te.new_states(n, dev())
    out, cnt = te.text_batch(torch.from_numpy(buf).to(dev()), lens, states, flags)
    sync()
    return out, cnt.cpu().numpy(), states


# ---- 1. every golden vector from its text --------------------------------------------------------
CASES = refcases.EVERY + refcases.MORE


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_vectors_from_text(case):
    g = gu.load(case["name"])
    te, m, kind = tx_engine(case["mode"], case["mkw"], case["amplitude"], case["lut"], case["float_samples"],
                            ascii=case["tx_ascii"])
    text = bytes(g["text"])
    out, cnt, states = run_rows(te, [text, text])
    a = as_f32(out)
    assert cnt[0] == cnt[1] == int(g["audio_len"][0])
    st = states.cpu().numpy()
    assert (st[:, 8:12].view(np.uint32) == 0).all()          # transmitting = 0 after the trailer
    if case["lut"] > 0:
        for r in range(2):
            assert gu.sha(a[r, :cnt[r]]) == bytes(g["audio_sha256"]), (case["name"], r)
        return
    # --lut=0: sin() in double precision against glibc's sinf: 1 ulp (float) / 1 LSB (int16)
    want = txorc.tx_events(m, list(text), kind, case["amplitude"], 0, case["float_samples"])
    assert gu.sha(want) == bytes(g["audio_sha256"])
    got = a[0, :cnt[0]]
    if case["float_samples"]:
        ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        ulps[(got == 0) & (want == 0)] = 0
        diff = int(np.count_nonzero(ulps))
        print("%s: %d of %d float samples differ from the reference, at most %d ulp"
              % (case["name"], diff, got.size, int(ulps.max())))
        assert ulps.max() <= 1
    else:
        lsb = np.abs(np.round(got * 32768.0) - np.round(want * 32768.0))
        print("%s: %d of %d int16 samples differ from the reference, at most %d LSB"
              % (case["name"], int(np.count_nonzero(lsb)), got.size, int(lsb.max())))
        assert lsb.max() <= 1


# ---- 2. a ragged batch ---------------------------------------------------------------------------
RAGGED = [("1200", {}, 400), ("300", {}, 400), ("rtty", dict(sample_rate=8000), 400), ("tdd", {}, 400),
          ("same", {}, 400), ("callerid", {}, 400), ("0.5", {}, 1),
          ("1200", dict(startbits=2, stopbits=3.0), 400), ("1200", dict(stopbits=1.5), 400)]


@pytest.mark.parametrize("fmt", ["float", "int16"])
def test_ragged_batch(fmt):
    """4096 streams (64 emulated), text lengths 0..400 with zeros among them, over nine framings; every
    row equal to the oracle's transmitter, empty rows write nothing."""
    rng = np.random.default_rng(23)
    per = 8 if emulated() else 4096 // len(RAGGED) + 1
    for mode, kw, maxlen in RAGGED:
        if emulated() and mode == "0.5":
            continue                                                # 1.3 M samples a byte: too long emulated
        te, m, kind = tx_engine(mode, kw, float_samples=(fmt == "float"))
        texts = []
        for i in range(per):
            n = 0 if i % 7 == 0 else int(rng.integers(0, maxlen + 1) if i % 16 == 1 else rng.integers(0, min(maxlen, 40) + 1))
            if emulated():
                n = min(n, 70)
            texts.append(bytes(int(x) for x in rng.integers(1, 256 if i % 3 == 0 else 127, n)))
        n = len(texts)
        stride = max(len(t) for t in texts)
        out = torch.full((n, (te.max_samples(stride, mm.TX_FINAL) + 7) & ~7), 7,
                         dtype=torch.float32 if fmt == "float" else torch.int16, device=dev())
        buf = np.zeros((n, stride), np.uint8)
        for i, t in enumerate(texts):
            buf[i, :len(t)] = np.frombuffer(t, np.uint8)
        lens = torch.tensor([len(t) for t in texts], dtype=torch.int32).to(dev())
        _, cnt = te.text_batch(torch.from_numpy(buf).to(dev()), lens, te.new_states(n, dev()), mm.TX_FINAL, out=out)
        sync()
        cnt = cnt.cpu().numpy()
        a = as_f32(out)
        for i, t in enumerate(texts):
            want = txorc.tx_events(m, list(t), kind, 1.0, 4096, fmt == "float")
            assert cnt[i] == want.size, (mode, kw, i, cnt[i], want.size)
            assert np.array_equal(a[i, :cnt[i]], want), (mode, kw, i)
            if orc.have_ref() and len(t) and kind == "ascii8":
                # the reference's own encoder (stateless for ascii8) + the oracle's word-level transmitter
                assert np.array_equal(want, orc.tx_words(m, orc.ref_encode("ascii8", t), 1.0, 4096, fmt == "float"))
            if not len(t):
                fill = np.float32(7) if fmt == "float" else np.float32(7 / 32768)
                assert (a[i] == fill).all(), (mode, i)           # nothing written


# ---- 3. cut invariance, idle ticks -----------------------------------------------------------------------
@pytest.mark.parametrize("mode,kw", [("rtty", dict(sample_rate=8000)), ("same", {}), ("1200", {})])
def test_live_transmitter_cuts(mode, kw):
    """The same texts fed through LiveTransmitter in random cuts equal one call; with empty ticks (idle
    tone, preamble again on the next byte) they equal the oracle's transmitter with idle events."""
    rng = np.random.default_rng(31)
    n = 6 if emulated() else 256
    maxlen = 70 if emulated() else 120
    texts = [bytes(int(x) for x in rng.integers(32, 127, int(rng.integers(1, maxlen)))) for _ in range(n)]
    te, m, kind = tx_engine(mode, kw)
    whole, wcnt, _ = run_rows(te, texts)
    whole = as_f32(whole)
    for idle in (False, True):
        tx = mm.LiveTransmitter(mode, kw.get("sample_rate", 48000), nstreams=n, max_text=16, idle=idle,
                                device=dev(), **{OVERRIDE_NAMES.get(k, k): v for k, v in kw.items() if k != "sample_rate"})
        pos = [0] * n
        parts = [[] for _ in range(n)]
        events = [[] for _ in range(n)]
        while any(p < len(t) for p, t in zip(pos, texts)):
            buf = np.zeros((n, 16), np.uint8)
            lens = np.zeros(n, np.int32)
            for s in range(n):
                k = int(rng.integers(0 if idle else 1, 17))
                k = min(k, len(texts[s]) - pos[s])
                buf[s, :k] = np.frombuffer(texts[s][pos[s]:pos[s] + k], np.uint8)
                lens[s] = k
                if k:
                    events[s].extend(texts[s][pos[s]:pos[s] + k])
                elif idle:
                    events[s].append(txorc.IDLE)
                pos[s] += k
            audio, cnt = tx.feed(torch.from_numpy(buf).to(dev()), torch.from_numpy(lens).to(dev()))
            sync()
            a, c = as_f32(audio), cnt.cpu().numpy()
            for s in range(n):
                parts[s].append(a[s, :c[s]])
        audio, cnt = tx.finish()
        sync()
        a, c = as_f32(audio), cnt.cpu().numpy()
        for s in range(n):
            got = np.concatenate(parts[s] + [a[s, :c[s]]])
            if not idle:
                assert np.array_equal(got, whole[s, :wcnt[s]]), (mode, s)
            else:
                want = txorc.tx_events(m, events[s], kind)
                assert np.array_equal(got, want), (mode, s, got.size, want.size)


# ---- 4. loopback ------------------------------------------------------------------------------------------
LOOP = [("rtty", dict(sample_rate=8000)), ("tdd", {}), ("same", {}), ("callerid", {}), ("1200", {})]


@pytest.mark.parametrize("fmt", ["float", "int16"])
@pytest.mark.parametrize("mode,kw", LOOP, ids=[m for m, _ in LOOP])
def test_loopback_through_the_receiver(mode, kw, fmt):
    sr = kw.get("sample_rate", 48000)
    n = 2 if emulated() else 64
    rng = np.random.default_rng(41)
    if mode == "callerid":
        g = gu.load("70-callerid-mdmf")
        texts, wants = [bytes(g["text"])] * n, [bytes(g["stdout"])] * n
    else:
        texts = [bytes(int(x) for x in rng.integers(32, 127, 8 if emulated() else int(rng.integers(10, 60))))
                 for _ in range(n)]
        wants = list(texts)
    tx = mm.LiveTransmitter(mode, sr, nstreams=n, max_text=max(len(t) for t in texts), float_samples=(fmt == "float"),
                            idle=False, device=dev())
    kind = tx.engine.encoder
    if kind == mm.ENCODE_BAUDOT:                                   # upper case, non-encodables dropped
        wants = []
        for t in texts:
            w = txorc.encode("baudot", t)
            wants.append(orc.decode_words("baudot", 5, w, resets=[1] + [0] * (len(w) - 1)))
    buf = np.zeros((n, max(len(t) for t in texts)), np.uint8)
    for i, t in enumerate(texts):
        buf[i, :len(t)] = np.frombuffer(t, np.uint8)
    lens = torch.tensor([len(t) for t in texts], dtype=torch.int32).to(dev())
    a1, c1 = tx.feed(torch.from_numpy(buf).to(dev()), lens)
    a2, c2 = tx.finish()
    sync()
    c1, c2 = c1.cpu().numpy(), c2.cpu().numpy()
    total = int((c1 + c2).max())
    pad = int(sr)                                                   # a second of silence behind every stream
    rows = torch.zeros((n, (total + pad + 7) & ~7), dtype=a1.dtype, device=dev())
    for s in range(n):
        rows[s, :c1[s]] = a1[s, :c1[s]]
        rows[s, c1[s]:c1[s] + c2[s]] = a2[s, :c2[s]]
    rx_mode = "callerid" if mode == "callerid" else mode
    if fmt == "float":
        rx = mm.LiveReceiver(rx_mode, sr, nstreams=n, max_chunk=rows.shape[1], device=dev())
        t1, n1 = rx.feed(rows)
        t2, n2 = rx.finish()
        sync()
        got = [bytes(t1[s, :int(n1[s])].cpu().numpy()) + bytes(t2[s, :int(n2[s])].cpu().numpy()) for s in range(n)]
    else:
        eng = mm.RxEngine.for_mode(rx_mode, sr)
        frames, states = eng.rx_batch(rows)                          # int16 rows: fsk_b200_rx_batch_s16
        dec = mm.decoder_for_mode(rx_mode, eng.params.n_data_bits)
        out, cnt = eng.decode_batch(dec, frames, states)
        sync()
        got = [bytes(out[s, :int(cnt[s])].cpu().numpy()) for s in range(n)]
    for s in range(n):
        assert got[s] == wants[s], (mode, fmt, s, got[s][:60], wants[s][:60])


# ---- 5. errors ---------------------------------------------------------------------------------------------
def test_errors_launch_nothing():
    te, m, kind = tx_engine("1200", {})
    L = mm.lib()
    n, stride = 4, 16
    text = torch.zeros((n, stride), dtype=torch.uint8, device=dev())
    lens = torch.zeros((n,), dtype=torch.int32, device=dev())
    states = te.new_states(n, dev())
    need = te.max_samples(stride, mm.TX_FINAL)
    out = torch.zeros((n, need), dtype=torch.int16, device=dev())
    cnt = torch.zeros((n,), dtype=torch.int32, device=dev())
    p = lambda t: C.c_void_p(t.data_ptr())
    before = mm.launch_count()
    assert L.fsk_b200_tx_text_batch(te._te, p(text), n, stride, p(lens), mm.TX_FINAL, p(states), p(out),
                                    need - 1, p(cnt), None) == -22
    assert L.fsk_b200_tx_text_batch(te._te, None, n, stride, p(lens), mm.TX_FINAL, p(states), p(out),
                                    need, p(cnt), None) == -22
    assert L.fsk_b200_tx_text_batch(te._te, p(text), n, stride, None, mm.TX_FINAL, p(states), p(out),
                                    need, p(cnt), None) == -22
    assert L.fsk_b200_tx_text_batch(te._te, p(text), n, stride, p(lens), mm.TX_FINAL, None, p(out),
                                    need, p(cnt), None) == -22
    assert L.fsk_b200_tx_text_batch(None, p(text), n, stride, p(lens), mm.TX_FINAL, p(states), p(out),
                                    need, p(cnt), None) == -22
    assert mm.launch_count() == before
    cfg = mm.tx_config_from(mm.rx_config_for_mode("1200"))
    cfg.n_data_bits = 33
    assert not L.fsk_b200_tx_engine_new(C.byref(cfg), C.byref(mm.TxSignal(1.0, 4096, 0)), 0)
    with pytest.raises(RuntimeError):
        mm.TxEngine(cfg)
    assert L.fsk_b200_tx_text_batch(te._te, p(text), n, stride, p(lens), mm.TX_FINAL, p(states), p(out),
                                    need, p(cnt), None) == 0
    sync()
    assert mm.launch_count() == before + 1
