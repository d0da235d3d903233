"""The batched transmitter with a tone pair per stream (fsk_b200_tx_text_batch_tones, TxEngine.text_batch(...,
tones=...), LiveTransmitter(tones=...)): each stream against the oracle's transmitter for a mode with that
pair (tests/txorc.py) and against fsk_b200_tx_text_batch on an engine built for that pair, byte for byte,
over random framings, every k_tx_synth shape (int16 / float32, 16-byte and scalar stores, table in shared
memory, in global memory, none), ragged ticks, pairs changed between ticks and invalid pairs.  The CPU test
pins the oracle to the reference CLI's `--tx -M m -S s [--inverted]` at pairs no golden vector uses.

Under FSK_B200_EMU=1 (tests/emu) the gpu tests run on the host emulation of the kernel at reduced sizes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import minimodem_b200 as mm
import orc
from gpudev import dev, emulated, sync, upload
import txorc

torch = pytest.importorskip("torch")

F32 = np.float32


NAMES = dict(mark="f_mark", space="f_space", startbits="nstartbits", stopbits="nstopbits")


def random_framing(rng):
    """a preset mode (300, 1200, rtty, tdd, same) or a random rate / baud / framing, as the instantiation
    tests draw them: 1..32 data bits, 0..2 start bits, 0 / 1 / 1.5 / 2 stop bits, bit order, start/stop
    inversion.  Returns (mode, kw, baudot)."""
    pick = int(rng.integers(0, 7))
    if pick < 5:
        mode = ["300", "1200", "rtty", "tdd", "same"][pick]
        kw = dict(sample_rate=8000 if mode == "rtty" else 48000)
        if mode in ("300", "1200") and rng.integers(0, 2):
            kw.update(n_data_bits=int(rng.choice([7, 8])), invert_start_stop=bool(rng.integers(0, 2)),
                      msb_first=bool(rng.integers(0, 2)), stopbits=float(rng.choice([1.0, 1.5, 2.0])))
        return mode, kw, mode in ("rtty", "tdd")
    while True:
        baud = int(rng.choice([45, 110, 300, 600, 1200, 2400]))
        rate = int(rng.choice([8000, 11025, 22050, 48000]))
        if 4 <= rate / baud <= 400:
            break
    kw = dict(sample_rate=rate, n_data_bits=int(rng.integers(1, 33)), startbits=int(rng.choice([0, 1, 2])),
              stopbits=float(rng.choice([0.0, 1.0, 1.5, 2.0])), msb_first=bool(rng.integers(0, 2)),
              invert_start_stop=bool(rng.integers(0, 2)))
    return str(baud), kw, bool(rng.integers(0, 2) and kw["n_data_bits"] == 5)


def base_config(mode, kw):
    rx = mm.rx_config_for_mode(mode, kw["sample_rate"], **{NAMES.get(k, k): v for k, v in kw.items()
                                                          if k != "sample_rate"})
    return mm.tx_config_from(rx)


def engine(mode, kw, baudot, pair=None, vol=1.0, lut=4096, float_samples=False):
    """a TxEngine for the framing, built for `pair` = (mark Hz, space Hz) when given"""
    cfg = base_config(mode, kw)
    if pair is not None:
        cfg.f_mark, cfg.f_space = F32(pair[0]), F32(pair[1])
    return mm.TxEngine(cfg, mm.ENCODE_BAUDOT if baudot else mm.ENCODE_ASCII8, vol, lut, float_samples)


def oracle_mode(mode, kw, pair):
    """orc.Mode of the framing with its tone pair replaced (the CLI's -M / -S, after --inverted)"""
    m = orc.Mode(mode, **kw)
    m.mark_f, m.space_f = F32(pair[0]), F32(pair[1])
    return m


def random_pairs(rng, n, rate):
    """n valid pairs below Nyquist, about a third of them swapped (--inverted)"""
    hi = max(rate // 2 - 100, 400)
    marks = rng.integers(300, hi, n).astype(np.float32) + F32(0.25) * rng.integers(0, 4, n).astype(np.float32)
    spaces = rng.integers(300, hi, n).astype(np.float32)
    inv = rng.integers(0, 3, n) == 0
    return marks, spaces, inv


def text_rows(texts, stride=None):
    stride = max(stride or 0, max((len(t) for t in texts), default=0), 1)
    buf = np.zeros((len(texts), stride), np.uint8)
    for i, t in enumerate(texts):
        buf[i, :len(t)] = np.frombuffer(bytes(t), np.uint8)
    lens = torch.tensor([len(t) for t in texts], dtype=torch.int32).to(dev())
    return upload(buf), lens


def as_f32(a):
    return a.astype(np.float32) * F32(1 / 32768) if a.dtype == np.int16 else a


# ---- 1. a pair per stream, bit for bit ---------------------------------------------------------------------------
SHAPES = [(fmt, align, lut) for fmt in ("f32", "s16") for align in ("aligned", "odd-stride") for lut in (0, 4096, 65536)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,align,lut", SHAPES, ids=["%s-%s-lut%d" % s for s in SHAPES])
def test_pairs_per_stream_bit_for_bit(fmt, align, lut):
    """Random framings, every stream on its own random pair (some swapped): each row and state equals
    fsk_b200_tx_text_batch on an engine built for that pair, byte for byte, and the oracle's transmitter
    (bit-exact with a table; with --lut=0 within 1 ulp, 2 at a volume other than 1, or 1 LSB, as the
    fixed-pair tests allow); nothing is
    written past a row's count."""
    float_samples = fmt == "f32"
    dtype = torch.float32 if float_samples else torch.int16
    sentinel = -7.25 if float_samples else -7777
    nconf = 2 if emulated() else 4
    for c in range(nconf):
        seed = 900 + 100 * SHAPES.index((fmt, align, lut)) + c
        rng = np.random.default_rng(seed)
        mode, kw, baudot = random_framing(rng)
        vol = float(rng.choice([1e-5, 0.3, 1.0, 1.7]))
        n = 5 if emulated() else 12
        maxlen = 4 if emulated() else 12
        texts = [bytes(int(x) for x in rng.integers(1, 256, 0 if i == 2 else int(rng.integers(1, maxlen + 1))))
                 for i in range(n)]
        marks, spaces, inv = random_pairs(rng, n, kw["sample_rate"])
        te = engine(mode, kw, baudot, vol=vol, lut=lut, float_samples=float_samples)
        tones = te.tone_pairs(marks, spaces, inv, device=dev())
        pairs = tones.cpu().numpy()
        text, lens = text_rows(texts)
        flags = int(rng.choice([0, mm.TX_FINAL, mm.TX_IDLE_IF_EMPTY | mm.TX_FINAL]))
        need = te.max_samples(text.shape[1], flags)
        stride = need | 1 if align == "odd-stride" else (need + 7) & ~7
        out = torch.full((n, stride), sentinel, dtype=dtype, device=dev())
        states = te.new_states(n, dev())
        _, cnt = te.text_batch(text, lens, states, flags, out=out, tones=tones)
        sync()
        got, cnt, st = out.cpu().numpy(), cnt.cpu().numpy(), states.cpu().numpy()
        for s in range(n):
            pair = tuple(pairs[s])
            assert pair == ((spaces[s], marks[s]) if inv[s] else (marks[s], spaces[s]))
            fixed = engine(mode, kw, baudot, pair, vol, lut, float_samples)
            fout = torch.full((1, stride), sentinel, dtype=dtype, device=dev())
            fst = fixed.new_states(1, dev())
            _, fcnt = fixed.text_batch(text[s:s + 1].contiguous(), lens[s:s + 1].contiguous(), fst, flags, out=fout)
            sync()
            assert int(fcnt[0]) == cnt[s], (mode, kw, s)
            assert np.array_equal(fout.cpu().numpy()[0].view(np.uint8), got[s].view(np.uint8)), (mode, kw, pair, s)
            assert np.array_equal(fst.cpu().numpy()[0], st[s]), (mode, kw, pair, s)
            assert (got[s, cnt[s]:] == sentinel).all(), (mode, kw, s, "wrote past its count")
            events = list(texts[s]) + ([txorc.IDLE] if not texts[s] and flags & mm.TX_IDLE_IF_EMPTY else [])
            if not flags & mm.TX_FINAL:
                continue                                # the oracle always ends with the trailer
            want = txorc.tx_events(oracle_mode(mode, kw, pair), events, "baudot" if baudot else "ascii8",
                                   vol, lut, float_samples)
            row = as_f32(got[s, :cnt[s]])
            assert row.size == want.size, (mode, kw, pair, s, row.size, want.size)
            if lut:
                assert np.array_equal(row, want), (mode, kw, pair, s)
            elif float_samples:
                ulps = np.abs(row.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
                ulps[(row == 0) & (want == 0)] = 0
                # the sine within 1 ulp; at a volume other than 1 the product is rounded once more
                assert ulps.max(initial=0) <= (1 if vol == 1.0 else 2), (mode, kw, vol, pair, s)
            else:
                assert np.abs(np.round(row * 32768) - np.round(want * 32768)).max(initial=0) <= 1, (mode, kw, pair, s)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_the_engines_own_pair_equals_text_batch(fmt):
    """Every stream on the engine's own pair: rows, counts and states equal fsk_b200_tx_text_batch's."""
    rng = np.random.default_rng(77)
    te = engine("1200", dict(sample_rate=48000), False, float_samples=fmt == "f32")
    n = 6 if emulated() else 300
    texts = [bytes(int(x) for x in rng.integers(32, 127, int(rng.integers(0, 20)))) for _ in range(n)]
    text, lens = text_rows(texts)
    tones = te.tone_pairs(te.cfg.f_mark, te.cfg.f_space, device=dev()).expand(n, 2).contiguous()
    sa, sb = te.new_states(n, dev()), te.new_states(n, dev())
    a, ca = te.text_batch(text, lens, sa, mm.TX_FINAL)
    b, cb = te.text_batch(text, lens, sb, mm.TX_FINAL, tones=tones)
    sync()
    assert torch.equal(ca, cb) and torch.equal(sa, sb)
    for s in range(n):
        assert torch.equal(a[s, :int(ca[s])], b[s, :int(cb[s])]), s


# ---- 2. ticks and pair changes --------------------------------------------------------------------------------
def cut(rng, texts, width, idle):
    """texts cut into ragged ticks of at most `width` bytes (empty ticks too when idle)"""
    pos, ticks = [0] * len(texts), []
    while any(p < len(t) for p, t in zip(pos, texts)):
        tick = []
        for s, t in enumerate(texts):
            k = min(int(rng.integers(0 if idle else 1, width + 1)), len(t) - pos[s])
            tick.append(t[pos[s]:pos[s] + k])
            pos[s] += k
        ticks.append(tick)
    return ticks


@pytest.mark.gpu
@pytest.mark.parametrize("mode,kw", [("rtty", dict(sample_rate=8000)), ("300", {}), ("same", {})])
def test_ticks_and_pair_changes(mode, kw):
    """A text cut into ragged ticks (FSK_B200_TX_IDLE_IF_EMPTY, then FSK_B200_TX_FINAL) with a fixed pair per
    stream equals one call with FSK_B200_TX_FINAL when no tick is empty.  With streams moved to another pair
    between ticks, every tick equals the fixed-pair engines of that tick chained through the same states, and
    LiveTransmitter(tones=...) with the pairs written into its tensor between feeds gives the same audio."""
    kw = dict(kw, sample_rate=kw.get("sample_rate", 48000))
    baudot = mode == "rtty"
    rng = np.random.default_rng(55)
    n = 4 if emulated() else 24
    maxlen = 10 if emulated() else 60
    width = 4 if emulated() else 16
    texts = [bytes(int(x) for x in rng.integers(32, 127, int(rng.integers(1, maxlen)))) for _ in range(n)]
    te = engine(mode, kw, baudot)
    marks, spaces, inv = random_pairs(rng, n, kw["sample_rate"])
    tones = te.tone_pairs(marks, spaces, inv, device=dev())
    # fixed pair, no empty ticks: equal to one call
    text, lens = text_rows(texts)
    whole, wcnt = te.text_batch(text, lens, te.new_states(n, dev()), mm.TX_FINAL, tones=tones)
    sync()
    whole, wcnt = whole.cpu().numpy(), wcnt.cpu().numpy()
    states = te.new_states(n, dev())
    parts = [[] for _ in range(n)]
    ticks = cut(rng, texts, width, idle=False)
    for i, tick in enumerate(ticks + [[b""] * n]):
        flags = mm.TX_FINAL if i == len(ticks) else 0
        t, l = text_rows(tick, width)
        a, c = te.text_batch(t, l, states, flags, tones=tones)
        sync()
        a, c = a.cpu().numpy(), c.cpu().numpy()
        for s in range(n):
            parts[s].append(a[s, :c[s]])
    for s in range(n):
        assert np.array_equal(np.concatenate(parts[s]), whole[s, :wcnt[s]]), (mode, s)

    # pairs that change between ticks, idle ticks among them
    ticks = cut(rng, texts, width, idle=True)
    nt = len(ticks) + 1
    all_pairs = []
    for i in range(nt):
        m2, s2, i2 = random_pairs(rng, n, kw["sample_rate"])
        keep = rng.integers(0, 2, n) == 0
        m2, s2, i2 = np.where(keep, marks, m2), np.where(keep, spaces, s2), np.where(keep, inv, i2)
        all_pairs.append(te.tone_pairs(m2, s2, i2, device=dev()))
    live_tones = all_pairs[0].clone()
    tx = mm.LiveTransmitter(mode, kw["sample_rate"], nstreams=n, max_text=width, idle=True, device=dev(),
                            tones=live_tones, **{NAMES.get(k, k): v for k, v in kw.items() if k != "sample_rate"})
    states = te.new_states(n, dev())
    chained = [te.new_states(1, dev()) for _ in range(n)]
    engines = {}
    for i in range(nt):
        final = i == len(ticks)
        tick = [b""] * n if final else ticks[i]
        flags = mm.TX_FINAL if final else mm.TX_IDLE_IF_EMPTY
        t, l = text_rows(tick, width)
        a, c = te.text_batch(t, l, states, flags, tones=all_pairs[i])
        live_tones.copy_(all_pairs[i])
        la, lc = tx.finish() if final else tx.feed(t, l)
        sync()
        a, c, la, lc = a.cpu().numpy(), c.cpu().numpy(), la.cpu().numpy(), lc.cpu().numpy()
        pairs = all_pairs[i].cpu().numpy()
        for s in range(n):
            pair = tuple(float(x) for x in pairs[s])
            if pair not in engines:
                engines[pair] = engine(mode, kw, baudot, pair)
            fa, fc = engines[pair].text_batch(t[s:s + 1].contiguous(), l[s:s + 1].contiguous(), chained[s], flags)
            sync()
            fc = int(fc[0])
            assert fc == c[s] == lc[s], (mode, i, s, fc, c[s], lc[s])
            assert np.array_equal(fa.cpu().numpy()[0, :fc], a[s, :c[s]]), (mode, i, s, pair)
            assert np.array_equal(la[s, :lc[s]], a[s, :c[s]]), (mode, i, s)
    st = states.cpu().numpy()
    for s in range(n):
        assert np.array_equal(chained[s].cpu().numpy()[0], st[s]), s
    assert torch.equal(tx.states.cpu(), states.cpu())


# ---- 3. invalid pairs -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_invalid_pairs_are_skipped(fmt):
    """A pair with a NaN, an infinity, 0 or a negative frequency: out_len 0, the row and the state keep their
    sentinels; the streams around it are sent as with their own pairs."""
    float_samples = fmt == "f32"
    te = engine("1200", dict(sample_rate=48000), False, float_samples=float_samples)
    bad = [(np.nan, 2200.0), (1200.0, np.nan), (np.inf, 2200.0), (1200.0, -np.inf), (0.0, 2200.0),
           (1200.0, 0.0), (-1200.0, 2200.0), (1200.0, -1.0)]
    good = (1300.0, 2100.0)
    pairs = []
    for b in bad:
        pairs += [good, b]
    pairs.append(good)
    n = len(pairs)
    tones = torch.tensor(pairs, dtype=torch.float32).to(dev())
    texts = [b"pair %d" % i for i in range(n)]
    text, lens = text_rows(texts)
    sentinel = -3.5 if float_samples else -333
    need = te.max_samples(text.shape[1], mm.TX_FINAL)
    out = torch.full((n, need), sentinel, dtype=torch.float32 if float_samples else torch.int16, device=dev())
    states = torch.full((n, mm.TX_STATE_BYTES), 0xA5, dtype=torch.uint8, device=dev())
    states[0::2] = 0
    cnt = torch.full((n,), 12345, dtype=torch.int32, device=dev())
    te.text_batch(text, lens, states, mm.TX_FINAL, out=out, out_len=cnt, tones=tones)
    sync()
    o, st, c = out.cpu().numpy(), states.cpu().numpy(), cnt.cpu().numpy()
    fixed = engine("1200", dict(sample_rate=48000), False, good, float_samples=float_samples)
    for s in range(n):
        if s % 2:
            assert c[s] == 0 and (o[s] == sentinel).all() and (st[s] == 0xA5).all(), (s, pairs[s])
            continue
        fa, fc = fixed.text_batch(text[s:s + 1].contiguous(), lens[s:s + 1].contiguous(), fixed.new_states(1, dev()),
                                  mm.TX_FINAL)
        sync()
        assert c[s] == int(fc[0]) and np.array_equal(o[s, :c[s]], fa.cpu().numpy()[0, :c[s]]), s
        assert (o[s, c[s]:] == sentinel).all(), s


# ---- 4. loopback ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_bell103_originate_and_answer_in_one_call_loop_back(fmt):
    """Bell103 originate (1270/1070) and answer (2225/2025) streams sent in one call and decoded by
    rx_batch_tones with the same pairs give back their text."""
    rng = np.random.default_rng(8)
    n = 2 if emulated() else 64
    te = engine("300", dict(sample_rate=48000), False, float_samples=fmt == "f32")
    ans = np.arange(n) % 2 == 1
    marks = np.where(ans, 2225.0, 1270.0)
    spaces = np.where(ans, 2025.0, 1070.0)
    texts = [bytes(int(x) for x in rng.integers(32, 127, 6 if emulated() else int(rng.integers(10, 40))))
             for _ in range(n)]
    text, lens = text_rows(texts)
    audio, cnt = te.text_batch(text, lens, te.new_states(n, dev()), mm.TX_FINAL,
                               tones=te.tone_pairs(marks, spaces, device=dev()))
    sync()
    c = cnt.cpu().numpy()
    pad = 48000 // 2
    rows = torch.zeros((n, (int(c.max()) + pad + 7) & ~7), dtype=audio.dtype, device=dev())
    for s in range(n):
        rows[s, :c[s]] = audio[s, :c[s]]
    rx = mm.RxEngine.for_mode("300", 48000)
    bands = rx.tone_bands(marks, spaces, device=dev())
    frames, states = rx.rx_batch_tones(rows, bands)
    out, oc = rx.decode_batch(mm.decoder_for_mode("300", rx.params.n_data_bits), frames, states)
    sync()
    for s in range(n):
        assert bytes(out[s, :int(oc[s])].cpu().numpy()) == texts[s], s


# ---- 5. refusals ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_launch_nothing():
    te = engine("1200", dict(sample_rate=48000), False)
    L = mm.lib()
    n, stride = 4, 16
    text = torch.zeros((n, stride), dtype=torch.uint8, device=dev())
    lens = torch.zeros((n,), dtype=torch.int32, device=dev())
    tones = te.tone_pairs(1300.0, 2100.0, device=dev()).expand(n, 2).contiguous()
    states = te.new_states(n, dev())
    need = te.max_samples(stride, mm.TX_FINAL)
    out = torch.zeros((n, need), dtype=torch.int16, device=dev())
    cnt = torch.zeros((n,), dtype=torch.int32, device=dev())
    p = lambda t: C.c_void_p(t.data_ptr())
    call = L.fsk_b200_tx_text_batch_tones
    before = mm.launch_count()
    assert call(te._te, p(text), n, stride, p(lens), None, mm.TX_FINAL, p(states), p(out), need, p(cnt), None) == -22
    assert call(te._te, p(text), n, stride, p(lens), p(tones), mm.TX_FINAL, p(states), p(out), need - 1, p(cnt),
                None) == -22
    assert call(te._te, p(text), n, stride, p(lens), p(tones), 4, p(states), p(out), need, p(cnt), None) == -22
    for i in range(6):
        args = [te._te, p(text), n, stride, p(lens), p(tones), mm.TX_FINAL, p(states), p(out), need, p(cnt), None]
        args[[0, 1, 4, 7, 8, 10][i]] = None
        assert call(*args) == -22, i
    assert mm.launch_count() == before
    assert call(te._te, p(text), n, stride, p(lens), p(tones), mm.TX_FINAL, p(states), p(out), need, p(cnt),
                None) == 0
    sync()
    assert mm.launch_count() == before + 1


def test_tone_pairs_refuses_invalid_frequencies():
    """CPU: TxEngine.tone_pairs raises ValueError for a frequency that is not finite or not > 0, and swaps
    the inverted pairs."""
    dv = torch.device("cpu")
    for m, s in ((np.nan, 1000.0), (1000.0, np.inf), (0.0, 1000.0), (1000.0, -5.0)):
        with pytest.raises(ValueError):
            mm.TxEngine.tone_pairs([1200.0, m], [2200.0, s], device=dv)
    t = mm.TxEngine.tone_pairs([1270.0, 2225.0], [1070.0, 2025.0], [False, True], device=dv).cpu().numpy()
    assert t.dtype == np.float32 and t.tolist() == [[1270.0, 1070.0], [2025.0, 2225.0]]


# ---- 6. CPU: the oracle against the reference CLI at new pairs ------------------------------------------------
CLI_MODES = [("1200", 48000), ("300", 48000), ("rtty", 8000), ("600", 22050)]


@pytest.mark.ref
@pytest.mark.parametrize("flt", [False, True], ids=["int16", "float"])
def test_tx_oracle_matches_the_reference_cli_at_random_pairs(flt, tmp_path):
    """The oracle's transmitter against the unmodified reference CLI's `--tx -M m -S s [--inverted]`, by hash,
    on a dozen random pairs that no preset and no golden vector uses."""
    import hashlib
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import read_wav
    rng = np.random.default_rng(2024 + flt)
    for i in range(12):
        mode, rate = CLI_MODES[i % len(CLI_MODES)]
        mark = float(rng.integers(300, rate // 2 - 100)) + float(rng.choice([0.0, 0.5, 0.25]))
        space = float(rng.integers(300, rate // 2 - 100))
        inv = bool(rng.integers(0, 2))
        args = [mode, "--samplerate", str(rate), "-M", repr(mark), "-S", repr(space)]
        if inv:
            args.append("--inverted")
        if flt:
            args.append("--float-samples")
        text = bytes(rng.integers(32, 127, 12, dtype=np.uint8)) + b"\n"
        wav = str(tmp_path / ("x%d.wav" % i))
        subprocess.run([orc.REF_CLI, "--tx", "--file", wav] + args, input=text, check=True)
        audio, _, _ = read_wav(wav)
        m = orc.Mode(mode, sample_rate=rate, mark=mark, space=space, inverted=inv)
        mine = txorc.tx_events(m, list(text), "baudot" if mode == "rtty" else "ascii8", 1.0, 4096, flt)
        assert mine.size == audio.size, (args, mine.size, audio.size)
        assert hashlib.sha256(mine.tobytes()).digest() == hashlib.sha256(audio.astype(np.float32).tobytes()).digest(), args


# ---- 7. CPU: the gpu tests above on the emulated kernel ---------------------------------------------------------
def test_tx_tones_gpu_tests_on_the_emulated_kernel():
    """This file's gpu tests against the emulation build of the same kernel source, at reduced sizes."""
    from gpudev import run_emulated
    tail = run_emulated("", "late", 1500, module="test_gpu_tx_tones.py")
    assert " passed" in tail and "failed" not in tail
