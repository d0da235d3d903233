"""The live receiver on 16-bit PCM: fsk_b200_stream_push_s16 (int16 rows fed int16 chunks, copied bit for bit),
fsk_b200_rx_batch_s16_runs (does the plain int16 rx call have a build for this launch shape?) and
LiveReceiver(pcm16=True).

- The int16 push is the float push on the widened samples (x / 32768): the same fill, states and dropped, and
  rows that widen to the float rows, for every channel count, event and overflow; the same refusals, plus the
  row layout of the _s16 rx calls.
- LiveReceiver(pcm16=True) prints the reference CLI's stdout for its vectors however the audio is cut, and
  gives, feed by feed, the text, counts, stream and decoder states and dropped of the float receiver fed the
  widened chunks: plain, tones, channels, auto-carrier and streams that open and end on their own.
- Where the plain int16 call has no build the receiver keeps float rows and widens every chunk; the query
  agrees with the call on every preset.

The CPU tests run the `gpu` tests of this file on the host SIMT emulation of the kernels (tests/emu), with
copies landing at issue and as late as the code's waits allow."""
import ctypes as C
import subprocess
import zlib

import numpy as np
import pytest

import autoorc
import golden_util as gu
import orc
import refcases
from gpudev import bands_tensor, dev, emulated, mm, pcm, state_rows, sync, torch, upload, widen
from rxcases import ANSWER, ORIGINATE, TONE_PRESETS, call_audio, cuts, duplex_audio, random_states

EINVAL, ENOTSUP = 22, 95
OPEN, END, ENDED = 1, 2, 2


# --------------------------------------------------------------------------
# CPU
# --------------------------------------------------------------------------
@pytest.mark.parametrize("async_mode", ["eager", "late"])
def test_live_pcm16_on_the_emulated_kernels(async_mode):
    """The `gpu` tests below on the host SIMT emulation of the kernels."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", async_mode, 3000, module="test_gpu_live_pcm16.py")
    assert " passed" in tail and "failed" not in tail


def test_the_int16_push_and_the_query_are_exported():
    names = {"fsk_b200_stream_push_s16", "fsk_b200_rx_batch_s16_runs"}
    assert names <= set(mm().EXPORTS)
    nm = subprocess.run(["nm", "-D", "--defined-only", mm().LIB_PATH], stdout=subprocess.PIPE, check=True)
    exported = {f[2] for f in (line.split() for line in nm.stdout.decode().splitlines()) if len(f) == 3}
    assert names <= exported


def test_stream_push_refuses_mixed_sample_types():
    t = torch()
    fill = t.zeros((2,), dtype=t.int32)
    states = t.zeros((2, mm().STATE_WORDS), dtype=t.int32)
    for rows, chunk in ((t.int16, t.float32), (t.float32, t.int16), (t.int32, t.int32), (t.float64, t.float64)):
        with pytest.raises(TypeError, match="float32 or both int16"):
            mm().stream_push(t.zeros((2, 64), dtype=rows), fill, states, t.zeros((2, 8), dtype=chunk), 8)


# --------------------------------------------------------------------------
# 1. the int16 push is the float push on the widened samples
# --------------------------------------------------------------------------
def flag_some(rng, st, nrows, k):
    """per row: no channel flagged, some, or all"""
    for r in range(nrows):
        pre = int(rng.integers(0, 3))
        for c in range(r * k, r * k + k):
            on = pre == 2 or (pre == 1 and rng.random() < 0.5)
            st["done"][c] = (int(st["done"][c]) & ~ENDED) | (ENDED if on else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 3])
def test_int16_push_equals_the_float_push(k):
    """Random rows, fills, states (some flagged STREAM_ENDED), chunk lengths per row and common, chunks that
    overflow the row; channels disabled or not; row events NULL or OPEN / END / OPEN | END (other bits too).
    After both pushes: the rows' first fill[r] samples widened, fill, every state word and dropped are equal."""
    t = torch()
    rng = np.random.default_rng(1616 + k)
    stride, nrows, nb, width = 392, 24, 40, 256
    overflowed = False
    for with_bands in (False, True):
        for with_events in (False, True):
            for per_row in (True, False):
                fill = rng.integers(0, stride + 1, nrows).astype(np.int32)
                rows16 = rng.integers(-32768, 32768, (nrows, stride)).astype(np.int16)
                st0 = random_states(rng, nrows * k, fill, k)
                flag_some(rng, st0, nrows, k)
                bands = None
                if with_bands:
                    bands = rng.integers(0, nb, (nrows * k, 2)).astype(np.uint32)
                    off = rng.random(nrows * k) < 0.4
                    bands[off, int(rng.integers(2))] = nb
                bt = bands_tensor(bands) if bands is not None else None
                chunk16 = rng.integers(-32768, 32768, (nrows, width)).astype(np.int16)
                clen = upload(rng.integers(0, width + 1, nrows).astype(np.int32)) if per_row else int(rng.integers(0, width + 1))
                ev = None
                if with_events:
                    ev = upload(np.array([(r % 4) | (int(rng.integers(0, 64)) << 2) for r in range(nrows)], np.uint8))
                out = {}
                for name, rows, chunk in (("f32", widen(rows16), widen(chunk16)), ("s16", rows16, chunk16)):
                    R, F, S = upload(rows), upload(fill), state_rows(st0)
                    D = upload(np.full(nrows, -1, np.int32))
                    mm().stream_push(R, F, S, upload(chunk), clen, dropped=D, channels_per_row=k, tone_bands=bt,
                                     nbands=nb, row_events=ev)
                    sync()
                    out[name] = R.cpu().numpy(), F.cpu().numpy(), S.cpu().numpy(), D.cpu().numpy()
                    assert R.dtype == (t.int16 if name == "s16" else t.float32)
                (rf, ff, sf, df), (rs, fs, ss, ds) = out["f32"], out["s16"]
                what = (k, with_bands, with_events, per_row)
                assert (ff == fs).all() and (df == ds).all(), what
                assert sf.tobytes() == ss.tobytes(), what
                overflowed |= bool((ds > 0).any() and (fs == stride).any())
                for r in range(nrows):
                    n = int(fs[r])
                    assert widen(rs[r, :n]).tobytes() == rf[r, :n].tobytes(), (what, r)
    assert overflowed


@pytest.mark.gpu
def test_int16_push_refuses_where_the_float_push_does():
    """Every refusal of the float push is the int16 push's, -EINVAL with nothing launched; int16 rows must
    also be 16-byte aligned with a stride of a multiple of 8 samples, as the _s16 rx calls require."""
    t = torch()
    L = mm().lib()
    p = lambda a, off=0: C.c_void_p(a.data_ptr() + off)
    st = t.zeros((4, mm().STATE_WORDS), dtype=t.int32).to(dev())
    fill = t.zeros((2,), dtype=t.int32).to(dev())
    ev = t.full((2,), OPEN | END, dtype=t.uint8).to(dev())
    bufs = {"f32": t.zeros((2, 4096), dtype=t.float32).to(dev()), "s16": t.zeros((2, 4096), dtype=t.int16).to(dev())}
    push = {"f32": L.fsk_b200_stream_push_events, "s16": L.fsk_b200_stream_push_s16}

    def args(x, **kw):
        a = dict(samples=p(x), nrows=2, stride=4096, fill=p(fill), k=2, bands=None, nb=0, states=p(st), chunk=p(x),
                 chunk_stride=4096, clen=None, clen_all=0, dropped=None, events=p(ev), stream=None)
        a.update(kw)
        return list(a.values())
    both = [dict(k=0), dict(k=1 << 30), dict(nrows=1 << 31, k=1), dict(fill=None), dict(states=None),
            dict(samples=None), dict(chunk=None, clen_all=5), dict(stride=4092, off=4), dict(off=8),
            dict(events=None, k=0)]
    n0 = mm().launch_count()
    for case in both:
        rc = {}
        for src, x in bufs.items():
            kw = dict(case)
            off = kw.pop("off", 0)
            if off:
                kw["samples"] = p(x, off)
            rc[src] = push[src](*args(x, **kw))
        assert rc["f32"] == rc["s16"] == -EINVAL, (case, rc)
    x = bufs["s16"]
    for stride in (4092, 4, 12):                     # a whole number of floats, not of 16-byte int16 blocks
        assert push["f32"](*args(bufs["f32"], stride=stride, nrows=0)) == 0
        assert push["s16"](*args(x, stride=stride)) == -EINVAL, stride
        assert b"multiple of 8 int16 samples" in L.fsk_b200_last_error()
    assert push["s16"](*args(x, samples=p(x, 2), stride=4088)) == -EINVAL
    assert mm().launch_count() == n0
    assert push["s16"](*args(x, nrows=0)) == 0 and push["s16"](*args(x, nrows=0, k=0)) == -EINVAL
    assert mm().launch_count() == n0
    assert push["s16"](*args(x)) == 0
    sync()
    assert mm().launch_count() == n0 + 1


# --------------------------------------------------------------------------
# 2. the reference CLI's vectors through LiveReceiver(pcm16=True)
# --------------------------------------------------------------------------
VECTORS = ["small-1200", "small-300", "small-rtty", "small-same", "opt-sync-byte-600", "70-callerid-mdmf",
           "71-callerid-sdmf", "81-tdd", "cli-auto-carrier", "cli-auto-carrier-rtty"]
LONG = {"81-tdd"}                                     # minutes of audio: too slow for the emulator


def vector_pcm(name):
    """the int16 audio the reference read: audio_s16 where committed, else the exact int16 of the oracle's
    transmitter (its float output is a whole number of 1/32768 steps)"""
    case = refcases.BY_NAME[name]
    g = gu.load(name)
    if "audio_s16" in g.files:
        return case, g, g["audio_s16"]
    a = gu.audio(case, g)
    x = pcm(a)
    assert widen(x).tobytes() == a.tobytes(), name
    return case, g, x


def overrides(case):
    names = dict(mark="f_mark", space="f_space", bandwidth="band_width", startbits="nstartbits", stopbits="nstopbits")
    return {names.get(k, k): v for k, v in case["rx_mkw"].items() if k != "sample_rate"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", VECTORS)
def test_reference_vectors_in_random_cuts(name):
    """Each stream gets the vector's int16 audio in its own random cut, stream 1 a trickle; every stream's
    text adds up to the reference CLI's stdout byte for byte.  The --auto-carrier runs with auto_carrier=."""
    if emulated() and name in LONG:
        pytest.skip("too long for the emulator")
    case, g, a = vector_pcm(name)
    rate = int(case["rx_mkw"].get("sample_rate", 48000))
    kw = overrides(case)
    if name.startswith("cli-auto-carrier"):
        kw["auto_carrier"] = autoorc.DEFAULT_THRESHOLD
    nstreams, max_chunk = (3 if emulated() else 4), 2048
    lr = mm().LiveReceiver(case["rx_mode"], sample_rate=rate, nstreams=nstreams, max_chunk=max_chunk, device=dev(),
                           pcm16=True, **kw)
    assert lr.rows.dtype == torch().int16
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    fed = [0] * nstreams
    text = [b""] * nstreams

    def take(out, cnt):
        o, c = out.cpu().numpy(), cnt.cpu().numpy()
        for i in range(nstreams):
            text[i] += o[i, :c[i]].tobytes()
    while any(f < a.size for f in fed):
        chunk = np.zeros((nstreams, max_chunk), np.int16)
        clen = np.zeros(nstreams, np.int32)
        for i in range(nstreams):
            n = int(min(rng.integers(1, max_chunk + 1) if i else max_chunk, a.size - fed[i]))
            if i == 1:
                n = min(n, 333)
            chunk[i, :n] = a[fed[i]:fed[i] + n]
            clen[i], fed[i] = n, fed[i] + n
        take(*lr.feed(upload(chunk), upload(clen)))
    take(*lr.finish())
    sync()
    assert int(lr.dropped.sum()) == 0
    assert "src=s16" in lr.engine.last_kernel()
    for i in range(nstreams):
        assert text[i] == bytes(g["stdout"]), (name, i)


# --------------------------------------------------------------------------
# 3. tick by tick, the float receiver fed the widened chunks
# --------------------------------------------------------------------------
TWINS = {
    "plain": dict(mode="1200", rate=48000),
    "rtty": dict(mode="rtty", rate=8000),
    "tones": dict(mode="300", rate=48000, chans="oa", k=1),
    "channels-2": dict(mode="300", rate=48000, chans="oa", k=2),
    "channels-3": dict(mode="300", rate=48000, chans="oxa", k=3),
    "auto": dict(mode="1200", rate=48000, auto=True),
    "events": dict(mode="1200", rate=48000, events=True),
    "events-channels": dict(mode="300", rate=48000, chans="oa", k=2, events=True),
}


def twin_receivers(c, nrows, max_chunk):
    kw = {}
    if "chans" in c:
        # per channel "o" originate, "a" answer, "x" disabled; one channel per row: the two rows alternate
        e0 = mm().RxEngine.for_mode(c["mode"], c["rate"])
        nb = int(e0.params.nbands)
        pair = {"o": list(mm().tone_bands(e0.params, *ORIGINATE)), "a": list(mm().tone_bands(e0.params, *ANSWER)),
                "x": [nb, nb]}
        chans = c["chans"][:c["k"]] if c["k"] > 1 else "".join(c["chans"][r % 2] for r in range(nrows))
        bands = np.array([pair[ch] for ch in (chans * nrows if c["k"] > 1 else chans)], np.int32)
        kw = dict(tones=upload(bands), channels_per_row=c["k"])
    if c.get("auto"):
        kw = dict(auto_carrier=autoorc.DEFAULT_THRESHOLD)
    return [mm().LiveReceiver(c["mode"], c["rate"], nrows, max_chunk=max_chunk, device=dev(), pcm16=p, **kw)
            for p in (False, True)]


def snapshot(rx, out):
    text, cnt = out
    sync()
    text, cnt = text.cpu().numpy(), cnt.cpu().numpy()
    return ([text[i, :cnt[i]].tobytes() for i in range(len(cnt))], cnt.tobytes(), rx.states.cpu().numpy().tobytes(),
            rx.dstates.cpu().numpy().tobytes(), rx.dropped.cpu().numpy().tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TWINS))
def test_pcm16_receiver_equals_the_float_receiver_feed_by_feed(name):
    """The same int16 audio, the same cuts: LiveReceiver(pcm16=True) fed int16 chunks and the float receiver
    fed the widened chunks return identical text, counts, stream states, decoder states and dropped after every
    feed and after finish().  With events, streams open and end at random ticks (a second call per row, and
    noise after an end that is dropped)."""
    c = TWINS[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    nrows = 4 if emulated() else 48
    m = orc.Mode(c["mode"], sample_rate=c["rate"])
    max_chunk = 1500 if c["rate"] == 48000 else 500
    rf, rs = twin_receivers(c, nrows, max_chunk)
    assert rs.rows.dtype == torch().int16 and rf.rows.dtype == torch().float32
    # per row: (start tick, audio, pieces) for one call, or two with events
    sched = []
    for r in range(nrows):
        calls, tick = [], int(rng.integers(0, 3))
        for _ in range(2 if c.get("events") else 1):
            x = duplex_audio(rng, int(rng.integers(2, 4))) if "chans" in c else call_audio(rng, m, int(rng.integers(2, 5)))
            x = pcm(x)
            pieces = cuts(rng, x.size, max_chunk)
            calls.append((tick, x, pieces))
            tick += len(pieces) + int(rng.integers(1, 4))
        sched.append(calls)
    nt = max(cs[-1][0] + len(cs[-1][2]) for cs in sched) + 1
    ntext = 0
    for tick in range(nt):
        chunk = np.zeros((nrows, max_chunk), np.int16)
        clen = np.zeros(nrows, np.int32)
        opened, ended = np.zeros(nrows, bool), np.zeros(nrows, bool)
        for r in range(nrows):
            live = False
            for (t0, x, pieces) in sched[r]:
                if t0 <= tick < t0 + len(pieces):
                    i = tick - t0
                    off = sum(pieces[:i])
                    chunk[r, :pieces[i]] = x[off:off + pieces[i]]
                    clen[r] = pieces[i]
                    opened[r], ended[r], live = i == 0, i == len(pieces) - 1, True
            if c.get("events") and not live and rng.random() < 0.3:
                clen[r] = int(rng.integers(1, max_chunk + 1))
                chunk[r, :clen[r]] = rng.integers(-3000, 3000, clen[r])
        ev = dict(opened=upload(opened), ended=upload(ended)) if c.get("events") else {}
        a = snapshot(rf, rf.feed(upload(widen(chunk)), upload(clen), **ev))
        b = snapshot(rs, rs.feed(upload(chunk), upload(clen), **ev))
        assert a == b, (name, tick)
        ntext += sum(len(x) for x in b[0])
    assert "src=s16" in rs.engine.last_kernel() and "src=f32" in rf.engine.last_kernel()
    a, b = snapshot(rf, rf.finish()), snapshot(rs, rs.finish())
    assert a == b, name
    assert ntext + sum(len(x) for x in b[0]) > 0


@pytest.mark.gpu
def test_pcm16_receiver_refuses_a_float_chunk():
    lr = mm().LiveReceiver("1200", 48000, 2, max_chunk=64, device=dev(), pcm16=True)
    with pytest.raises(TypeError, match="int16"):
        lr.feed(torch().zeros((2, 64), dtype=torch().float32).to(dev()))
    lf = mm().LiveReceiver("1200", 48000, 2, max_chunk=64, device=dev())
    with pytest.raises(TypeError, match="float32"):
        lf.feed(torch().zeros((2, 64), dtype=torch().int16).to(dev()))


# --------------------------------------------------------------------------
# 4. both row paths, and the query against the call
# --------------------------------------------------------------------------
# a framing whose per-candidate launch shape has no int16 build (fsk_b200_rx_batch_s16_runs says 0)
NO_S16 = dict(mode="1200", rate=48000, n_data_bits=24)


@pytest.mark.gpu
def test_the_query_picks_the_row_type():
    """A preset the int16 kernel takes: int16 rows, the rx call runs on them (src=s16).  A framing it does not
    take (the query says so): float32 rows, every chunk widened, odd chunk widths included, and the text of
    the float receiver."""
    t = torch()
    lr = mm().LiveReceiver("1200", 48000, 3, max_chunk=1000, device=dev(), pcm16=True)
    assert lr.engine.rx_batch_s16_runs(3) and lr.rows.dtype == t.int16 and lr.stride % 8 == 0
    lr.feed(upload(np.zeros((3, 1000), np.int16)))
    sync()
    assert "src=s16" in lr.engine.last_kernel()
    c = NO_S16
    over = dict(n_data_bits=c["n_data_bits"])
    eng = mm().RxEngine.for_mode(c["mode"], c["rate"], **over)
    assert not eng.rx_batch_s16_runs(3)
    rng = np.random.default_rng(24)
    m = orc.Mode(c["mode"], sample_rate=c["rate"], **over)
    streams = [pcm(call_audio(rng, m, 4)) for _ in range(3)]
    max_chunk = 999
    rs, rf = [mm().LiveReceiver(c["mode"], c["rate"], 3, max_chunk=max_chunk, device=dev(), pcm16=p, **over)
              for p in (True, False)]
    assert rs.rows.dtype == t.float32
    fed = [0] * 3
    got, want = [b""] * 3, [b""] * 3
    while any(f < a.size for a, f in zip(streams, fed)):
        w = int(rng.integers(1, max_chunk + 1))             # any width, multiples of 4 or not
        chunk = np.zeros((3, w), np.int16)
        clen = np.zeros(3, np.int32)
        for i, a in enumerate(streams):
            n = min(w, a.size - fed[i])
            chunk[i, :n], clen[i], fed[i] = a[fed[i]:fed[i] + n], n, fed[i] + n
        sa, sb = snapshot(rs, rs.feed(upload(chunk), upload(clen))), snapshot(rf, rf.feed(upload(widen(chunk)), upload(clen)))
        assert sa == sb
        got = [g + x for g, x in zip(got, sa[0])]
        want = [g + x for g, x in zip(want, sb[0])]
    assert snapshot(rs, rs.finish()) == snapshot(rf, rf.finish())
    assert "src=f32" in rs.engine.last_kernel()
    assert sum(len(x) for x in got) > 0 and got == want


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [8000, 48000])
def test_the_query_agrees_with_the_call_on_every_preset(rate):
    """fsk_b200_rx_batch_s16_runs is 1 exactly where fsk_b200_rx_batch_s16 launches and 0 exactly where it
    returns -ENOTSUP with nothing launched; -EINVAL for a NULL engine."""
    t = torch()
    L = mm().lib()
    x = t.zeros((3, 2048), dtype=t.int16).to(dev())
    assert L.fsk_b200_rx_batch_s16_runs(None, 3) == -EINVAL
    seen = set()
    for name in TONE_PRESETS:
        try:
            eng = mm().RxEngine.for_mode(name, rate)
        except RuntimeError:                             # tones above this rate's Nyquist band ("12000" at 8 kHz)
            continue
        mf = eng.max_frames(2048)
        fr = t.zeros((3, mf, 5), dtype=t.int32).to(dev())
        st = t.zeros((3, mm().STATE_WORDS), dtype=t.int32).to(dev())
        runs = L.fsk_b200_rx_batch_s16_runs(eng._e, 3)
        n0 = mm().launch_count()
        rc = L.fsk_b200_rx_batch_s16(eng._e, C.c_void_p(x.data_ptr()), 3, 2048, None, 2048,
                                     C.c_void_p(fr.data_ptr()), mf, C.c_void_p(st.data_ptr()), None)
        sync()
        assert (runs, rc) in ((1, 0), (0, -ENOTSUP)), (name, rate, runs, rc)
        assert mm().launch_count() == n0 + runs, (name, rate)
        assert eng.rx_batch_s16_runs(3) == bool(runs)
        seen.add(runs)
    assert seen == {0, 1}                                # the UIC presets have no int16 build


# --------------------------------------------------------------------------
# 5. loopback from the live transmitter's int16 audio
# --------------------------------------------------------------------------
LOOP = [("rtty", 8000), ("tdd", 48000), ("same", 48000), ("callerid", 48000), ("1200", 48000)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate", LOOP, ids=[m for m, _ in LOOP])
def test_loopback_from_the_live_transmitter(mode, rate):
    """LiveTransmitter's int16 audio (its default, like minimodem --tx), fed in chunks to
    LiveReceiver(pcm16=True), gives the transmitted text back."""
    import txorc
    t = torch()
    n = 2 if emulated() else 32
    rng = np.random.default_rng(zlib.crc32(mode.encode()))
    if mode == "callerid":
        g = gu.load("70-callerid-mdmf")
        texts, wants = [bytes(g["text"])] * n, [bytes(g["stdout"])] * n
    else:
        texts = [bytes(int(v) for v in rng.integers(32, 127, 8 if emulated() else int(rng.integers(10, 40))))
                 for _ in range(n)]
        wants = list(texts)
    tx = mm().LiveTransmitter(mode, rate, nstreams=n, max_text=max(len(x) for x in texts), idle=False, device=dev())
    if tx.engine.encoder == mm().ENCODE_BAUDOT:
        wants = []
        for x in texts:
            w = txorc.encode("baudot", x)
            wants.append(orc.decode_words("baudot", 5, w, resets=[1] + [0] * (len(w) - 1)))
    buf = np.zeros((n, max(len(x) for x in texts)), np.uint8)
    for i, x in enumerate(texts):
        buf[i, :len(x)] = np.frombuffer(x, np.uint8)
    a1, c1 = tx.feed(upload(buf), upload(np.array([len(x) for x in texts], np.int32)))
    a2, c2 = tx.finish()
    sync()
    assert a1.dtype == t.int16
    a1, c1, a2, c2 = a1.cpu().numpy(), c1.cpu().numpy(), a2.cpu().numpy(), c2.cpu().numpy()
    audio = [np.concatenate([a1[s, :c1[s]], a2[s, :c2[s]], np.zeros(rate, np.int16)]) for s in range(n)]
    max_chunk = rate // 5
    rx = mm().LiveReceiver(mode, rate, nstreams=n, max_chunk=max_chunk, device=dev(), pcm16=True)
    assert rx.rows.dtype == t.int16
    got = [b""] * n
    for o in range(0, max(a.size for a in audio), max_chunk):
        chunk = np.zeros((n, max_chunk), np.int16)
        clen = np.zeros(n, np.int32)
        for s, a in enumerate(audio):
            piece = a[o:o + max_chunk]
            chunk[s, :piece.size], clen[s] = piece, piece.size
        text, cnt = snapshot(rx, rx.feed(upload(chunk), upload(clen)))[:2]
        got = [g + x for g, x in zip(got, text)]
    got = [g + x for g, x in zip(got, snapshot(rx, rx.finish())[0])]
    for s in range(n):
        assert got[s] == wants[s], (mode, s, got[s][:60], wants[s][:60])
