"""Live streams that end and start on their own: FSK_B200_STREAM_ENDED in every rx call, and the row events
(FSK_B200_ROW_OPEN / FSK_B200_ROW_END) of fsk_b200_stream_push_events.

- A stream whose state carries the flag stops by the loop's own rule (src/minimodem.c:1229) whatever holdback
  the engine has: it gives the records and state of the same engine at holdback 0, and its neighbours give
  those of the batch without the flag.  This holds in every rx family.
- Rows that end at their own tick through ROW_END give, concatenated, the records of one pass over the whole
  stream; the rows still being fed are unchanged, tick by tick.  ROW_OPEN starts a fresh stream.
- The push is pinned to a numpy model of its rule, and LiveReceiver with calls arriving and leaving at random
  gives, per call, the text of a one-pass decode of that call from fresh decoder state.

"One pass" is one plain rx call of the same family over the whole stream at holdback 0; "equal" is byte for
byte.  The CPU tests run the `gpu` tests of this file on the host SIMT emulation of the kernels (tests/emu),
with copies landing at issue and as late as the code's waits allow."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest

import autoorc
import orc
import rxfam
from gpudev import bands_tensor, dev, emulated, mm, pcm, records, rows, state_rows, sync, torch, upload
import rxcases
from rxcases import (ANSWER, ORIGINATE, call_audio, channel_rows, cuts, duplex_audio, random_states,
                     shape_case)

EINVAL = 22
ENDED = 2
OPEN, END = 1, 2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SESSION = ("carrier", "noconfidence", "track_amplitude", "peak_confidence", "carrier_nsamples",
           "confidence_total", "amplitude_total", "nframes_decoded", "done")


# --------------------------------------------------------------------------
# CPU
# --------------------------------------------------------------------------
@pytest.mark.parametrize("async_mode", ["eager", "late"])
def test_stream_lifetimes_on_the_emulated_kernels(async_mode):
    """The `gpu` tests below on the host SIMT emulation of the kernels (the TMA bulk fill excepted)."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", async_mode, 3000, module="test_gpu_stream_lifetimes.py")
    assert " passed" in tail and "failed" not in tail


def test_header_constants_are_the_bindings():
    src = open(os.path.join(ROOT, "include", "fsk_b200.h")).read()
    val = lambda name: int(re.search(r"#define %s\s+(\d+)u" % name, src).group(1))
    assert val("FSK_B200_STREAM_ENDED") == mm().STREAM_ENDED == ENDED
    assert val("FSK_B200_ROW_OPEN") == mm().ROW_OPEN == OPEN
    assert val("FSK_B200_ROW_END") == mm().ROW_END == END
    assert "fsk_b200_stream_push_events" in mm().EXPORTS


def test_check_not_truncated_ignores_the_flag():
    st = np.zeros(3, mm().STATE_DTYPE)
    st["nframes"] = 4
    st["done"] = [1, ENDED | 1, 0]
    mm().check_not_truncated(torch().from_numpy(st[:2].view(np.int32).reshape(2, -1).copy()), 4)
    st["done"][2] = ENDED
    with pytest.raises(RuntimeError, match="stream 2"):
        mm().check_not_truncated(torch().from_numpy(st.view(np.int32).reshape(3, -1).copy()), 4)


# --------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------
def flagged(n, spw=8):
    """about half the streams, both values at every slot of a group of up to 8 streams per warp"""
    return np.array([(i + i // spw) % 2 == 1 for i in range(n)])


def with_flags(nstreams, flags, st=None):
    st = np.zeros(nstreams, mm().STATE_DTYPE) if st is None else st.copy()
    st["done"] = np.where(flags, ENDED, st["done"])
    return state_rows(st)


def window_of(eng, call):
    return eng.auto_stream_window() if call == "auto" else eng.stream_window()


FLAG_FAMS = list(rxfam.FAMILIES)


def flag_case(fam):
    """(engine factory, call, src, rows, per-row lengths, bands or None, k): 19 streams (more than one block
    of most launches, the last one partial), the six of the family's case repeated"""
    if fam.startswith("channels"):
        k = int(fam[-1])
        streams, lens, b = channel_rows("1200", 48000, 7, k, 77 + k)
        return (lambda: mm().RxEngine.for_mode("1200", 48000)), "tones", "f32", streams, lens * 7 // 8, b, k
    if fam.startswith("generic"):
        rng = np.random.default_rng(25)
        m = orc.Mode("25", sample_rate=48000)
        streams = []
        for i in range(7):
            w = rng.integers(0, 256, 3, dtype=np.uint64).astype(np.uint32)
            x = np.concatenate([np.zeros(int(rng.integers(0, 4000)), np.float32), orc.tx_words(m, w, 0.7, 4096, True)])
            streams.append((x + np.float32(0.01) * rng.standard_normal(x.size)).astype(np.float32))
        lens = np.array([x.size * 7 // 8 for x in streams], np.int32)
        return ((lambda: mm().RxEngine.for_mode("25", 48000)), "rx", "s16" if fam.endswith("s16") else "f32",
                streams, lens, None, 1)
    f = rxfam.FAMILIES[fam]
    preset = ("300", 48000) if fam.startswith("prefix") else ("1200", 48000)
    make, streams, lens, bands, _ = shape_case(fam, preset)
    idx = [i % len(streams) for i in range(19)]
    b = None if bands is None else np.array([bands[i] for i in idx], np.uint32)
    # every row cut inside its transmission, so that the holdback holds records back
    return make, f["call"], f["src"], [streams[i] for i in idx], lens[idx] * 7 // 8, b, 1


def rx_any(eng, fam, src, streams, lens, bands, states=None, auto_states=None, max_frames=None, k=None):
    """one rx call of the family on the streams as `src` rows; returns (records per channel, states, device
    states, auto states as numpy or None)"""
    r = rxfam.call(eng, fam, [pcm(a) for a in streams] if src == "s16" else streams, lens, bands=bands,
                   states=states, auto_states=auto_states, max_frames=max_frames, k=k)
    return r.recs, r.st, r.states, (None if r.auto is None else r.auto.cpu().numpy().copy())


# --------------------------------------------------------------------------
# 1. the flag in every rx family
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fam", FLAG_FAMS)
def test_the_flag_ends_a_stream_in_every_rx_family(fam, monkeypatch):
    """Holdback stream_window(), about half the states flagged: a flagged stream gives the records and state
    (flag aside) of the same engine at holdback 0, an unflagged one those of the batch with no flag."""
    rxfam.skip_tma(fam)
    make, call, src, streams, lens, bands, k = flag_case(fam)
    eng = rxfam.new_engine(monkeypatch, fam, make)
    nch = len(streams) * k
    flags = flagged(nch)
    eng.set_holdback(0)
    r0, s0, _, a0 = rx_any(eng, fam, src, streams, lens, bands)
    rxfam.check_launch(eng, fam)
    eng.set_holdback(window_of(eng, call))
    rh, sh, _, ah = rx_any(eng, fam, src, streams, lens, bands)
    rxfam.check_launch(eng, fam)
    rf, sf, _, af = rx_any(eng, fam, src, streams, lens, bands, states=with_flags(nch, flags))
    rxfam.check_launch(eng, fam)
    for c in range(nch):
        want_r, want_s = (r0[c], s0[c]) if flags[c] else (rh[c], sh[c])
        assert rf[c] == want_r, (fam, c, bool(flags[c]))
        got = sf[c].copy()
        if flags[c]:
            assert got["done"] & ENDED, (fam, c)
        got["done"] &= ~np.uint32(ENDED)
        assert got.tobytes() == want_s.tobytes(), (fam, c, bool(flags[c]))
        if a0 is not None:
            assert af[c].tobytes() == (a0 if flags[c] else ah)[c].tobytes(), (fam, c)


# --------------------------------------------------------------------------
# 2. the skip rule
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
def test_skip_rule_and_overflow_of_a_flagged_stream(src):
    """done = 1 and done = 1 | ENDED come back untouched with no records; done = ENDED runs; a flagged stream
    stopped by a 3-record buffer resumes (done == ENDED, nframes == 3) to the one-pass records."""
    make, _, _, streams, lens, _, _ = flag_case("per-candidate")
    eng = make()
    streams, lens = streams[:6], lens[:6]
    eng.set_holdback(0)
    whole, sw, _, _ = rx_any(eng, "per-candidate", src, streams, lens, None)
    eng.set_holdback(eng.stream_window())
    st0 = np.zeros(6, mm().STATE_DTYPE)
    st0["done"] = [1, 1 | ENDED, 1 | 4, ENDED, ENDED, 4]
    st0["pos"][:3] = 77
    recs, st, _, _ = rx_any(eng, "per-candidate", src, streams, lens, None, states=state_rows(st0))
    for s in (0, 1, 2, 5):
        assert recs[s] == b"" and st[s].tobytes() == st0[s].tobytes(), s
    assert recs[3] == whole[3] and recs[4] == whole[4]
    # overflow and resume
    states = with_flags(6, np.ones(6, bool))
    got = [b""] * 6
    for call in range(10000):
        recs, st, states, _ = rx_any(eng, "per-candidate", src, streams, lens, None, states=states, max_frames=3)
        got = [g + r for g, r in zip(got, recs)]
        if (st["done"] == (1 | ENDED)).all():
            break
        assert (st["nframes"][st["done"] == ENDED] == 3).all() and (st["done"] & ENDED).all()
        with pytest.raises(RuntimeError):
            mm().check_not_truncated(states, 3)
        st["nframes"][:] = 0
        states = state_rows(st)
    assert call >= 2 and got == whole
    st["nframes"], st["done"] = sw["nframes"], sw["done"]
    assert st.tobytes() == sw.tobytes()


# --------------------------------------------------------------------------
# the live driver: push with events, one rx call per tick
# --------------------------------------------------------------------------
class Live:
    def __init__(self, eng, call, nrows, k, stride, bands=None):
        t = torch()
        z = lambda shape: t.zeros(shape, dtype=t.int32).to(dev())
        self.eng, self.call, self.nrows, self.k, self.stride = eng, call, nrows, k, stride
        self.rows = t.zeros((nrows, stride), dtype=t.float32).to(dev())
        self.fill, self.dropped = z((nrows,)), z((nrows,))
        self.states = z((nrows * k, mm().STATE_WORDS))
        self.auto = t.zeros((nrows, mm().AUTO_STATE_BYTES), dtype=t.uint8).to(dev()) if call == "auto" else None
        self.bands = None if bands is None else bands_tensor(bands)
        self.nb = int(eng.params.nbands)
        self.max_frames = eng.max_frames(stride)

    def tick(self, chunk, clen, events):
        """returns the records of this tick per channel and the states"""
        t = torch()
        ev = upload(np.asarray(events, np.uint8))
        if self.auto is not None:
            self.auto.masked_fill_(upload((np.asarray(events) & OPEN) != 0)[:, None], 0)
        mm().stream_push(self.rows, self.fill, self.states, upload(chunk), upload(np.asarray(clen, np.int32)),
                         dropped=self.dropped, channels_per_row=self.k, tone_bands=self.bands, nbands=self.nb,
                         row_events=ev)
        n = self.stride
        if self.call == "rx":
            fr, self.states = self.eng.rx_batch(self.rows, nsamples=n, nsamples_each=self.fill,
                                                max_frames=self.max_frames, states=self.states)
        elif self.call == "tones":
            fr, self.states = self.eng.rx_batch_tones(self.rows, self.bands, nsamples=n, nsamples_each=self.fill,
                                                      max_frames=self.max_frames, states=self.states,
                                                      channels_per_row=self.k)
        else:
            fr, self.states, self.auto = self.eng.rx_batch_auto(self.rows, nsamples=n, nsamples_each=self.fill,
                                                                max_frames=self.max_frames, states=self.states,
                                                                auto_states=self.auto)
        sync()
        return records(fr, self.states)


def live_geometry(eng, call):
    window = window_of(eng, call)
    max_chunk = (3 * window + 3) & ~3
    return window, max_chunk, (window + int(eng.params.frame_nsamples) + 2 * max_chunk + 64 + 3) & ~3


STAGGER = {
    "rx": ("per-candidate", None),
    "tones": ("tones", None),
    "channels": ("channels-2", None),
    "auto": ("auto", None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("what", list(STAGGER))
def test_staggered_ends_through_the_events(what, monkeypatch):
    """Each row ends at its own tick through ROW_END on its last chunk: its concatenated records are those of
    one pass, and its final session state is the one pass's.  The rows still being fed give, tick by tick,
    the records of a run in which no row ends.  The tone call with one channel disabled per row (k = 3)."""
    fam = STAGGER[what][0]
    make, call, src, streams, lens, bands, k = flag_case(fam)
    streams = [a[:int(n)] for a, n in zip(streams, lens)][:6]
    if bands is not None:
        bands = bands[:6 * k]
    if what == "tones":           # three channels per row: the row's pair, a disabled one, the pair again
        nb = int(make().params.nbands)
        bands = np.array([p for b in bands for p in (list(b), [nb, 3], list(b))], np.uint32)
        k = 3
        call = "tones"
    eng = rxfam.new_engine(monkeypatch, fam, make)
    eng.set_holdback(0)
    whole, sw, _, _ = rx_any(eng, fam, "f32", streams, [a.size for a in streams], bands, k=k)
    window, max_chunk, stride = live_geometry(eng, call)
    eng.set_holdback(window)
    rng = np.random.default_rng(zlib.crc32(what.encode()))
    plan = [cuts(rng, a.size, max_chunk) for a in streams]
    nt = max(len(p) for p in plan) + 2
    a, b = Live(eng, call, 6, k, stride, bands), Live(eng, call, 6, k, stride, bands)
    got, last = [b""] * (6 * k), [b""] * (6 * k)
    fed = [0] * 6
    ticks = 0
    for tick in range(nt):
        chunk = np.zeros((6, max_chunk), np.float32)
        clen = np.zeros(6, np.int32)
        ev = np.zeros(6, np.uint8)
        for r in range(6):
            if tick < len(plan[r]):
                c = plan[r][tick]
                chunk[r, :c] = streams[r][fed[r]:fed[r] + c]
                clen[r] = c
                fed[r] += c
                if tick == len(plan[r]) - 1:
                    ev[r] = END
        ra, sa = a.tick(chunk, clen, ev)
        rb, _ = b.tick(chunk, clen, np.zeros(6, np.uint8))
        for c in range(6 * k):
            r = c // k
            if tick < len(plan[r]):
                got[c] += ra[c]
            else:                       # an ended row is skipped: its state stays as the end left it
                assert sa[c].tobytes() == last[c], (what, tick, c)
            last[c] = sa[c].tobytes()
            if tick < len(plan[r]) - 1:
                assert ra[c] == rb[c], (what, tick, c)
                ticks += 1
    assert ticks >= 6
    assert (a.dropped.cpu().numpy() == 0).all()
    for c in range(6 * k):
        assert got[c] == whole[c], (what, c)
        assert sa[c]["done"] == (ENDED | (sw[c]["done"] if bands is None or max(bands[c]) < a.nb else 0)), c
        for f in SESSION[:-1]:
            assert sa[c][f] == sw[c][f], (what, c, f)


# --------------------------------------------------------------------------
# 4. reopen
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_reopen_abandon_whole_stream_and_dropped_chunks():
    """ROW_OPEN after an end (on a new tone pair), ROW_OPEN on a live row (the old stream abandoned
    mid-way) and OPEN | END in one push give the records of a fresh one-pass run; chunks to an ended row
    are counted in dropped and change neither its fill, its records nor its states."""
    make, call, src, streams, lens, bands, k = flag_case("tones")
    eng = make()
    streams = [a[:int(n)] for a, n in zip(streams, lens)][:6]
    bands = bands[:6]
    window, max_chunk, stride = live_geometry(eng, "tones")
    eng.set_holdback(0)
    whole, _, _, _ = rx_any(eng, "tones", "f32", streams, [a.size for a in streams], bands)
    eng.set_holdback(window)
    # the first stream of every row runs on another row's pair: rows are reopened on their own pair
    first_bands = np.roll(bands, 1, axis=0)
    live = Live(eng, "tones", 6, 1, (stride + streams[0].size + 3) & ~3, first_bands)   # row 0 takes a whole stream
    rng = np.random.default_rng(4)
    # phase 1: rows 0-2 get a stream and end it; rows 3-5 get half of another row's stream and stay live
    olds = [streams[(r + 1) % 6] for r in range(6)]
    plans = [cuts(rng, olds[r].size if r < 3 else olds[r].size // 2, max_chunk) for r in range(6)]
    fed = [0] * 6
    for tick in range(max(len(p) for p in plans)):
        chunk = np.zeros((6, max_chunk), np.float32)
        clen = np.zeros(6, np.int32)
        ev = np.zeros(6, np.uint8)
        for r in range(6):
            if tick < len(plans[r]):
                c = plans[r][tick]
                chunk[r, :c], clen[r] = olds[r][fed[r]:fed[r] + c], c
                fed[r] += c
                if r < 3 and tick == len(plans[r]) - 1:
                    ev[r] = END
        live.tick(chunk, clen, ev)
    # chunks to ended rows are dropped and change nothing
    fill0, st0 = live.fill.cpu().numpy().copy(), mm().states_to_numpy(live.states).copy()
    rows0 = live.rows.cpu().numpy().copy()
    chunk = rng.standard_normal((6, max_chunk)).astype(np.float32)
    clen = np.array([100, 5, max_chunk, 0, 0, 0], np.int32)
    recs, st = live.tick(chunk, clen, np.array([0, END, 0, 0, 0, 0], np.uint8))
    assert (live.dropped.cpu().numpy()[:3] == clen[:3]).all()
    assert (live.fill.cpu().numpy()[:3] == fill0[:3]).all() and (live.rows.cpu().numpy()[:3] == rows0[:3]).all()
    assert st[:3].tobytes() == st0[:3].tobytes() and (st["done"][:3] == 1 | ENDED).all()
    # phase 2: every row reopened on its own pair; row 0 takes its whole stream in one OPEN | END push
    live.bands.copy_(bands_tensor(bands))
    plans = [[streams[0].size]] + [cuts(rng, streams[r].size, max_chunk) for r in range(1, 6)]
    fed = [0] * 6
    got = [b""] * 6
    wide = max(max_chunk, streams[0].size)
    for tick in range(max(len(p) for p in plans)):
        chunk = np.zeros((6, wide), np.float32)
        clen = np.zeros(6, np.int32)
        ev = np.zeros(6, np.uint8)
        for r in range(6):
            if tick < len(plans[r]):
                c = plans[r][tick]
                chunk[r, :c], clen[r] = streams[r][fed[r]:fed[r] + c], c
                fed[r] += c
                ev[r] |= OPEN if tick == 0 else 0
                ev[r] |= END if tick == len(plans[r]) - 1 else 0
        recs, st = live.tick(chunk, clen, ev)
        got = [g + (x if tick < len(plans[r]) else b"") for r, (g, x) in enumerate(zip(got, recs))]
    assert got == whole
    assert (st["done"] & ENDED).all()


# --------------------------------------------------------------------------
# 5. the push against a numpy model
# --------------------------------------------------------------------------
def push_model(rows_, fill, states, k, bands, nbands, chunk, clen, events):
    rows_, fill, states = rows_.copy(), fill.copy(), states.copy()
    dropped = np.zeros(len(fill), np.int64)
    stride = rows_.shape[1]
    for r in range(len(fill)):
        ch = list(range(r * k, r * k + k))
        ev = int(events[r])
        if not ev & OPEN and all(int(states["done"][c]) & ENDED for c in ch):
            dropped[r] = int(clen[r])
            continue
        if ev & OPEN:
            fill[r] = 0
            for c in ch:
                states[c] = np.zeros(1, states.dtype)[0]
        have = int(fill[r])
        act = [c for c in ch if bands is None or (bands[c][0] < nbands and bands[c][1] < nbands)]
        m = min((min(int(states["pos"][c]), have) for c in act), default=have)
        tail = have - m
        old = rows_[r].copy()
        rows_[r, :tail] = old[m:have]
        ln = int(clen[r])
        drop = max(0, ln - (stride - tail))
        ln -= drop
        rows_[r, tail:tail + ln] = chunk[r, :ln]
        fill[r], dropped[r] = tail + ln, drop
        for c in ch:
            p = min(int(states["pos"][c]), have)
            states["pos"][c] = p - min(p, m)
            states["nframes"][c] = 0
            states["done"][c] = (int(states["done"][c]) & ENDED) | (ENDED if ev & END else 0)
    return rows_, fill, states, dropped


@pytest.mark.gpu
def test_push_follows_the_event_rule():
    """fsk_b200_stream_push_events against a numpy model: every event value (other bits too), k in
    {1, 2, 5, 33}, disabled channels, flags set before the push on some, all or none of a row's channels;
    with row_events NULL the push is the channel push of test_gpu_channels' model, flags or not."""
    t = torch()
    rng = np.random.default_rng(2026)
    stride, nrows, nb = 384, 24, 40
    for k in (1, 2, 5, 33):
        for with_bands in (False, True):
            fill = rng.integers(0, stride + 1, nrows).astype(np.int32)
            rows0 = rng.standard_normal((nrows, stride)).astype(np.float32)
            st0 = random_states(rng, nrows * k, fill, k)
            pre = rng.integers(0, 3, nrows)                       # 0: no flag, 1: some channels, 2: all
            for r in range(nrows):
                for c in range(r * k, r * k + k):
                    on = pre[r] == 2 or (pre[r] == 1 and (c == r * k or rng.random() < 0.5) and c != r * k + k - 1)
                    st0["done"][c] = (int(st0["done"][c]) & ~ENDED) | (ENDED if on else 0)
            events = np.array([(r % 4) | (int(rng.integers(0, 64)) << 2) for r in range(nrows)], np.uint8)
            bands = None
            if with_bands:
                bands = rng.integers(0, nb, (nrows * k, 2)).astype(np.uint32)
                off = rng.random(nrows * k) < 0.4
                bands[off, int(rng.integers(2))] = nb
            chunk = rng.standard_normal((nrows, 200)).astype(np.float32)
            clen = rng.integers(0, 201, nrows).astype(np.int32)
            want = push_model(rows0, fill.astype(np.int64), st0, k, bands, nb, chunk, clen, events)
            R, F, S, D = upload(rows0), upload(fill), state_rows(st0), upload(np.full(nrows, -1, np.int32))
            bt = upload(bands.view(np.int32)) if bands is not None else None
            mm().stream_push(R, F, S, upload(chunk), upload(clen), dropped=D, channels_per_row=k, tone_bands=bt, nbands=nb,
                             row_events=upload(events))
            sync()
            what = (k, with_bands)
            assert (R.cpu().numpy() == want[0]).all(), what
            assert (F.cpu().numpy() == want[1]).all(), what
            got = np.frombuffer(S.cpu().numpy().tobytes(), mm().STATE_DTYPE)
            for c in range(nrows * k):
                assert got[c].tobytes() == want[2][c].tobytes(), (what, c, events[c // k], pre[c // k])
            assert (D.cpu().numpy() == want[3]).all(), what
            # row_events NULL: the channel push as it was (done = 0, no row dropped for its flags)
            want = rxcases.push_model(rows0, fill.astype(np.int64), st0, k, bands, nb, chunk, clen)
            R, F, S, D = upload(rows0), upload(fill), state_rows(st0), upload(np.full(nrows, -1, np.int32))
            mm().stream_push(R, F, S, upload(chunk), upload(clen), dropped=D, channels_per_row=k, tone_bands=bt, nbands=nb)
            sync()
            assert (R.cpu().numpy() == want[0]).all() and (F.cpu().numpy() == want[1]).all(), what
            assert S.cpu().numpy().tobytes() == want[2].tobytes() and (D.cpu().numpy() == want[3]).all(), what


# --------------------------------------------------------------------------
# 6. LiveReceiver with churn
# --------------------------------------------------------------------------


CHURN = {
    "bell202": dict(mode="1200", rate=48000),
    "rtty": dict(mode="rtty", rate=8000),
    "callerid": dict(mode="callerid", rate=48000),
    "bell103-duplex": dict(mode="300", rate=48000, k=2),
    "bell202-auto": dict(mode="1200", rate=48000, auto=True),
}


def one_pass_texts(c, calls, kind):
    """per call, the text of one rx call over its whole audio at holdback 0, decoded from fresh state"""
    eng = mm().RxEngine.for_mode(c["mode"], c["rate"])
    k = c.get("k", 1)
    if c.get("auto"):
        eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    buf, n = rows(calls, np.float32, 4)
    lens = upload(np.array([a.size for a in calls], np.int32))
    if k > 1:
        bands = eng.tone_bands([ORIGINATE[0], ANSWER[0]] * len(calls), [ORIGINATE[1], ANSWER[1]] * len(calls),
                               device=dev())
        fr, st = eng.rx_batch_tones(upload(buf), bands, nsamples=n, nsamples_each=lens, channels_per_row=k)
    elif c.get("auto"):
        fr, st, _ = eng.rx_batch_auto(upload(buf), nsamples=n, nsamples_each=lens)
    else:
        fr, st = eng.rx_batch(upload(buf), nsamples=n, nsamples_each=lens)
    out, cnt = eng.decode_batch(kind, fr, st)
    sync()
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    return [out[i, :cnt[i]].tobytes() for i in range(len(calls) * k)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CHURN))
def test_live_receiver_with_calls_that_come_and_go(name):
    """Calls arrive at random ticks, last random lengths and are fed in random chunks; between calls a row
    idles (or is fed noise after its end, counted in dropped).  Each call's text is the one-pass decode of
    its audio from fresh decoder state; an ended row returns count 0 until it is reopened."""
    from minimodem_b200.serving import LiveReceiver
    t = torch()
    c = CHURN[name]
    k = c.get("k", 1)
    nrows = 8 if emulated() else 200
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    m = orc.Mode(c["mode"], sample_rate=c["rate"])
    kw = {}
    if k > 1:
        e0 = mm().RxEngine.for_mode(c["mode"], c["rate"])
        kw = dict(tones=e0.tone_bands([ORIGINATE[0], ANSWER[0]] * nrows, [ORIGINATE[1], ANSWER[1]] * nrows,
                                      device=dev()), channels_per_row=k)
    if c.get("auto"):
        kw = dict(auto_carrier=autoorc.DEFAULT_THRESHOLD)
    max_chunk = 2000 if c["rate"] == 48000 else 700
    rx = LiveReceiver(c["mode"], c["rate"], nrows, max_chunk=max_chunk, device=dev(), **kw)
    # per row: idle ticks, then a call, then idle ticks, then a second call
    sched = []
    calls = []
    for r in range(nrows):
        ev = []
        tick = int(rng.integers(0, 4))
        for _ in range(2):
            x = duplex_audio(rng, int(rng.integers(2, 5))) if k > 1 else call_audio(rng, m, int(rng.integers(2, 6)))
            pieces = cuts(rng, x.size, max_chunk)
            ev.append((tick, len(calls), x, pieces))
            calls.append(x)
            tick += len(pieces) + int(rng.integers(0, 4))
        sched.append(ev)
    want = one_pass_texts(c, calls, rx.kind)
    assert sum(len(w) for w in want) > 0
    nt = max(e[-1][0] + len(e[-1][3]) for e in sched) + 1
    got = [b""] * (len(calls) * k)
    ended_once = np.zeros(nrows, bool)
    for tick in range(nt):
        chunk = np.zeros((nrows, max_chunk), np.float32)
        clen = np.zeros(nrows, np.int32)
        opened, ended = np.zeros(nrows, bool), np.zeros(nrows, bool)
        cur = [None] * nrows
        for r in range(nrows):
            for (t0, ci, x, pieces) in sched[r]:
                if t0 <= tick < t0 + len(pieces):
                    i = tick - t0
                    off = sum(pieces[:i])
                    chunk[r, :pieces[i]] = x[off:off + pieces[i]]
                    clen[r] = pieces[i]
                    opened[r] = i == 0
                    ended[r] = i == len(pieces) - 1
                    cur[r] = ci
            if cur[r] is None and ended_once[r] and rng.random() < 0.5:
                clen[r] = int(rng.integers(1, max_chunk + 1))     # noise after the end: dropped
                chunk[r, :clen[r]] = rng.standard_normal(clen[r]).astype(np.float32)
        text, cnt = rx.feed(upload(chunk), upload(clen),
                            opened=upload(opened), ended=upload(ended))
        sync()
        text, cnt = text.cpu().numpy(), cnt.cpu().numpy()
        dropped = rx.dropped.cpu().numpy()
        for r in range(nrows):
            for j in range(k):
                ch = r * k + j
                if cur[r] is None:
                    assert cnt[ch] == 0, (name, tick, r)
                    if ended_once[r]:
                        assert dropped[r] == clen[r], (name, tick, r)
                else:
                    got[cur[r] * k + j] += text[ch, :cnt[ch]].tobytes()
            ended_once[r] |= ended[r]
    assert ended_once.all()
    assert got == want, name


# --------------------------------------------------------------------------
# 7. host calls and refusals
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
def test_host_calls_honour_the_flag(src):
    make, _, _, streams, lens, _, _ = flag_case("per-candidate")
    streams = [a[:int(n) * 4 // 5] for a, n in zip(streams, lens)]     # cut inside the transmission
    eng = make()
    buf, n = rows([pcm(a) for a in streams] if src == "s16" else streams,
                     np.int16 if src == "s16" else np.float32, 8)
    fn = eng.rx_batch_host_s16 if src == "s16" else eng.rx_batch_host
    eng.set_holdback(0)
    f0, s0 = fn(buf, nsamples=n)
    eng.set_holdback(eng.stream_window())
    fh, sh = fn(buf, nsamples=n)
    flags = flagged(len(streams))
    st = np.zeros(len(streams), mm().STATE_DTYPE)
    st["done"] = np.where(flags, ENDED, 0)
    ff, sf = fn(buf, nsamples=n, states_out=st)
    for s in range(len(streams)):
        wf, ws = (f0, s0) if flags[s] else (fh, sh)
        nfr = int(ws["nframes"][s])
        assert sf["nframes"][s] == nfr and ff[s, :nfr].tobytes() == wf[s, :nfr].tobytes(), s
        g = sf[s].copy()
        g["done"] &= ~np.uint32(ENDED)
        assert g.tobytes() == ws[s].tobytes(), s


@pytest.mark.gpu
def test_push_events_refusals_launch_nothing():
    t = torch()
    L = mm().lib()
    x = t.zeros((2, 4096), dtype=t.float32).to(dev())
    st = t.zeros((4, mm().STATE_WORDS), dtype=t.int32).to(dev())
    fill = t.zeros((2,), dtype=t.int32).to(dev())
    ev = t.full((2,), OPEN | END, dtype=t.uint8).to(dev())
    p = lambda a: C.c_void_p(a.data_ptr())
    push = L.fsk_b200_stream_push_events
    n0 = mm().launch_count()
    assert push(p(x), 2, 4096, p(fill), 0, None, 0, p(st), p(x), 4096, None, 0, None, p(ev), None) == -EINVAL
    assert push(p(x), 2, 4096, p(fill), 1 << 30, None, 0, p(st), p(x), 4096, None, 0, None, p(ev), None) == -EINVAL
    assert push(p(x), 1 << 31, 4096, p(fill), 1, None, 0, p(st), p(x), 4096, None, 0, None, p(ev), None) == -EINVAL
    assert push(p(x), 2, 4096, None, 2, None, 0, p(st), p(x), 4096, None, 0, None, p(ev), None) == -EINVAL
    assert push(p(x), 2, 4096, p(fill), 2, None, 0, None, p(x), 4096, None, 0, None, p(ev), None) == -EINVAL
    assert push(C.c_void_p(x.data_ptr() + 4), 2, 4092, p(fill), 2, None, 0, p(st), p(x), 4096, None, 0, None,
                p(ev), None) == -EINVAL
    assert mm().launch_count() == n0
    assert push(p(x), 0, 4096, p(fill), 2, None, 0, p(st), p(x), 4096, None, 0, None, p(ev), None) == 0
    assert mm().launch_count() == n0
