"""Case and signal builders that more than one rx test file uses: random framings, tone pairs and their
streams, tone-pair channel rows, the launch-shape and carrier-session cases, the live-receiver drivers and
the reference vectors through rx_batch.  Every builder seeds as it always has, so a case is the same array in
every file and every session."""
import copy
import os
import re
import zlib

import numpy as np

import autoorc
import golden_util as gu
import gpudev
import minimodem_b200 as mm
import orc
import refcases
import rxfam
import tie_screen
from gpudev import dev, pcm, sync, upload

f32 = np.float32
BAUDS = [75, 110, 150, 300, 600, 1200, 2400, 4800]
RATES = [8000, 11025, 16000, 22050, 44100, 48000]

_SHAPE_CASES = {}
_SESSION_CASES = {}
_DUPLEX = []


# ---------------------------------------------------------------------------------------------------
# random framings (test_gpu_instantiations' classes: "short", "tile" and "long" bit periods)
# ---------------------------------------------------------------------------------------------------
PAIRS = {"short": [(b, r) for b in BAUDS for r in RATES if 10 <= r / b <= 60],
         "tile": [(600, 48000), (300, 48000), (1200, 48000)],
         "long": [(25, 48000), (20, 44100)]}


def framing(cls, n, seed):
    """(mode, kw, expect override or None): a random framing of class `cls` whose expect string has n
    windows -- its own if it has n, else its own cut to n or continued with don't-care windows"""
    rng = np.random.default_rng(seed)
    pairs = PAIRS[cls]
    while True:
        baud, rate = pairs[int(rng.integers(0, len(pairs)))]
        kw = dict(sample_rate=rate)
        kw["n_data_bits"] = int(rng.choice([5, 6, 7, 8, 9, 12, 16] if n < 24 else [n - 8, n - 6, n - 4]))
        kw["startbits"] = int(rng.choice([1, 1, 2]))
        kw["stopbits"] = float(rng.choice([1.0, 1.0, 1.5, 2.0]))
        kw["msb_first"] = bool(rng.integers(0, 2))
        kw["invert_start_stop"] = bool(rng.integers(0, 2))
        kw["inverted"] = bool(rng.integers(0, 2))
        if cls == "tile" and kw["stopbits"] == 1.5:
            continue
        try:
            m = orc.Mode(str(baud), **kw)
            d = m.derived()
            orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
        except Exception:
            continue
        if max(m.mark_f, m.space_f) >= rate / 2 - m.band_width:
            continue
        own = bytes(d.expect_data)
        exp = None if len(own) == n else (own[:n] if len(own) > n else own + b"d" * (n - len(own)))
        return str(baud), kw, exp


def oracle_mode(mode, kw, exp):
    m = orc.Mode(mode, **kw)
    m.expect_data_string = exp
    return m


def engine(mode, kw, exp):
    names = dict(startbits="nstartbits", stopbits="nstopbits")
    ov = {names.get(k, k): v for k, v in kw.items() if k != "sample_rate"}
    cfg = mm.rx_config_for_mode(mode, kw.get("sample_rate", 48000), **ov)
    if exp is not None:
        cfg.expect_data_string = exp
    return mm.RxEngine(mm.rx_params(cfg))


# ---------------------------------------------------------------------------------------------------
# tone pairs
# ---------------------------------------------------------------------------------------------------
# (G, W, L) of AUTO_COMBOS -> a preset (mode, sample rate) whose per-stream-table launch shape it is
COVER = {
    (8, 3, 2): ("1200", 48000),
    (16, 2, 4): ("rtty", 8000),
    (16, 3, 4): ("300", 48000),
    (16, 3, 1): ("uic-train", 8000),
    (32, 1, 4): ("rtty", 48000),
    (32, 2, 4): ("110", 48000),
    (32, 3, 2): ("uic-ground", 48000),
}


KEYS = sorted(COVER)


def auto_combos():
    """the (G, W, L) shapes of the kernel source's AUTO_COMBOS list"""
    src = open(os.path.join(gpudev.ROOT, "minimodem_b200", "csrc", "fsk_b200_kernels.cu")).read()
    m = re.search(r"#define AUTO_COMBOS\(X\)((?:[^\n]*\\\n)*[^\n]*)", src)
    return {tuple(int(v) for v in t) for t in re.findall(r"X\((\d+), (\d+), (\d+)\)", m.group(1))}


# the presets of the tone calls
TONE_PRESETS = ["rtty", "tdd", "same", "callerid", "uic-train", "uic-ground", "V.21", "2400", "1200", "600", "300",
           "110", "12000", "45.45"]


# Bell103 full duplex
ORIGINATE, ANSWER = (1270.0, 1070.0), (2225.0, 2025.0)


def on_pair(mode, rate, mark, space):
    """orc.Mode of `mode` on the tone pair (mark, space), also for the presets whose tones the CLI fixes"""
    m = orc.Mode(mode, sample_rate=rate)
    m.mark_f, m.space_f = f32(mark), f32(space)
    return m


def fsk_audio(bits, spb, mark, space, rate, amplitude):
    """Phase-continuous FSK: sample i carries bit floor(i / spb), at the exact (fractional) bit period."""
    n = int(len(bits) * spb)
    b = np.asarray(bits, np.int64)[np.minimum((np.arange(n) / spb).astype(np.int64), len(bits) - 1)]
    f = np.where(b == 1, mark, space)
    return (amplitude * np.sin(2 * np.pi * np.cumsum(f) / rate)).astype(np.float32)


def transmission(rng, m, nwords, amplitude):
    """nwords random data words on m's tones: the oracle's transmitter, or for UIC (expect string 11110010
    and 39 data bits, no start or stop bits) synthesised frames after a mark leader"""
    if m.expect_data_string is not None:
        bits = [1] * 10
        for _ in range(nwords):
            bits += [1, 1, 1, 1, 0, 0, 1, 0] + [int(v) for v in rng.integers(0, 2, 39)]
        bits += [1] * 2
        return fsk_audio(bits, float(m.sample_rate) / float(m.data_rate), float(m.mark_f), float(m.space_f),
                         m.sample_rate, amplitude)
    words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
    return orc.tx_words(m, words, amplitude, 4096, True)


def random_pair(rng, bw, nbands):
    """independent mark and space bands, either order, at least two bands apart; each tone up to 0.3 band
    off its band's centre"""
    while True:
        bm, bs = (int(v) for v in rng.integers(2, nbands - 2, 2))
        if abs(bm - bs) >= 2:
            break
    return float(f32((bm + rng.uniform(-0.3, 0.3)) * bw)), float(f32((bs + rng.uniform(-0.3, 0.3)) * bw))


def lay_out(rng, m, audio, sigma):
    lead = np.zeros(int(rng.integers(0, 3 * m.derived().frame_nsamples)), np.float32)
    tail = np.zeros(int(rng.integers(0, m.derived().frame_nsamples)), np.float32)
    x = np.concatenate([lead, audio, tail])
    return (x + f32(sigma) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32), lead.size


def duplex_case():
    """six Bell103 streams, originate and answer in turn, then one line carrying both directions, given once
    with each pair: (streams, pairs, the oracle's result per stream)"""
    if _DUPLEX:
        return _DUPLEX[0]
    rng = np.random.default_rng(103)
    mo, ma = on_pair("300", 48000, *ORIGINATE), on_pair("300", 48000, *ANSWER)
    streams, pairs = [], []
    for s in range(6):
        m = mo if s % 2 == 0 else ma
        x, _ = lay_out(rng, m, transmission(rng, m, int(rng.integers(5, 9)), float(rng.uniform(0.3, 1.0))), 1e-3)
        streams.append(x)
        pairs.append(ORIGINATE if s % 2 == 0 else ANSWER)
    # one line carrying both directions at once, given twice: once with each pair
    a, b = transmission(rng, mo, 8, 0.5), transmission(rng, ma, 8, 0.5)
    both = np.zeros(max(a.size, b.size) + 2000, np.float32)
    both[1000:1000 + a.size] += a
    both[1500:1500 + b.size] += b
    streams += [both, both]
    pairs += [ORIGINATE, ANSWER]
    want = [orc.rx_run(on_pair("300", 48000, *p), x, literal=False) for x, p in zip(streams, pairs)]
    _DUPLEX.append((streams, pairs, want))
    return _DUPLEX[0]


def tone_mark(rng, m, b_shift, nbands):
    """a random mark tone of this mode's band grid whose space band (b_shift away) lies inside it, off its band
    centre by up to 0.3 band"""
    bw = float(m.band_width)
    lo, hi = max(2, 2 - b_shift), min(nbands - 3, nbands - 3 - b_shift)
    bm = int(rng.integers(lo, max(lo + 1, hi)))
    return float(bm * bw + rng.uniform(-0.3, 0.3) * bw)


def tone_burst(rng, m, mark, b_shift, nwords, amplitude, space=None):
    """nwords random data words on (mark, space = mark + b_shift bands).  UIC frames (the expect string
    11110010 and 39 data bits, no start or stop bits) come from fsk_audio after a mark leader; everything
    else from the oracle's transmitter."""
    space = mark + b_shift * float(m.band_width) if space is None else space
    if m.expect_data_string is not None:
        bits = [1] * 10
        for _ in range(nwords):
            bits += [1, 1, 1, 1, 0, 0, 1, 0] + [int(v) for v in rng.integers(0, 2, 39)]
        bits += [1] * 2
        return fsk_audio(bits, float(m.sample_rate) / float(m.data_rate), mark, space, m.sample_rate, amplitude)
    tx = orc.Mode(m.mode, sample_rate=m.sample_rate, mark=mark, space=space)
    tx.do_tx_sync_bytes = min(tx.do_tx_sync_bytes, m.do_tx_sync_bytes)
    words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
    return orc.tx_words(tx, words, amplitude, 4096, True)


def tone_stream(rng, m, b_shift, nbands, nwords):
    """One transmission of random data words on a random tone pair of this mode's band grid (tone_mark,
    tone_burst)."""
    mark = tone_mark(rng, m, b_shift, nbands)
    return tone_burst(rng, m, mark, b_shift, nwords, float(rng.uniform(0.3, 1.0)))


# ---------------------------------------------------------------------------------------------------
# tone-pair channels over shared rows
# ---------------------------------------------------------------------------------------------------
def disabled_pair(rng, nb):
    return [[nb, 5], [5, nb], [0xFFFFFFFF, 0xFFFFFFFF]][int(rng.integers(3))]


def channel_rows(mode, rate, nrows, k, seed):
    """nrows rows, each the sum of min(k, 2) transmissions on random valid pairs with lead-ins and AWGN;
    k pairs per row: the row's signals first, then random valid pairs or disabled ones (k >= 3 has at least
    one disabled channel per row).  Returns (streams, lengths, bands [nrows*k][2] uint32)."""
    rng = np.random.default_rng(seed)
    eng = mm.RxEngine.for_mode(mode, rate)
    bw, nb = float(eng.params.band_width), int(eng.params.nbands)
    streams, lens, bands = [], [], []
    for r in range(nrows):
        pairs = [random_pair(rng, bw, nb) for _ in range(min(k, 2))]
        x = np.zeros(0, np.float32)
        for fm, fs in pairs:
            m = on_pair(mode, rate, fm, fs)
            a, _ = lay_out(rng, m, transmission(rng, m, int(rng.integers(3, 6)), float(rng.uniform(0.3, 0.8))),
                              0.0)
            if a.size > x.size:
                a, x = x, a
            x = x.copy()
            x[:a.size] += a
        x = (x + f32(rng.uniform(1e-4, 2e-3)) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
        lens.append(x.size if r else int(x.size * 0.7))          # row 0 cut short of its stride
        row = [list(mm.tone_bands(eng.params, *p)) for p in pairs]
        for j in range(len(pairs), k):
            if j == len(pairs) or rng.random() < 0.4:
                row.append(disabled_pair(rng, nb))
            else:
                row.append(list(mm.tone_bands(eng.params, *random_pair(rng, bw, nb))))
        bands += row
    return streams, np.array(lens, np.int32), np.array(bands, np.uint32)


def run_channels(eng, buf, n, lens, bands, k, states=None, max_frames=None, per_row=True):
    fr, st = eng.rx_batch_tones(upload(buf), bands, nsamples=n, nsamples_each=upload(lens) if per_row else None,
                                states=states, max_frames=max_frames, channels_per_row=k)
    sync()
    return fr, st


def check_channels_against_oracle(eng, mode, rate, lines, pairs_per_row, k, what):
    """pairs_per_row: per row, k (mark Hz, space Hz) pairs.  Every channel against the screened oracle on
    its row and pair; the device decoder's text against the oracle's for every robust channel."""
    flat = [p for ps in pairs_per_row for p in ps]
    bands = eng.tone_bands([p[0] for p in flat], [p[1] for p in flat], device=dev())
    buf, n = gpudev.rows(lines, np.float32, 4)
    lens = np.array([a.size for a in lines], np.int32)
    frames, states = run_channels(eng, buf, n, lens, bands, k)
    assert eng.last_kernel().endswith(" channels=%d" % k), eng.last_kernel()
    screened = [tie_screen.screen(on_pair(mode, rate, *p), lines[c // k]) for c, p in enumerate(flat)]
    fr, st = mm.frames_to_numpy(frames), mm.states_to_numpy(states)
    assert (st["done"] == 1).all()
    rxfam.check_against_oracle(screened, fr, st, what)
    out, cnt = eng.decode_batch(mm.decoder_for_mode(mode, int(eng.params.n_data_bits)), frames, states)
    sync()
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    rx = orc.Mode(mode, sample_rate=rate)
    texts = []
    for c, (w, robust) in enumerate(screened):
        texts.append(out[c, :cnt[c]].tobytes())
        if robust:
            assert texts[-1] == orc.decode_records(rx, rx.decoder, orc.frame_records(w["frames"])), (what, c)
    return texts


def push_model(rows_, fill, states, k, bands, nbands, chunk, clen):
    rows_, fill, states = rows_.copy(), fill.copy(), states.copy()
    dropped = np.zeros(len(fill), np.int64)
    stride = rows_.shape[1]
    for r in range(len(fill)):
        have = int(fill[r])
        ch = range(r * k, r * k + k)
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
            states["done"][c] = 0
    return rows_, fill, states, dropped


def random_states(rng, n, fill, k):
    st = np.frombuffer(rng.integers(0, 2**32, n * mm.STATE_WORDS, dtype=np.uint64).astype(np.uint32).tobytes(),
                       mm.STATE_DTYPE).copy()
    for c in range(n):
        have = int(fill[c // k])
        u = rng.random()
        st["pos"][c] = (int(rng.integers(0, have + 1)) if u < 0.7 else
                        have + int(rng.integers(1, 1000)) if u < 0.9 else int(rng.integers(2**32, 2**40)))
    return st


# ---------------------------------------------------------------------------------------------------
# the launch-shape cases (test_gpu_launch_shapes) and the carrier-session cases (test_gpu_carrier_sessions)
# ---------------------------------------------------------------------------------------------------
def shape_case(fam, which):
    """(engine factory, streams, lengths, per-stream tone bands or None, oracle Mode) for a family and a
    preset (mode, rate) or "random".  6 streams: ragged lead-ins, sigma = 0.01 noise (1e-4 for the auto
    call, whose streams start with silence longer than the deepest ring), every third stream drops the
    carrier and finds it again, the last one is cut mid-frame.  Computed once per (call, which)."""
    f = rxfam.FAMILIES[fam]
    key = (f["call"], f.get("cls"), f.get("n"), which)
    if key in _SHAPE_CASES:
        return _SHAPE_CASES[key]
    rng = np.random.default_rng(zlib.crc32(repr(key).encode()))
    if which == "random":
        mode, kw, exp = framing(f["cls"], f["n"], 7000 + f["n"])
        m = oracle_mode(mode, kw, exp)
        make = lambda: engine(mode, kw, exp)
    else:
        mode, rate = which
        m = orc.Mode(mode, sample_rate=rate)
        make = lambda: mm.RxEngine.for_mode(mode, rate)
    spb = float(m.derived().nsamples_per_bit)
    streams, bands = [], []
    probe = make()
    p = probe.params
    nb = int(p.nbands)
    for s in range(6):
        if f["call"] == "auto":
            bs = autoorc.b_shift(m)
            parts = [np.zeros(int(rng.integers(20000, 26000)), np.float32), tone_stream(rng, m, bs, nb, 5)]
            if s % 3 == 1:
                parts += [np.zeros(int(rng.uniform(30, 50) * spb), np.float32), tone_stream(rng, m, bs, nb, 4)]
            sigma = 1e-4
        else:
            tm = m
            if f["call"] == "tones":
                fm, fs = random_pair(rng, float(m.band_width), nb)
                bands.append([int(v) for v in mm.tone_bands(p, fm, fs)])
                tm = on_pair(m.mode, m.sample_rate, fm, fs)
                tm.__dict__.update({k: v for k, v in m.__dict__.items() if k not in ("mark_f", "space_f")})
            words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
            parts = [np.zeros(int(rng.integers(0, 3 * spb + 1)), np.float32),
                     orc.tx_words(tm, words(int(rng.integers(6, 10))), float(rng.uniform(0.3, 1.0)), 4096, True)]
            if s % 3 == 1:
                parts += [np.zeros(int(rng.uniform(20, 40) * spb), np.float32),
                          orc.tx_words(tm, words(4), float(rng.uniform(0.3, 1.0)), 4096, True)]
            sigma = 0.01
        x = np.concatenate(parts)
        if s == 5:
            x = x[:int(x.size * rng.uniform(0.6, 0.9))]
        x = (x + np.float32(sigma) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        streams.append(x)
    _SHAPE_CASES[key] = (make, streams, np.array([x.size for x in streams], np.int32), bands or None, m)
    return _SHAPE_CASES[key]


SIGMA_BG = 0.003
# the auto call's background: a gap stays silent to the carrier scan (at 0.003 a scan window's largest band
# sits near the 0.001 threshold, and a gap turns into a run of threshold near-ties)
SIGMA_BG_AUTO = 1e-4
NOISE_SIGMAS = (0.05, 0.2, 0.5)
NSTREAMS = 8
KINDS = ("burst", "gap", "noise", "fade", "sag", "cut")
# the auto call's own: a burst on one pair followed directly by one on another pair, and a burst whose space
# band lies outside the band grid (the scan finds it and rejects it)
AUTO_KINDS = ("retune", "low")


def session_stream(rng, m, end_in_gap, auto=None):
    """(samples, noise-only ranges [(start, end)]): every kind of segment once (noise twice) and up to two more, in
    random order, under sigma = 0.003 background.  auto = (b_shift, nbands): the auto call's stream -- every
    burst on its own random pair of the band grid, the AUTO_KINDS too, sigma = 1e-4 background."""
    spb = float(m.derived().nsamples_per_bit)
    words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
    # a burst of 3..10 frames; SAME's counts its one sync byte (the transmitter's preamble is 16 of them)
    tm = copy.copy(m)
    tm.do_tx_sync_bytes = min(m.do_tx_sync_bytes, 1)
    if auto is None:
        burst = lambda amp: orc.tx_words(tm, words(int(rng.integers(3, 11)) - tm.do_tx_sync_bytes), amp, 4096, True)
        kinds = KINDS + ("noise",)
    else:
        bs, nb = auto
        pair_burst = lambda mark, amp: tone_burst(rng, tm, mark, bs, int(rng.integers(3, 11)) - tm.do_tx_sync_bytes,
                                                  amp)
        burst = lambda amp: pair_burst(tone_mark(rng, m, bs, nb), amp)
        kinds = KINDS + ("noise",) + AUTO_KINDS
    parts, noise, at = [], [], 0
    kinds = list(rng.permutation(kinds)) + list(rng.choice(KINDS, int(rng.integers(0, 3))))
    kinds.append("gap" if end_in_gap else "burst")
    for kind in kinds:
        amp = float(rng.uniform(0.2, 1.0))
        if kind == "gap":
            a = np.zeros(int(rng.uniform(1, 60) * spb), np.float32)
        elif kind == "noise":           # long enough to acquire a false carrier in every preset's case; longer
            # ones pile up near-ties of the threshold and the search limit on noise candidates (the auto call's
            # at most 60 bits: every strike there rescans, and 120 screened out more than one stream in ten)
            a = (float(rng.choice(NOISE_SIGMAS)) * rng.standard_normal(int(rng.uniform(20, 120 if auto is None else 60)
                                                                           * spb))).astype(np.float32)
            noise.append((at, at + a.size))
        elif kind == "fade":            # squelched at 1/8..1/5 of the level, held at 1/3
            ratio = float(rng.uniform(1 / 8, 1 / 5)) if rng.random() < 0.6 else 1 / 3
            if auto is None:
                a = np.concatenate([burst(amp), burst(amp * ratio)])
            else:                       # on one pair
                mark = tone_mark(rng, m, bs, nb)
                a = np.concatenate([pair_burst(mark, amp), pair_burst(mark, amp * ratio)])
        elif kind == "sag":             # a noise burst at the signal's level inside a running burst
            a = burst(amp)
            n = int(rng.uniform(2, 6) * spb)
            p = int(rng.integers(a.size // 4, a.size // 2))
            a[p:p + n] += (0.7 * amp * rng.standard_normal(a[p:p + n].size)).astype(np.float32)
        elif kind == "cut":
            a = burst(amp)
            a = a[:int(rng.integers(a.size // 3, a.size))]
        elif kind == "retune":
            a = np.concatenate([burst(amp), burst(float(rng.uniform(0.2, 1.0)))])
        elif kind == "low":             # the space band below band 1, or past the last band
            bw = float(m.band_width)
            bm = int(rng.integers(1, 1 - bs + 1)) if bs < 0 else int(rng.integers(nb - bs, nb - 1))
            mark = float(bm * bw + rng.uniform(-0.3, 0.3) * bw)
            space = min(max(mark + bs * bw, -mark), float(m.sample_rate) / 2 - bw)
            a = tone_burst(rng, tm, mark, bs, int(rng.integers(3, 11)) - tm.do_tx_sync_bytes, amp, space=space)
        else:
            a = burst(amp)
        parts.append(a)
        at += a.size
    x = np.concatenate(parts)
    sigma = SIGMA_BG if auto is None else SIGMA_BG_AUTO
    return (x + f32(sigma) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32), noise


def drops(m, x, auto=False, inverted=False):
    """carrier drops (session reports before the end of the stream) of the oracle (the auto oracle) on x"""
    r = autoorc.rx_run(m, x, inverted=inverted) if auto else orc.rx_run(m, x, literal=False)
    return len(r["reports"]) - (1 if r["reports"] and r["reports"][-1][4] == len(r["frames"]) else 0)


def bisect_gap(make, dropped, hi):
    """the two gap lengths one sample either side of the drop: (make(lo), make(lo + 1))"""
    lo = 0
    assert not dropped(0) and dropped(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if dropped(mid):
            hi = mid
        else:
            lo = mid
    return make(lo), make(hi)


def boundary_streams(m, seed):
    """Two streams burst + silent gap + burst whose gaps are the longest without a carrier drop and the
    shortest with one (a bisection on the gap length on the oracle)."""
    rng = np.random.default_rng(seed)
    words = lambda k: rng.integers(0, 1 << m.n_data_bits, k, dtype=np.uint64).astype(np.uint32)
    a, b = orc.tx_words(m, words(4), 0.6, 4096, True), orc.tx_words(m, words(3), 0.6, 4096, True)
    hi = int(80 * float(m.derived().nsamples_per_bit))
    bg = (f32(SIGMA_BG) * rng.standard_normal(a.size + b.size + hi)).astype(np.float32)
    make = lambda gap: (np.concatenate([a, np.zeros(gap, np.float32), b]) + bg[:a.size + gap + b.size]).astype(np.float32)
    return bisect_gap(make, lambda gap: drops(m, make(gap)) > 0, hi)


def auto_drop_in_gap(m, x, gap_end, inverted=False):
    """the auto oracle on x drops a carrier (the 21st strike) and rescans before sample gap_end"""
    r = autoorc.rx_run(m, x, inverted=inverted, scans=True)
    return any(e["cause"] == "after-drop" and e["pos"] <= gap_end for e in r["scans"])


def auto_boundary_streams(m, b_shift, nbands, inverted, seed, same_pair):
    """boundary_streams for the auto call, the second burst on the first one's pair or on another: the gaps one
    sample either side of the one whose carrier drop comes before the second burst starts.  Returns the two
    streams and where their gaps end."""
    rng = np.random.default_rng(seed)
    ma = tone_mark(rng, m, b_shift, nbands)
    while True:
        mb = ma if same_pair else tone_mark(rng, m, b_shift, nbands)
        if same_pair or abs(mb - ma) > 2 * float(m.band_width):
            break
    a, b = tone_burst(rng, m, ma, b_shift, 4, 0.6), tone_burst(rng, m, mb, b_shift, 3, 0.6)
    hi = int(80 * float(m.derived().nsamples_per_bit))
    bg = (f32(SIGMA_BG_AUTO) * rng.standard_normal(a.size + b.size + hi)).astype(np.float32)
    make = lambda gap: (np.concatenate([a, np.zeros(gap, np.float32), b]) + bg[:a.size + gap + b.size]).astype(np.float32)
    short, past = bisect_gap(make, lambda gap: auto_drop_in_gap(m, make(gap), a.size + gap, inverted), hi)
    gap = short.size - a.size - b.size
    return short, past, a.size + gap, a.size + gap + 1


class Case:
    """channels (one per stream, or per (row, pair) for the channel call): oracle modes, rows, lengths, tone
    bands, the oracle's results with the screen's verdicts, noise ranges; `make` builds the engine"""


def session_case(f, which):
    """the carrier-session Case of family `f` (a registry entry, `call` "channels" for k = 2 channels per row)
    and a preset (mode, rate) or "random"; computed once per (call, src, which)"""
    call = "tones" if f["call"] == "channels" else f["call"]
    key = (f["call"], f["src"], which) if which != "random" else (f["call"], f["src"], f["cls"], f["n"])
    if f.get("inverted"):
        key += ("inverted",)
    if key in _SESSION_CASES:
        return _SESSION_CASES[key]
    seed = key[:1] + key[2:]                    # int16 rows: the float streams, quantized
    rng = np.random.default_rng(zlib.crc32(repr(("sessions",) + seed).encode()))
    c = Case()
    if which == "random":
        mode, kw, exp = framing(f["cls"], f["n"], 7000 + f["n"])
        m = oracle_mode(mode, kw, exp)
        c.make = lambda: engine(mode, kw, exp)
        c.mode, c.rate = mode, kw["sample_rate"]
    else:
        c.mode, c.rate = which
        m = orc.Mode(c.mode, sample_rate=c.rate)
        inv = dict(inverted=True) if f.get("inverted") else {}
        c.make = lambda: mm.RxEngine.for_mode(which[0], which[1], **inv)
    k = 2 if f["call"] == "channels" else 1
    c.inverted = bool(f.get("inverted", False))
    auto = None
    if call == "auto":
        p = mm.rx_params(mm.rx_config_for_mode(c.mode, c.rate))
        auto = (autoorc.b_shift(m, c.inverted), int(p.nbands))
    nch = NSTREAMS + (2 if auto is None else 4) if k == 1 else 2 * (NSTREAMS // 2 + 2)
    c.modes, c.hz, c.bands, c.noise, chans = [], [], [], [], []
    if call == "tones":
        p = mm.rx_params(mm.rx_config_for_mode(c.mode, c.rate))
        nb = int(p.nbands)
        for j in range(nch):
            fm, fs = random_pair(rng, float(m.band_width), nb)
            c.hz.append((fm, fs))
            c.bands.append([int(v) for v in mm.tone_bands(p, fm, fs)])
            tm = on_pair(m.mode, m.sample_rate, fm, fs)
            tm.__dict__.update({kk: v for kk, v in m.__dict__.items() if kk not in ("mark_f", "space_f")})
            c.modes.append(tm)
    else:
        c.modes = [m] * nch
    for j in range(NSTREAMS if auto else nch):
        chans.append(session_stream(rng, c.modes[j], j % 2 == 0, auto))
    if auto is not None:
        # the boundary streams: channels 8, 9 (the second burst on the first one's pair) and 10, 11 (on another)
        c.boundary, c.gap_end = [], {}
        for same in (True, False):
            short, past, e0, e1 = auto_boundary_streams(m, auto[0], auto[1], c.inverted,
                                                        zlib.crc32(repr(seed).encode()) + same, same)
            c.boundary += [(len(chans), 0), (len(chans) + 1, 1)]
            c.gap_end.update({len(chans): e0, len(chans) + 1: e1})
            chans += [(short, []), (past, [])]
    else:
        # the boundary streams: channels 8 and 9 (k = 1), or alone on rows 4 and 5 (k = 2)
        nb_at = [NSTREAMS, NSTREAMS + 1] if k == 1 else [NSTREAMS, NSTREAMS + 3]
        short, _ = boundary_streams(c.modes[nb_at[0]], zlib.crc32(repr(seed).encode()))
        _, past = boundary_streams(c.modes[nb_at[1]], zlib.crc32(repr(seed).encode()) + 1)
        chans[nb_at[0]] = (short, [])
        chans[nb_at[1]] = (past, [])
        c.boundary = [(nb_at[0], 0), (nb_at[1], 1)]
    if k == 2:
        for j in (NSTREAMS + 1, NSTREAMS + 2):      # the other channel of those rows carries nothing
            chans[j] = (np.zeros(1, np.float32), [])
    c.k = k
    c.rows = []
    for r in range(nch // k):
        xs = [chans[r * k + j][0] for j in range(k)]
        x = np.zeros(max(v.size for v in xs), np.float32)
        for v in xs:
            x[:v.size] += v
        c.rows.append(x)
    if f["src"] == "s16":                       # what the int16 rows carry, exactly
        c.rows = [pcm(x).astype(np.float32) / f32(32768) for x in c.rows]
    c.noise = [ch[1] for ch in chans]
    c.lens = np.array([x.size for x in c.rows], np.int32)
    c.row_of = [j // k for j in range(nch)]
    c.auto = auto
    if auto is None:
        c.screened = [tie_screen.screen(c.modes[j], c.rows[c.row_of[j]]) for j in range(nch)]
    else:
        c.screened = [autoorc.screen(m, x, c.inverted) for x in c.rows]
    _SESSION_CASES[key] = c
    return c


# ---------------------------------------------------------------------------------------------------
# live-receiver drivers
# ---------------------------------------------------------------------------------------------------
def cuts(rng, n, max_chunk):
    """random chunk sizes summing to n, some of them a handful of samples"""
    out = []
    while n > 0:
        c = int(rng.integers(1, 9)) if rng.random() < 0.25 else int(rng.integers(1, max_chunk + 1))
        out.append(min(c, n))
        n -= out[-1]
    return out


def call_audio(rng, m, nwords):
    if m.mode == "callerid":        # an SDMF message: type, length, date and time, number (decoded on its last byte)
        digits = [ord("0") + int(d) for d in rng.integers(0, 10, 8 + 10)]
        words = np.array([0x04, 18] + digits, np.uint32)
    else:
        words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([np.zeros(int(rng.integers(0, 3 * m.derived().frame_nsamples)), np.float32),
                        orc.tx_words(m, words, float(rng.uniform(0.3, 0.9)), 4096, True),
                        np.zeros(int(rng.integers(0, 2 * m.derived().frame_nsamples)), np.float32)])
    return (x + np.float32(3e-3) * rng.standard_normal(x.size)).astype(np.float32)


def duplex_audio(rng, nwords):
    mo, ma = on_pair("300", 48000, *ORIGINATE), on_pair("300", 48000, *ANSWER)
    a, b = call_audio(rng, mo, nwords), call_audio(rng, ma, nwords)
    x = np.zeros(max(a.size, b.size), np.float32)
    x[:a.size] += a
    x[:b.size] += b
    return x


def one_pass_text(mode, rate, rows, pairs, k, auto):
    """one rx call of the live receiver's family over the whole rows, decoded from fresh decoder state"""
    eng = mm.RxEngine.for_mode(mode, rate)
    buf, _ = gpudev.rows(rows, rows[0].dtype, 8)
    x = upload(buf)
    lens = upload(np.array([r.size for r in rows], np.int32))
    if pairs is not None:
        tb = eng.tone_bands([p[0] for p in pairs], [p[1] for p in pairs], device=dev())
        fr, st = eng.rx_batch_tones(x, tb, nsamples=buf.shape[1], nsamples_each=lens, channels_per_row=k)
    elif auto:
        eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
        fr, st, _ = eng.rx_batch_auto(x, nsamples=buf.shape[1], nsamples_each=lens)
    else:
        fr, st = eng.rx_batch(x, nsamples=buf.shape[1], nsamples_each=lens)
    out, cnt = eng.decode_batch(mm.decoder_for_mode(mode, int(eng.params.n_data_bits)), fr, st)
    sync()
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    return [out[s, :int(cnt[s])].tobytes() for s in range(len(cnt))]


def live_text(mode, rate, rows, pairs, k, auto, max_chunk, seed, cuts_at=(), pcm16=False):
    """LiveReceiver fed the rows in random chunks (a cut at every sample of `cuts_at`: (row, sample))"""
    from minimodem_b200.serving import LiveReceiver
    kw = {}
    if pairs is not None:
        eng = mm.RxEngine.for_mode(mode, rate)
        kw = dict(tones=eng.tone_bands([p[0] for p in pairs], [p[1] for p in pairs], device=dev()),
                  channels_per_row=k)
    if auto:
        kw = dict(auto_carrier=autoorc.DEFAULT_THRESHOLD)
    lr = LiveReceiver(mode, rate, len(rows), max_chunk=max_chunk, device=dev(), pcm16=pcm16, **kw)
    rng = np.random.default_rng(seed)
    cuts = []
    for r, x in enumerate(rows):
        c = set(int(v) for v in np.cumsum(rng.integers(1, max_chunk + 1, x.size // 2 + 2)) if v < x.size)
        c |= {p for rr, p in cuts_at if rr == r}
        c = sorted(c | {x.size})
        cuts.append([b - a for a, b in zip([0] + c, c)])
    assert all(max(v) <= max_chunk for v in cuts)
    nch = len(rows) * k
    texts = [b""] * nch

    def take(res):
        o, n = res
        o, n = o.cpu().numpy(), n.cpu().numpy()
        for s in range(nch):
            texts[s] += o[s, :int(n[s])].tobytes()
    fed = [0] * len(rows)
    for step in range(max(len(v) for v in cuts)):
        chunk = np.zeros((len(rows), max_chunk), rows[0].dtype)
        k_ = np.zeros(len(rows), np.int32)
        for r, x in enumerate(rows):
            if step < len(cuts[r]):
                k_[r] = cuts[r][step]
                chunk[r, :k_[r]] = x[fed[r]:fed[r] + k_[r]]
                fed[r] += int(k_[r])
        take(lr.feed(upload(chunk), upload(k_)))
    take(lr.finish())
    return texts


def records_of(frames, states, bands):
    """per stream: [(record bytes, band)] of the records an auto call wrote"""
    fr, st, b = mm.frames_to_numpy(frames), mm.states_to_numpy(states), bands.cpu().numpy()
    return [[(fr[s, i].tobytes(), int(b[s, i])) for i in range(int(st["nframes"][s]))] for s in range(len(st))]


def live_records(eng, streams, cut, cuts_at=()):
    """The live-stream recipe of include/fsk_b200.h with auto-carrier (eng: set_auto_carrier done):
    fsk_b200_stream_push, then fsk_b200_rx_batch_auto with the auto holdback, chunk by chunk -- chunks of
    `cut` samples, also cut at every sample of `cuts_at` --, the holdback off for the last call.  streams:
    float32 or int16.  Returns every stream's records and bands in order."""
    t = gpudev.torch()
    window = eng.auto_stream_window()
    eng.set_holdback(window)
    stride = (window + eng.params.frame_nsamples + cut + 7) & ~7
    max_frames = eng.max_frames(stride)
    S = len(streams)
    dt = t.int16 if streams[0].dtype == np.int16 else t.float32
    buf, n = gpudev.rows(streams, streams[0].dtype, 8)
    lens = np.array([len(a) for a in streams], np.int64)
    z = lambda shape, d: t.zeros(shape, dtype=d).to(dev())
    rows_, fill = z((S, stride), dt), z((S,), t.int32)
    states, auto = z((S, mm.STATE_WORDS), t.int32), z((S, mm.AUTO_STATE_BYTES), t.uint8)
    dropped = z((S,), t.int32)
    got = [[] for _ in streams]

    def step(chunk, valid):
        mm.stream_push(rows_, fill, states, chunk, valid, dropped=dropped)
        frames, _, _, bands = eng.rx_batch_auto(rows_, nsamples=stride, nsamples_each=fill, max_frames=max_frames,
                                                states=states, auto_states=auto, rec_band=True)
        sync()
        for s, r in enumerate(records_of(frames, states, bands)):
            got[s] += r
    at = sorted(set(range(0, n, cut)) | {int(p) for p in cuts_at if 0 < p < n})
    for o, e in zip(at, at[1:] + [n]):
        w = e - o
        step(upload(np.ascontiguousarray(buf[:, o:o + w])), upload(np.clip(lens - o, 0, w).astype(np.int32)))
    eng.set_holdback(0)
    step(z((S, 8), dt), 0)
    assert int(dropped.cpu().numpy().sum()) == 0
    return got


# ---------------------------------------------------------------------------------------------------
# the reference vectors through rx_batch
# ---------------------------------------------------------------------------------------------------
def engine_for(case_or_mode, rx=True):
    if isinstance(case_or_mode, dict):
        mode, kw = case_or_mode["rx_mode"], case_or_mode["rx_mkw"]
    else:
        mode, kw = case_or_mode
    names = dict(mark="f_mark", space="f_space", bandwidth="band_width", startbits="nstartbits",
                 stopbits="nstopbits", confidence="confidence_threshold", limit="confidence_search_limit")
    ov = {names.get(k, k): v for k, v in kw.items() if k not in ("sample_rate", "baudot")}
    if kw.get("baudot"):            # the -5 option
        ov["n_data_bits"] = 5
    cfg = mm.rx_config_for_mode(mode, kw.get("sample_rate", 48000), **ov)
    return mm.RxEngine(mm.rx_params(cfg)), cfg


def pad4(n):
    return (n + 3) & ~3


def rx_on_gpu(eng, streams, lanes=0):
    """streams: list of 1-D float32 arrays -> list of frame-record arrays."""
    n = max(len(a) for a in streams)
    stride = pad4(n)
    buf = np.zeros((len(streams), stride), np.float32)
    lens = np.zeros(len(streams), np.int32)
    for i, a in enumerate(streams):
        buf[i, :len(a)] = a
        lens[i] = len(a)
    if lanes:
        eng.tune(lanes_per_stream=lanes)
    frames, states = eng.rx_batch(upload(buf), nsamples=n, nsamples_each=upload(lens))
    sync()
    fr = mm.frames_to_numpy(frames)
    st = mm.states_to_numpy(states)
    assert (st["done"] == 1).all()
    return [fr[i, :st["nframes"][i]] for i in range(len(streams))], st


def check_reference_vector(case):
    """one reference vector through rx_batch: the oracle's records, the reference's decoded bytes (where the
    reference is built) and its stat line"""
    g = gu.load(case["name"])
    _, rx = gu.modes(case)
    a = gu.audio(case, g)
    if case["rxnoise"]:
        a = (a + np.float32(-0.5) * np.float32(np.float32(case["rxnoise"]) * 2)).astype(np.float32)
    eng, cfg = engine_for(case)
    want = orc.rx_run(rx, a, literal=False, rx_one=False)
    (recs,), st = rx_on_gpu(eng, [a])
    got = rxfam.as_oracle_frames(recs)
    rxfam.compare_frames(got, want["frames"], case["name"])
    if orc.have_ref():
        # byte-identical decode, the reference's own pass criterion (tests/self-test: cmp)
        frames = got
        if case["rx_one"]:          # --rx-one: stop at the first carrier drop (:1310)
            nacq = [i for i, f in enumerate(frames) if f[4]]
            if len(nacq) > 1:
                frames = frames[:nacq[1]]
        assert orc.ref_decode(rx, frames, decoder=refcases.decoder_of(case, rx)) == bytes(g["stdout"])
    # stat line (the -P tests grep it for "confidence=inf ... (rate perfect)")
    reps = rxfam.reports_of(recs, st[0])
    rxfam.compare_reports(reps, want["reports"], case["name"])
    lines = [orc.report_line(rx, r) for r in reps]
    wantl = gu.stat_lines(g)
    if case["rx_one"]:
        lines = lines[:1]
    assert len(lines) >= len(wantl) >= 1
    fa, fb = lines[0].split(), wantl[0].split()
    assert fa[:3] == fb[:3] and fa[4:] == fb[4:], (lines[0], wantl[0])
    assert gu.close(float(fa[3].split("=")[1]), float(fb[3].split("=")[1]), 2e-3, cond=gu.CONF_COND)
    if case["perfect"]:
        assert "confidence=inf" in lines[0] and "(rate perfect)" in lines[0]
