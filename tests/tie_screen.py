"""A deterministic near-tie screen for random rx cases (CPU only; used by tests/test_gpu_instantiations.py).

The device and the oracle may legitimately disagree on a random stream when one of the rx loop's
decisions sits on a knife edge: the device's window sums are formed in another order, and its sqrt and
divide are the approximate units.  Rather than tolerate such disagreements in the comparison, the
*inputs* are screened: a stream is run through the oracle's rx loop once as it is and K times with every
per-window tone magnitude moved by a tiny, seeded amount.  If every perturbed run gives the records of
the unperturbed one (and the frame search's decisive comparisons keep a margin), no error of the size
of the perturbation can change the records, and the device must reproduce them exactly.  Otherwise the
stream is "not robust" and the device only has to agree on the frame count.

The perturbed search is a `find_frame` callback for orc.rx_run: it visits the candidates in
orc_find_frame's order (oracle/fsk_oracle.c, orc_find_frame), takes each candidate's per-window mark and
space magnitudes from the oracle itself (Plan.frame_analyze with an all-'d' expect string), and applies
orc_frame_analyze's frame statistic to them in float32, in the oracle's serial order.  With delta = 0 it
is the oracle's search, bit for bit (test_tie_screen_replays_the_oracle_exactly).

The rx loop's own comparisons (oracle/fsk_oracle.c, orc_rx_run) are checked by `replay`: the loop's
bookkeeping restated in float32 on what each search returned.  A confidence moves a lot under the
perturbation, so the re-runs alone flag a tie of the threshold; an amplitude is a mean over the frame's
windows and moves by about delta / sqrt(n), and the refine trigger and refine-keep compare values the
re-runs may move together -- so the squelch, the refine trigger and refine-keep get explicit margins.
A comparison inside its margin is then decided the other way in one more run of the oracle's loop
(`flipped`): the stream is robust only if that run gives the same records too.  (A slowly drifting
frame, as SAME's 92.16 samples per bit, meets `confidence < 0.75 peak_confidence` close to the tie at
every realignment, and most such refines find the frame they started from: only the later peak changes.)"""

import numpy as np

import orc

f32 = np.float32
FLT_EPSILON = f32(1.1920928955078125e-07)

# A magnitude moves by DELTA * u * max(mark, space) of its window, u = +-1.  The device's per-bin
# deviation from the oracle is at most 2e-6 of the window's signal (DESIGN.md 5 item 3): 5x that.
DELTA = 1e-5
# magnitudes at or within this fraction of the signal above FLT_EPSILON stay put: the device decides
# the `noise > FLT_EPSILON` class on an fp64 re-sum, so it matches the oracle there exactly
EPS_GUARD = 1e-6
SEEDS = 4



def _mix(x):
    """splitmix64 finaliser on uint64 arrays (wrapping)."""
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return x


def signs(seed, call, cand, nwin):
    """u = +-1 for (seed, call, candidate, window, tone): shape [nwin, 2]."""
    with np.errstate(over="ignore"):
        k = _mix(np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(call))
        k = _mix(k ^ (np.uint64(cand) * np.uint64(0xD6E8FEB86659FD93)))
        idx = np.arange(2 * nwin, dtype=np.uint64)
        h = _mix(k + idx * np.uint64(0x9E3779B97F4A7C15))
    return np.where((h >> np.uint64(63)) == 1, 1.0, -1.0).reshape(nwin, 2)


def frame_stat(mark, space, expect):
    """orc_frame_analyze's statistic (CONFIDENCE_ALGO 6) on per-window magnitudes [ncand, n] float32,
    in float32 and the oracle's serial order.  Returns (confidence, bits, amplitude, snr) per candidate;
    a candidate that fails pass 1 (a required bit decided otherwise) has confidence 0."""
    ncand, n = mark.shape
    val = mark > space                                  # strict: a tie is space / 0
    sig = np.where(val, mark, space).astype(f32)
    noise = np.where(val, space, mark).astype(f32)
    req = np.array([c in b"01" for c in expect])
    want = np.array([c == ord("1") for c in expect])
    rejected = np.any(req & (val != want), axis=1)
    zero = np.zeros(ncand, f32)
    total_sig, total_noise, avg_mark, avg_space = zero.copy(), zero.copy(), zero.copy(), zero.copy()
    n_mark = np.zeros(ncand, np.int64)
    with np.errstate(all="ignore"):
        for b in range(n):                              # serial, as the oracle's loop
            total_sig = total_sig + sig[:, b]
            total_noise = np.where(noise[:, b] > FLT_EPSILON, total_noise + noise[:, b], total_noise)
            avg_mark = np.where(val[:, b], avg_mark + sig[:, b], avg_mark)
            avg_space = np.where(val[:, b], avg_space, avg_space + sig[:, b])
            n_mark += val[:, b]
        n_space = n - n_mark
        snr = total_sig / total_noise
        ampl = total_sig / f32(n)
        avg_mark = np.where(n_mark > 0, avg_mark / n_mark.astype(f32), avg_mark)
        avg_space = np.where(n_space > 0, avg_space / n_space.astype(f32), avg_space)
        div = zero.copy()
        for b in range(n):
            other = np.where(val[:, b], avg_mark, avg_space)
            div = div + np.abs(sig[:, b] - other) / other
        div = div * f32(2)
        div = div / f32(n)
        conf = snr * (f32(1) - div)
    conf = np.where(rejected, f32(0), conf).astype(f32)
    bits = (val.astype(np.uint64) << np.arange(n, dtype=np.uint64)).sum(axis=1)
    return conf, bits, ampl.astype(f32), snr


def bound(delta, c, snr):
    """How far a perturbation of delta can move a finite confidence, to first order and with a factor 2:
    snr moves by delta (1 + snr) of itself, the divergence by 4 delta."""
    return 2.0 * delta * (abs(float(c)) * (1.0 + abs(float(snr))) + 4.0 * abs(float(snr)))


class Search:
    """find_frame callback for orc.rx_run: the oracle's frame search on perturbed magnitudes.
    `margin_ok` turns False when a decisive comparison of the search is closer than the perturbation
    can move it."""

    def __init__(self, mode, delta=DELTA, seed=0):
        self.plan = orc.Plan(mode.sample_rate, mode.mark_f, mode.space_f, mode.band_width)
        self.delta = float(delta)
        self.seed = int(seed)
        self.call = 0
        self.margin_ok = True
        self.calls = []                                 # per call: (confidence, amplitude, snr, bits, start, step)

    def bound(self, c, snr):
        return bound(self.delta, c, snr)

    def find_frame(self, ctx, samples, frame_nsamples, first, tmax, step, limit, expect, bits_out, ampl_out,
                    start_out):
        call = self.call
        self.call += 1
        n = len(expect)
        spb = f32(frame_nsamples) / f32(n)
        order = []
        for j in range(1 << 30):                       # orc_find_frame's visiting order
            up = 1 if j % 2 else -1
            t = int(first) + up * ((j + 1) // 2) * int(step)
            if t >= int(tmax):
                break
            if t >= 0:
                order.append(t)
        best_t, best_c, best_a, best_bits = 0, f32(0), f32(0), 0
        if order:
            need = max(order) + int(frame_nsamples) + int(spb) + 4
            x = np.ctypeslib.as_array(samples, shape=(need,))
            mark = np.zeros((len(order), n), f32)
            space = np.zeros((len(order), n), f32)
            alld = b"d" * n
            for i, t in enumerate(order):
                _, _, _, sig, noise, val = self.plan.frame_analyze(x[t:], float(spb), alld)
                m = np.where(val == 1, sig, noise)
                s = np.where(val == 1, noise, sig)
                if self.delta:
                    u = signs(self.seed, call, i, n)
                    top = np.maximum(m, s).astype(np.float64)
                    keep_m = m <= FLT_EPSILON + EPS_GUARD * top
                    keep_s = s <= FLT_EPSILON + EPS_GUARD * top
                    m = np.where(keep_m, m, (m + self.delta * u[:, 0] * top).astype(f32))
                    s = np.where(keep_s, s, (s + self.delta * u[:, 1] * top).astype(f32))
                mark[i], space[i] = m, s
            conf, bits, ampl, snr = frame_stat(mark, space, expect)
            lim = f32(limit)
            bests, last = [], len(order) - 1
            for i, t in enumerate(order):
                if best_c < conf[i]:
                    best_t, best_c, best_a, best_bits = t, conf[i], ampl[i], int(bits[i])
                    bests.append(i)
                    if best_c >= lim:
                        last = i
                        break
            if self.delta and bests:
                self._check_margins(conf, snr, bests[-1], bests, last, lim)
        self.calls.append((best_c, best_a, float(snr[bests[-1]]) if order and bests else 0.0, best_bits, best_t,
                           int(step)))
        bits_out[0] = best_bits
        ampl_out[0] = float(best_a)
        start_out[0] = best_t
        return float(best_c)

    def _check_margins(self, conf, snr, w, bests, last, lim):
        def finite(i):
            return np.isfinite(conf[i]) and conf[i] != 0
        if not finite(w):
            return                                      # inf / 0: classes the device decides exactly
        bw = self.bound(conf[w], snr[w])
        for i in range(last + 1):                       # the winner against every candidate it met
            if i == w or not finite(i):
                continue
            if abs(float(conf[w]) - float(conf[i])) <= bw + self.bound(conf[i], snr[i]):
                self.margin_ok = False
        if np.isfinite(lim):                            # every best so far against the limit
            for i in bests:
                if finite(i) and abs(float(conf[i]) - float(lim)) <= self.bound(conf[i], snr[i]):
                    self.margin_ok = False


def replay(mode, calls, delta=0.0, events=None):
    """orc_rx_run's bookkeeping (oracle/fsk_oracle.c:488-562) in float32 on the searches' results, in the
    oracle's order: (frames, reports, ties).  `ties` lists every squelch, refine trigger or refine-keep
    (between two different winners) closer than a perturbation of `delta` can move it -- a confidence by
    Search.bound, an amplitude by delta of itself, both with a factor 2 -- as (call index, "conf" or
    "ampl", the value that decides it the other way).  inf and 0 are classes the device decides exactly.
    With delta = 0 the frames and reports are the oracle's.
    `events`, a list, receives (kind, coarse call index) of every loop event, the state at the end last."""
    ev = events.append if events is not None else (lambda e: None)
    d = mode.derived()
    thr, q, h = f32(mode.confidence_threshold), f32(0.75), f32(0.25)
    fin = lambda c: np.isfinite(c) and c != 0
    frames, reports, ties = [], [], []
    carrier, noconf, nfd, cns = False, 0, 0, 0
    peak, peak_b, track, ctot, atot = f32(0), 0.0, f32(0), f32(0), f32(0)
    i = 0
    while i < len(calls):
        conf, ampl, snr, bits, start, step = calls[i]
        i += 1
        b = bound(delta, conf, snr) if fin(conf) else 0.0
        if delta and fin(conf) and fin(peak) and abs(float(conf) - float(q * peak)) <= b + 0.75 * peak_b:
            ties.append((i - 1, "conf", _across(conf, f32(peak * q))))             # the refine trigger
        refine = bool(conf < peak * q)
        if refine:
            peak, peak_b = f32(0), 0.0
        if delta and track > 0 and abs(float(ampl) - float(h * track)) <= 2 * delta * (float(ampl) + 0.25 * float(track)):
            ties.append((i - 1, "ampl", _across(ampl, f32(track * h))))            # the squelch
        squelched = bool(ampl < track * h) and conf > thr
        if ampl < track * h:
            conf = f32(0)
        if conf <= thr:
            ev(("strike-squelch" if squelched else "strike-threshold", i - 1))
            noconf += 1
            if noconf > 20 and carrier:
                ev(("drop", i - 1))
                reports.append((nfd, cns, ctot, atot, len(frames)))
                carrier, cns, ctot, atot, nfd, track = False, 0, f32(0), f32(0), 0, f32(0)
            continue
        if carrier and noconf >= 15:
            ev(("held-15-strikes", i - 1))
        cns += int(d.frame_nsamples)
        acquired = 0
        if carrier:
            cns += int(start) - int(d.nsamples_overscan)
        else:
            carrier, acquired, refine = True, 1, True
            ev(("acquire", i - 1))
        if refine and not acquired:
            ev(("refine-in-session", i - 1))
        if refine and conf < np.inf and step > 1:
            c2, a2, snr2, bits2, start2, _ = calls[i]
            i += 1
            if delta and fin(c2) and (bits2, start2) != (bits, start) \
                    and abs(float(c2) - float(conf)) <= bound(delta, c2, snr2) + b:
                ties.append((i - 1, "conf", conf if c2 > conf else np.nextafter(conf, f32(np.inf))))  # refine-keep
            if c2 > conf:
                bits, ampl, start = bits2, a2, start2
        track = f32((track + ampl) / f32(2))
        if peak < conf:
            peak, peak_b = conf, b
        ctot, atot = f32(ctot + conf), f32(atot + ampl)
        nfd += 1
        noconf = 0
        frames.append((bits, conf, ampl, start, acquired))
    if carrier:
        ev(("open-at-end", i - 1))
        reports.append((nfd, cns, ctot, atot, len(frames)))
    if noconf:
        ev(("ends-mid-count", i - 1))
    return frames, reports, ties


def _across(v, edge):
    """the value nearest `edge` on the other side of `v < edge`"""
    return edge if v < edge else np.nextafter(edge, f32(0))


def flipped(mode, x, tie):
    """the oracle's rx loop on x with one search result replaced: tie = (call index, "conf" or "ampl",
    value), as replay lists them"""
    plan = orc.Plan(mode.sample_rate, mode.mark_f, mode.space_f, mode.band_width)
    j, what, value = tie
    n = [0]

    def find_frame(ctx, samples, frame_nsamples, first, tmax, step, limit, expect, bits_out, ampl_out, start_out):
        c = orc.lib().orc_find_frame(orc.C.byref(plan.p), samples, frame_nsamples, first, tmax, step, limit,
                                     expect, bits_out, ampl_out, start_out)
        n[0] += 1
        if n[0] - 1 == j:
            if what == "conf":
                c = float(value)
            else:
                ampl_out[0] = float(value)
        return c
    return orc.rx_run(mode, x, literal=False, find_frame=find_frame)


def record_key(res):
    """What must agree: the frames' count, bits, frame starts and acquire flags."""
    return [(f[0], f[3], f[4]) for f in res["frames"]]


def run(mode, x, delta=DELTA, seed=0):
    s = Search(mode, delta, seed)
    res = orc.rx_run(mode, x, literal=False, find_frame=s.find_frame)
    return res, s


def screen(mode, x, seeds=SEEDS):
    """(the oracle's rx_run result for x, robust?)"""
    want = orc.rx_run(mode, x, literal=False)
    key = record_key(want)
    for k in range(seeds):
        res, s = run(mode, x, DELTA, 1 + k)
        if not s.margin_ok or record_key(res) != key:
            return want, False
    _, s = run(mode, x, 0.0)
    for tie in replay(mode, s.calls, DELTA)[2]:
        if record_key(flipped(mode, x, tie)) != key:
            return want, False
    return want, True
