/*
 * fsk_b200_device.cuh -- device functions of the FSK engine (sm_90a).
 *
 * Two basic implementations of the same arithmetic:
 *
 *  FAST   frame_analyze_fast<G,W,L> / find_frame_fast_body: the stream's samples are in a
 *         per-stream shared-memory ring of R floats (R % 4 == 0) whose first
 *         window-length is mirrored behind its end, so a bit window is always one
 *         linear run; each lane owns W windows (and 1/L of their samples) and
 *         walks the twiddle table once for all of them (n outer, windows inner):
 *         one LDS.128 (twiddles) + W LDS.32 (samples) feed 4*W FMAs.  W, L are
 *         compile-time so accumulators and per-bit results stay in registers;
 *         frame statistics are butterfly-reduced over the group.
 *  GENERIC frame_analyze<G,Src> / find_frame: samples straight from global
 *         memory, run-time window split, IEEE sqrt/div, the reference's serial
 *         summation order, fp64 folding of the fp32 partial sums for very long
 *         windows.  Used when the windows do not fit shared memory (e.g. 0.5 baud).
 *
 * On top of FAST: MULTI (find_frame_multi: the candidates of a search from shared segment sums),
 * the sliding fine search (find_frame_slide) and PREFIX (pfx_build / pfx_round / pfx_search: every
 * candidate of a loop iteration from one chunk-prefix table; one stream per warp).
 *
 * All floating-point steps that decide anything follow the reference's order
 * (src/fsk.c:107-174, :178-446, :449-538); comments carry its line numbers.
 */
#ifndef FSK_B200_DEVICE_CUH
#define FSK_B200_DEVICE_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "fsk_b200_internal.h"

#define FSK_FLT_EPSILON 1.1920928955078125e-07f
#define ACC_BLOCK 64u		/* generic path: fp32 partial sums are folded into fp64 every ACC_BLOCK terms */
#define FAST_MAX_N 2048u	/* fast path: plain fp32 accumulation up to this many terms per lane */

/* ------------------------------------------------------------------------ */
/* bit decision + bookkeeping shared by both paths                          */
/* ------------------------------------------------------------------------ */

/* band_mag (src/fsk.c:107-114) for both tones, the decision (:158-169) and the
 * pass-1 check (:211); the result goes to the per-stream scratch: x = signal
 * magnitude, y = noise magnitude with the bit value in its sign. */
__device__ __forceinline__ bool decide_bit(float mag_mark, float mag_space, unsigned expect,
	float2 *slot)
{
    const bool one = mag_mark > mag_space;			/* strict: tie -> space */
    const float sig = one ? mag_mark : mag_space;
    const float noise = one ? mag_space : mag_mark;
    *slot = make_float2(sig, one ? -noise : noise);
    return expect != 2u && expect != (one ? 1u : 0u);
}

/* The reference drops off-tone magnitudes <= FLT_EPSILON from the noise sum
 * (src/fsk.c:279) so that exactly periodic tones give confidence = inf.  fp32
 * accumulation is good to ~2e-7 of the signal, not enough to classify a magnitude
 * that close to FLT_EPSILON: such (rare: synthetic, orthogonal-tone) windows are
 * re-summed in fp64, where float*float products are exact. */
__device__ __forceinline__ bool needs_resum(float mag_mark, float mag_space)
{
    const float lo = fminf(mag_mark, mag_space), hi = fmaxf(mag_mark, mag_space);
    return lo < FSK_FLT_EPSILON + 2e-6f * hi;
}

/* src/fsk.c:271-342 over the scratch of one candidate, bit index ascending, one
 * rounding per operation.  `owner(w)` tells whether this lane computes the
 * divergence term of window w.  All lanes of the group execute this and end up
 * with the same values. */
template <class ForOwn>
__device__ __forceinline__ float confidence_from_scratch(float2 *scr, unsigned nb, unsigned gmask,
	ForOwn for_own_windows, unsigned long long &bits_out, float &ampl_out)
{
    float total_sig = 0.f, total_noise = 0.f, avg_mark = 0.f, avg_space = 0.f;
    unsigned n_mark = 0;
    unsigned bits_lo = 0, bits_hi = 0;
    for (unsigned b = 0; b < nb; b++) {
	const float2 v = scr[b];
	const float noise = fabsf(v.y);
	const unsigned one = __float_as_uint(v.y) >> 31;	/* the bit value rides in the sign */
	total_sig += v.x;
	if (noise > FSK_FLT_EPSILON)				/* :279 */
	    total_noise += noise;
	avg_mark += one ? v.x : 0.f;		/* x + 0 is exact: same value as the reference's branch */
	avg_space += one ? 0.f : v.x;
	n_mark += one;
	const unsigned m = one << (b & 31u);
	bits_lo |= b < 32u ? m : 0u;
	bits_hi |= b < 32u ? 0u : m;
    }
    const unsigned n_space = nb - n_mark;
    const float snr = total_sig / total_noise;			/* :292, may be +inf */
    const float avg_bit_sig = total_sig / (float)(int)nb;	/* :295 */
    if (n_mark)
	avg_mark = avg_mark / (float)n_mark;			/* :298-301 */
    if (n_space)
	avg_space = avg_space / (float)n_space;

    /* divergence terms (:305-311): one division per bit, done by the window owners ... */
    __syncwarp(gmask);
    for_own_windows([&](unsigned w) {
	const float2 v = scr[w];
	const float other = (__float_as_uint(v.y) >> 31) ? avg_mark : avg_space;
	scr[w].x = fabsf(v.x - other) / other;
    });
    __syncwarp(gmask);
    /* ... and summed in bit order */
    float divergence = 0.f;
    for (unsigned b = 0; b < nb; b++)
	divergence += scr[b].x;
    divergence *= 2.f;						/* :312-313 */
    divergence = divergence / (float)(int)nb;

    bits_out = ((unsigned long long)bits_hi << 32) | bits_lo;
    ampl_out = avg_bit_sig;					/* :342 */
    return snr * (1.0f - divergence);				/* :336 */
}

/* ======================================================================== */
/* GENERIC path                                                             */
/* ======================================================================== */

/* straight from global memory, zero beyond the valid length.  Callers index it from the search position
 * (x = the row + pos, n = what is left of the row), so that base + offset stays small: an absolute index
 * near 2^32 would wrap past n and read the row's start */
struct GlobalSrc {
    const float *x;
    unsigned n;
    __device__ __forceinline__ float operator()(unsigned i) const { return i < n ? __ldg(x + i) : 0.0f; }
};

template <class Src>
__device__ __forceinline__ void resum_fp64(const Src &src, unsigned base, unsigned N,
	const float4 *__restrict__ tw, float mag_scalar, float &mag_mark, float &mag_space)
{
    double drm = 0., dim = 0., drs = 0., dis = 0.;
    for (unsigned n = 0; n < N; n++) {
	const double x = (double)src(base + n);
	const float4 c = tw[n];
	drm = fma(x, (double)c.x, drm);
	dim = fma(x, (double)c.y, dim);
	drs = fma(x, (double)c.z, drs);
	dis = fma(x, (double)c.w, dis);
    }
    const float frm = (float)drm, fim = (float)dim, frs = (float)drs, fis = (float)dis;
    mag_mark = sqrtf(frm * frm + fim * fim) * mag_scalar;
    mag_space = sqrtf(frs * frs + fis * fis) * mag_scalar;
}

template <int G, class Src>
__device__ __noinline__ float frame_analyze(const Src &src, unsigned t0,
	const fsk_b200_geom &geo, int sel, const float4 *__restrict__ tw, float2 *scr,
	unsigned g, unsigned gmask, unsigned long long &bits_out, float &ampl_out, float2 *mags_out = nullptr)
{
    const unsigned N = geo.bit_nsamples, nb = geo.n_bits, L = geo.lanes_per_window;
    const unsigned wpp = G / L;			/* windows analysed per pass */
    const unsigned part = g & (L - 1), wslot = g / L;
    bool mismatch = false;

    __syncwarp(gmask);				/* previous readers of scr are done */
    for (unsigned w0 = 0; w0 < nb; w0 += wpp) {
	const unsigned w = w0 + wslot;
	const bool active = w < nb;
	float rm = 0.f, im = 0.f, rs = 0.f, is = 0.f;
	if (active) {
	    const unsigned base = t0 + geo.bit_begin[w];
	    /* bounded fp32 partial sums folded into fp64 (very long windows stay accurate) */
	    double drm = 0., dim = 0., drs = 0., dis = 0.;
	    for (unsigned n0 = part; n0 < N; n0 += ACC_BLOCK * L) {
		const unsigned nend = min(N, n0 + ACC_BLOCK * L);
		float prm = 0.f, pim = 0.f, prs = 0.f, pis = 0.f;
		for (unsigned n = n0; n < nend; n += L) {
		    const float x = src(base + n);
		    const float4 c = tw[n];
		    prm = fmaf(x, c.x, prm);
		    pim = fmaf(x, c.y, pim);
		    prs = fmaf(x, c.z, prs);
		    pis = fmaf(x, c.w, pis);
		}
		drm += prm; dim += pim; drs += prs; dis += pis;
	    }
	    rm = (float)drm; im = (float)dim; rs = (float)drs; is = (float)dis;
	}
	for (unsigned o = L >> 1; o; o >>= 1) {
	    rm += __shfl_xor_sync(gmask, rm, o);
	    im += __shfl_xor_sync(gmask, im, o);
	    rs += __shfl_xor_sync(gmask, rs, o);
	    is += __shfl_xor_sync(gmask, is, o);
	}
	if (active && part == 0) {
	    float mag_mark = sqrtf(rm * rm + im * im) * geo.mag_scalar;
	    float mag_space = sqrtf(rs * rs + is * is) * geo.mag_scalar;
	    if (needs_resum(mag_mark, mag_space))
		resum_fp64(src, t0 + geo.bit_begin[w], N, tw, geo.mag_scalar, mag_mark, mag_space);
	    mismatch |= decide_bit(mag_mark, mag_space, geo.expect[sel][w], scr + w);
	    if (mags_out)		/* (signal, noise) per bit: the statistic below reuses the scratch */
		mags_out[w] = make_float2(scr[w].x, fabsf(scr[w].y));
	}
    }
    __syncwarp(gmask);
    if (__any_sync(gmask, mismatch)) {		/* pass 1 reject, src/fsk.c:211-212 */
	bits_out = 0;
	ampl_out = 0.f;
	return 0.f;
    }
    return confidence_from_scratch(scr, nb, gmask, [&](auto body) {
	if (part == 0)
	    for (unsigned w = wslot; w < nb; w += wpp)
		body(w);
    }, bits_out, ampl_out);
}

/* frame search: src/fsk.c:449-538 */
template <class Analyze>
__device__ __forceinline__ float search_frames(Analyze analyze, unsigned try_first, unsigned try_max,
	unsigned try_step, float limit, unsigned long long &best_bits, float &best_a, unsigned &best_t)
{
    float best_c = 0.f;
    best_t = 0;
    best_a = 0.f;
    best_bits = 0;
    for (int j = 0;; j++) {					/* :477-502 */
	const int up = (j & 1) ? 1 : -1;
	const int t = (int)try_first + up * ((j + 1) / 2) * (int)try_step;
	if (t >= (int)try_max)
	    break;
	if (t < 0)
	    continue;
	unsigned long long bits;
	float a;
	const float c = analyze((unsigned)t, bits, a);
	if (best_c < c) {			/* NaN and negatives never win */
	    best_t = (unsigned)t;
	    best_c = c;
	    best_a = a;
	    best_bits = bits;
	    if (best_c >= limit)
		break;				/* first to reach the limit wins */
	}
    }
    return best_c;
}

template <int G, class Src>
__device__ __forceinline__ float find_frame(const Src &src, unsigned base,
	const fsk_b200_geom &geo, int sel, const float4 *__restrict__ tw, float2 *scr,
	unsigned g, unsigned gmask, unsigned try_first, unsigned try_max, unsigned try_step,
	float limit, unsigned long long &best_bits, float &best_a, unsigned &best_t)
{
    return search_frames([&](unsigned t, unsigned long long &bits, float &a) {
	return frame_analyze<G, Src>(src, base + t, geo, sel, tw, scr, g, gmask, bits, a);
    }, try_first, try_max, try_step, limit, best_bits, best_a, best_t);
}

/* ======================================================================== */
/* FAST path                                                                */
/* ======================================================================== */

/* A per-stream ring of R floats (R % 4 == 0) followed by a MIRROR of its first
 * `pad` floats (pad >= bit_nsamples - 1, pad % 4 == 0): ring[R + k] == ring[k].
 * A bit window that starts anywhere in [0, R) is therefore one linear run, no
 * wrap handling inside the correlation loop.  `pos_off` is the ring offset of the
 * absolute sample index `pos` (pos_off == pos mod 4 is kept, so the 16-byte
 * chunks of the stream line up with 16-byte chunks of the ring). */
struct Ring {
    unsigned ring_s;		/* shared-window address of the ring */
    unsigned R, pad;
};

__device__ __forceinline__ unsigned ring_wrap(unsigned off, unsigned R) { return off >= R ? off - R : off; }

/* Fast-path arithmetic: sqrt.approx / div.approx (<= 2 ulp) instead of the IEEE sequences.
 * They feed magnitudes and the confidence statistic, which are compared to tolerance; the
 * generic path keeps IEEE operations. */
#ifndef FSK_EMU	/* inline PTX: the host emulation of the test harness (tests/emu) brings its own */
__device__ __forceinline__ float fast_sqrt(float x)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_div(float a, float b)
{
    /* .ftz: two instructions (MUFU.RCP + FMUL) instead of the denormal-safe sequence; the
     * operands are magnitudes and their sums, far from the denormal range */
    float r;
    asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
#endif

/* butterfly all-reduce over the G lanes of a group (every lane ends with the total) */
template <int G>
__device__ __forceinline__ float group_sum(float v, unsigned gmask)
{
#pragma unroll
    for (int o = G >> 1; o; o >>= 1)
	v += __shfl_xor_sync(gmask, v, o);
    return v;
}
template <int G>
__device__ __forceinline__ unsigned group_or(unsigned v, unsigned gmask)
{
#pragma unroll
    for (int o = G >> 1; o; o >>= 1)
	v |= __shfl_xor_sync(gmask, v, o);
    return v;
}
template <int G>
__device__ __forceinline__ unsigned group_add(unsigned v, unsigned gmask)
{
#pragma unroll
    for (int o = G >> 1; o; o >>= 1)
	v += __shfl_xor_sync(gmask, v, o);
    return v;
}

#ifndef FSK_EMU	/* inline PTX, see tests/emu */
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int NKEEP>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" :: "n"(NKEEP) : "memory"); }
#endif

/* What a lane needs to know about its W windows, computed once per kernel instead of per
 * candidate: the offset of each window inside a frame candidate, which of them this lane
 * post-processes, and the expected bit ('0', '1' or don't care) under both expect strings. */
template <int W>
struct LaneWin {
    unsigned beg[W];	/* bit_begin of window j (0 for a slot past n_bits) */
    unsigned own;	/* bit j: this lane decides window j */
    unsigned exp;	/* 2 bits per (sel, j): expect value 0, 1 or 2 */
};

template <int G, int W, int L>
__device__ __forceinline__ LaneWin<W> lane_windows(const fsk_b200_geom &geo, unsigned g)
{
    constexpr unsigned WPP = G / L;
    const unsigned part = g % L, wslot = g / L;
    LaneWin<W> lw;
    lw.own = 0;
    lw.exp = 0;
#pragma unroll
    for (int j = 0; j < W; j++) {
	const unsigned w = j * WPP + wslot;
	const bool valid = w < geo.n_bits;
	lw.beg[j] = valid ? geo.bit_begin[w] : 0u;
	if (valid && part == (unsigned)(j % L))
	    lw.own |= 1u << j;
	const unsigned e0 = valid ? geo.expect[0][w] : 2u, e1 = valid ? geo.expect[1][w] : 2u;
	lw.exp |= (e0 << (2 * j)) | (e1 << (2 * (j + W)));
    }
    return lw;
}

/* the W windows of this lane against both tones, its share n = part, part+L, ... of the samples */
template <int W, int L>
__device__ __forceinline__ void corr_pass(float (&acc)[W][4], const float *const (&p)[W],
	const float4 *tw, unsigned part, unsigned N)
{
#pragma unroll 4
    for (unsigned n = part; n < N; n += L) {
	const float4 c = tw[n];
#pragma unroll
	for (int j = 0; j < W; j++) {
	    const float x = p[j][n];
	    acc[j][0] = fmaf(x, c.x, acc[j][0]);
	    acc[j][1] = fmaf(x, c.y, acc[j][1]);
	    acc[j][2] = fmaf(x, c.z, acc[j][2]);
	    acc[j][3] = fmaf(x, c.w, acc[j][3]);
	}
    }
}

/* best candidate of a search (src/fsk.c:504-508), returned in registers */
struct Found {
    float confidence, amplitude;
    unsigned start, bits_lo, bits_hi;
};

/* From the (per-lane partial) sums of this lane's W windows to the frame statistic: the exchange
 * between the L lanes of a window, the per-window decision (src/fsk.c:158-169, :211), the sums
 * and the confidence (:271-336).  CONSEC: window j of the lane is bit wslot*W + j (MULTI) instead
 * of j*(G/L) + wslot.  p[j] = first sample of window j (for the fp64 re-sum). */
template <int G, int W, int L, bool CONSEC>
__device__ __forceinline__ float frame_finish(float (&acc)[W][4], const float *const (&p)[W],
	const unsigned own_mask, const unsigned exp_bits, const fsk_b200_geom &geo, const float4 *tw, int sel,
	unsigned g, unsigned gmask, unsigned &bits_lo_out, unsigned &bits_hi_out, float &ampl_out,
	float2 *bit_mags = nullptr)
{
    constexpr unsigned WPP = G / L;
    const unsigned N = geo.bit_nsamples, nb = geo.n_bits;
    const unsigned part = g % L, wslot = g / L;
    constexpr int KW = (W + L - 1) / L;
    constexpr bool XCHG = (L == 2);
    /* XCHG (L == 2): instead of an all-reduce that leaves every sum on both lanes of a window, the
     * two lanes swap the partial sums of the window the OTHER one post-processes (same two
     * addends, so the same sums): 4 shuffles per round instead of 8 */
    float ax[KW][4];
    if (XCHG) {
#pragma unroll
	for (int k = 0; k < KW; k++) {
	    const int j0 = 2 * k, j1 = 2 * k + 1;
#pragma unroll
	    for (int c = 0; c < 4; c++) {
		if (j1 < W) {
		    const float send = part ? acc[j0][c] : acc[j1][c];
		    const float mine = part ? acc[j1][c] : acc[j0][c];
		    ax[k][c] = mine + __shfl_xor_sync(gmask, send, 1);
		} else
		    ax[k][c] = acc[j0][c] + __shfl_xor_sync(gmask, acc[j0][c], 1);
	    }
	}
    } else if (L > 1) {
#pragma unroll
	for (int o = L >> 1; o; o >>= 1) {
#pragma unroll
	    for (int j = 0; j < W; j++) {
#pragma unroll
		for (int k = 0; k < 4; k++)
		    acc[j][k] += __shfl_xor_sync(gmask, acc[j][k], o);
	    }
	}
    }

    /* per-window decision (src/fsk.c:158-169) and this lane's share of the sums (:271-289).
     * After the butterfly all L lanes of a window hold its sums, so they share the work:
     * lane part p decides the windows j = p, p+L, ... (KW = ceil(W/L) rounds instead of W).
     * Magnitudes stay unscaled (the 2/N of src/fsk.c:132 is applied once, to the amplitude);
     * the FLT_EPSILON threshold of :279 is scaled the other way instead. */
    const float eps_u = geo.eps_unscaled;
    float tn = 0.f, am = 0.f, as = 0.f;
    unsigned nm = 0, blo = 0, bhi = 0;
    float sig[KW];
    bool one[KW], own[KW];
    bool mismatch = false;
#pragma unroll
    for (int k = 0; k < KW; k++) {
	const unsigned jsel = part + (unsigned)(k * L);		/* this lane's window in round k */
	float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
	const float *q = p[0];
#pragma unroll
	for (int pp = 0; pp < L; pp++) {
	    const int j = pp + k * L;
	    if (j < W && part == (unsigned)pp) {
		if (!XCHG) {
		    a0 = acc[j][0]; a1 = acc[j][1]; a2 = acc[j][2]; a3 = acc[j][3];
		}
		q = p[j];
	    }
	}
	if (XCHG) {
	    a0 = ax[k][0]; a1 = ax[k][1]; a2 = ax[k][2]; a3 = ax[k][3];
	}
	own[k] = (own_mask >> jsel) & 1u;
	sig[k] = 0.f;
	one[k] = false;
	if (own[k]) {
	    float mag_mark = fast_sqrt(a0 * a0 + a1 * a1);
	    float mag_space = fast_sqrt(a2 * a2 + a3 * a3);
	    const float mag_hi = fmaxf(mag_mark, mag_space);
	    /* (a window whose fp32 sums are exactly zero -- silence -- stays zero in fp64 too) */
	    if (mag_hi != 0.f && fminf(mag_mark, mag_space) < eps_u + 2e-6f * mag_hi) {
		/* too close to the :279 threshold for fp32 sums (see needs_resum): fp64 re-sum */
		double drm = 0., dim = 0., drs = 0., dis = 0.;
#pragma unroll 1
		for (unsigned i = 0; i < N; i++) {
		    const double x = (double)q[i];
		    const float4 c = tw[i];
		    drm = fma(x, (double)c.x, drm);
		    dim = fma(x, (double)c.y, dim);
		    drs = fma(x, (double)c.z, drs);
		    dis = fma(x, (double)c.w, dis);
		}
		const float frm = (float)drm, fim = (float)dim, frs = (float)drs, fis = (float)dis;
		mag_mark = sqrtf(frm * frm + fim * fim);
		mag_space = sqrtf(frs * frs + fis * fis);
	    }
	    const unsigned w = CONSEC ? wslot * (unsigned)W + jsel : jsel * WPP + wslot;
	    one[k] = mag_mark > mag_space;			/* strict: tie -> space */
	    sig[k] = one[k] ? mag_mark : mag_space;
	    const float noise = one[k] ? mag_space : mag_mark;
	    const unsigned e = (exp_bits >> (2u * (jsel + (sel ? (unsigned)W : 0u)))) & 3u;
	    mismatch |= e != 2u && e != (one[k] ? 1u : 0u);	/* pass 1, :211 */
	    if (bit_mags)		/* diagnostics: the (signal, noise) magnitudes of src/fsk.c:158-169, scaled as there */
		bit_mags[w] = make_float2(sig[k] * geo.mag_scalar, noise * geo.mag_scalar);
	    if (noise > eps_u)					/* :279 */
		tn += noise;
	    if (one[k]) {
		am += sig[k];
		nm++;
		if (w < 32u) blo |= 1u << w; else bhi |= 1u << (w - 32u);
	    } else {
		as += sig[k];
	    }
	}
    }
    /* pass 1 reject, src/fsk.c:211-212.  No vote: a lane that saw a mismatch poisons the noise sum
     * with +inf, and the verdict is read off the reduced sum (one convergence point fewer per
     * candidate; a noise sum that overflowed by itself would give confidence 0, which never wins
     * either). */
    if (mismatch)
	tn = INFINITY;
    /* total_sig = sum over marks + sum over spaces; the mark count rides above the bits when
     * the frame is short enough (disjoint bit positions: OR == ADD) */
    /* one butterfly for all four: the shuffles share a single convergence guard */
    unsigned packed = blo | (nm << 24);
#pragma unroll
    for (int o = G >> 1; o; o >>= 1) {
	tn += __shfl_xor_sync(gmask, tn, o);
	am += __shfl_xor_sync(gmask, am, o);
	as += __shfl_xor_sync(gmask, as, o);
	packed += __shfl_xor_sync(gmask, packed, o);
    }
    if (tn == INFINITY) {
	bits_lo_out = bits_hi_out = 0;
	ampl_out = 0.f;
	return 0.f;
    }
    const float ts = am + as;
    if (nb <= 24u) {
	blo = packed & 0xffffffu;
	nm = packed >> 24;
    } else {
	nm = group_add<G>(nm, gmask);
	blo = group_or<G>(blo, gmask);
	if (nb > 32u)
	    bhi = group_or<G>(bhi, gmask);
    }

    const unsigned n_space = nb - nm;
    const float snr = fast_div(ts, tn);					/* :292, may be +inf */
    const float avg_bit_sig = ts * geo.inv_n_bits * geo.mag_scalar;	/* :295, with the 2/N of :132 */
    if (nm)
	am = fast_div(am, (float)nm);					/* :298-301 */
    if (n_space)
	as = fast_div(as, (float)n_space);
    float dv = 0.f;						/* :305-311 */
#pragma unroll
    for (int k = 0; k < KW; k++) {
	if (own[k]) {
	    const float other = one[k] ? am : as;
	    dv += fast_div(fabsf(sig[k] - other), other);
	}
    }
    float divergence = group_sum<G>(dv, gmask);
    divergence *= 2.f;						/* :312-313 */
    divergence = divergence * geo.inv_n_bits;

    bits_lo_out = blo;
    bits_hi_out = bhi;
    ampl_out = avg_bit_sig;					/* :342 */
    return snr * (1.0f - divergence);				/* :336 */
}

/* One candidate frame start, fast path.  Lane g of the group owns the windows
 * w = j*(G/L) + g/L (j < W) and, of each, the samples n = g%L, g%L + L, ...
 * Everything stays in registers: the per-bit (sig, noise, bit) values never go
 * to memory, and the frame statistics of src/fsk.c:271-336 are formed by
 * butterfly reductions over the group instead of a serial loop over the bits
 * (same terms, different but fixed summation order). */
template <int G, int W, int L, bool CONSEC = false, class LW = LaneWin<W> >
__device__ __forceinline__ float frame_analyze_fast(const Ring rg, unsigned cand_off,
	const fsk_b200_geom &geo, const LW &lw, int sel, unsigned tw_s,
	unsigned g, unsigned gmask, unsigned &bits_lo_out, unsigned &bits_hi_out, float &ampl_out,
	bool &pending, float2 *bit_mags = nullptr)
{
    /* ring and twiddles are handed over as shared-window addresses and turned back into
     * pointers here, so that the compiler keeps them in the shared address space (LDS with
     * 32-bit addresses and immediate offsets) even though this code is not inlined */
    const float *ring = static_cast<const float *>(__cvta_shared_to_generic(rg.ring_s));
    const float4 *tw = static_cast<const float4 *>(__cvta_shared_to_generic(tw_s));
    /* cand_off: ring offset (< R) of the candidate's first sample */
    const unsigned N = geo.bit_nsamples, R = rg.R;
    const unsigned part = g % L;

    /* slots past n_bits read window 0: harmless, their results are dropped */
    const float *p[W];
#pragma unroll
    for (int j = 0; j < W; j++)
	p[j] = ring + ring_wrap(cand_off + lw.beg[j], R);

    float acc[W][4];
#pragma unroll
    for (int j = 0; j < W; j++)
	acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;

    /* `pending`: copies into this ring may still be in flight */
    if (pending) {
	cp_async_wait<0>();
	__syncwarp(gmask);
	pending = false;
    }
    corr_pass<W, L>(acc, p, tw, part, N);
    return frame_finish<G, W, L, CONSEC>(acc, p, lw.own, lw.exp, geo, tw, sel, g, gmask, bits_lo_out,
	    bits_hi_out, ampl_out, bit_mags);
}

/* frame search, src/fsk.c:449-538 */
template <int G, int W, int L>
__device__ __forceinline__ Found find_frame_fast_body(const Ring rg, unsigned pos_off,
	const fsk_b200_geom &geo, const LaneWin<W> lw, int sel, unsigned tw_s,
	unsigned g, unsigned gmask, unsigned try_first, unsigned try_max, unsigned try_step, float limit,
	bool pending, unsigned &ncand)
{
    /* pending: the caller's latest copies into the ring are still in flight; the first candidate
     * waits as late as it can */
    Found best = { 0.f, 0.f, 0u, 0u, 0u };
    for (int j = 0;; j++) {					/* :477-502 */
	const int up = (j & 1) ? 1 : -1;
	const int t = (int)try_first + up * ((j + 1) / 2) * (int)try_step;
	if (t >= (int)try_max)
	    break;
	if (t < 0)
	    continue;
	unsigned lo, hi;
	float a;
	ncand++;
	const float c = frame_analyze_fast<G, W, L>(rg, ring_wrap(pos_off + (unsigned)t, rg.R), geo, lw, sel,
		tw_s, g, gmask, lo, hi, a, pending);
	if (best.confidence < c) {			/* NaN and negatives never win */
	    best = Found{ c, a, (unsigned)t, lo, hi };
	    if (c >= limit)
		break;				/* first to reach the limit wins */
	}
    }
    return best;
}

/* The fine search of the rx loop (src/minimodem.c:1357-1389: try_step = try_max/8, no limit) by SLIDING.
 * Its candidates are `step` samples apart, a fraction of a bit window, so the window sums of a candidate
 * are those of its neighbour minus the `step` samples that left each window plus the `step` that entered:
 * 2*step multiply-adds per window instead of bit_nsamples.  For that the correlation phase must not
 * restart with the candidate: the table is indexed by (candidate offset + sample) -- geom.tw_entries
 * covers try_max + bit_nsamples + a step -- which changes every window sum by a unit phase factor only,
 * i.e. not its magnitude (src/fsk.c:107-114 takes the magnitude).  The candidates are visited in
 * ascending order instead of the zig-zag of src/fsk.c:477-484; among equal confidences the one the
 * reference would have met first is kept, which is what its strict `best_c < c` does.  Works for any
 * frame geometry (no tiling needed); fp32 error grows by a few 1e-7 of the window's terms per slide. */
template <int G, int W, int L>
__device__ __forceinline__ Found find_frame_slide(const Ring rg, unsigned pos_off,
	const fsk_b200_geom &geo, const LaneWin<W> &lw, int sel, unsigned tw_s, unsigned g, unsigned gmask,
	unsigned try_first, unsigned try_max, unsigned step, unsigned &ncand)
{
    const float *ring = static_cast<const float *>(__cvta_shared_to_generic(rg.ring_s));
    const float4 *tw = static_cast<const float4 *>(__cvta_shared_to_generic(tw_s));
    const unsigned N = geo.bit_nsamples, R = rg.R;
    const unsigned part = g % L;
    /* the set src/fsk.c:477-484 visits: first + k*step for -k_dn <= k <= k_up (the scan ends at the first
     * upward step that reaches try_max, so it never gets further down than it got up) */
    const unsigned k_up = (try_max - 1u - try_first) / step;
    const unsigned k_dn = min(try_first / step, k_up);
    unsigned t = try_first - k_dn * step;
    const unsigned ncands = k_dn + k_up + 1u;

    const float *p[W];
    float acc[W][4];
#pragma unroll
    for (int j = 0; j < W; j++) {
	p[j] = ring + ring_wrap(ring_wrap(pos_off + t, R) + lw.beg[j], R);
	acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    }
    corr_pass<W, L>(acc, p, tw + t, part, N);	/* the lowest candidate: a full correlation, phase index t + n */
    /* the largest sample that has left each window since its last full correlation (see below) */
    float gone[W];
#pragma unroll
    for (int j = 0; j < W; j++)
	gone[j] = 0.f;

    Found best = { 0.f, 0.f, 0u, 0u, 0u };
    unsigned best_order = 0;
#pragma unroll 1
    for (unsigned i = 0;; i++) {
	ncand++;
	float wsum[W][4];
#pragma unroll
	for (int j = 0; j < W; j++)
#pragma unroll
	    for (int k = 0; k < 4; k++)
		wsum[j][k] = acc[j][k];			/* frame_finish may reduce in place */
	unsigned lo, hi;
	float a;
	const float c = frame_finish<G, W, L, false>(wsum, p, lw.own, lw.exp, geo, tw, sel, g, gmask, lo, hi, a);
	/* place in the reference's visiting order: first, +1, -1, +2, -2, ... */
	const unsigned order = t >= try_first ? (t == try_first ? 0u : 2u * ((t - try_first) / step) - 1u)
	    : 2u * ((try_first - t) / step);
	if (best.confidence < c || (best.confidence == c && c > 0.f && order < best_order)) {
	    best = Found{ c, a, t, lo, hi };
	    best_order = order;
	}
	if (i + 1u == ncands)
	    break;
	/* slide every window from t to t + step */
	const unsigned base = ring_wrap(pos_off + t, R);
	const float *pr[W], *pa[W];
#pragma unroll
	for (int j = 0; j < W; j++) {
	    const unsigned w0 = ring_wrap(base + lw.beg[j], R);
	    pr[j] = ring + w0;					/* the samples that leave: [t, t + step) of the window */
	    pa[j] = ring + ring_wrap(w0 + N, R);		/* the samples that enter: [t + N, t + N + step) */
	}
	const float4 *twr = tw + t, *twa = tw + t + N;
#pragma unroll 2
	for (unsigned n = part; n < step; n += L) {
	    const float4 cr = twr[n], ca = twa[n];
#pragma unroll
	    for (int j = 0; j < W; j++) {
		const float xr = pr[j][n], xa = pa[j][n];
		gone[j] = fmaxf(gone[j], fabsf(xr));
		acc[j][0] = fmaf(xa, ca.x, fmaf(-xr, cr.x, acc[j][0]));
		acc[j][1] = fmaf(xa, ca.y, fmaf(-xr, cr.y, acc[j][1]));
		acc[j][2] = fmaf(xa, ca.z, fmaf(-xr, cr.z, acc[j][2]));
		acc[j][3] = fmaf(xa, ca.w, fmaf(-xr, cr.w, acc[j][3]));
	    }
	}
	t += step;
	/* A sum that kept a loud sample (a click) carries a few ulp of it after the sample has left: past 16x
	 * this lane's share of the window that is beyond the error the slide is allowed, and far past it the
	 * window cancels to nothing.  A NaN or inf that left turned the sums into NaN (the unordered test).
	 * Either way the windows are correlated afresh, as the lowest candidate was. */
	bool stale = false;
#pragma unroll
	for (int j = 0; j < W; j++) {
	    p[j] = ring + ring_wrap(ring_wrap(pos_off + t, R) + lw.beg[j], R);	/* window starts (fp64 re-sum) */
	    const float amax = fmaxf(fmaxf(fabsf(acc[j][0]), fabsf(acc[j][1])), fmaxf(fabsf(acc[j][2]), fabsf(acc[j][3])));
	    stale |= !(gone[j] <= 16.f * amax);
	}
	/* the lanes of a window hold shares of its sums that only add up together: all lanes of the group start
	 * afresh, each with its samples n = part (mod L) as at the lowest candidate */
	if (__any_sync(gmask, stale)) {
#pragma unroll
	    for (int j = 0; j < W; j++) {
		acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
		gone[j] = 0.f;
	    }
	    corr_pass<W, L>(acc, p, tw + t, part, N);
	}
    }
    return best;
}

/* ======================================================================== */
/* MULTI: shared-segment search (plan: fsk_b200_internal.h, fsk_b200_mplan)  */
/* ======================================================================== */
/* The candidates of one search read the same samples cut at different places.  A batch of up to
 * three candidates lays a grid of bit periods (length N = bit_nsamples, the windows tile) over the
 * ring, anchored at one candidate, and cuts every period at the offsets rho1 <= rho2 where the
 * other candidates' windows begin.  Lane (slot, part) owns the W CONSECUTIVE periods
 * m = slot*W + j and, of each, the samples n = part, part+L, ...; one walk over the twiddle
 * table gives it the three segment sums of each of its periods (acc[j][c], c = 0..2: each sample
 * is multiplied once, whatever the number of candidates).  Window w of a candidate that starts
 * `rho_c` into the periods is then
 *      tail segments (>= c) of period w + shift,  plus
 *      head segments (<  c) of period w + shift + 1, rotated by the tones' phase advance over
 *      one period (geom.rot; the correlation phase restarts at every period),
 * the second half coming from the next lane for the last of a lane's periods (shift = -1: the
 * first half comes from the previous lane instead).  The magnitude of that sum is the reference's
 * |X_k| of the window (src/fsk.c:157-159) up to a unit phase factor.  Periods n_bits (heads only)
 * and -1 (tails only, for candidates before the anchor) take the slots after the last window;
 * when only one is free they share it (mbatch.csplit). */
template <int W>
struct LaneWinM {
    unsigned beg[W];	/* ring distance of period j from the anchor (0 for a slot past the last period) */
    unsigned own;	/* bit j: this lane decides window j (one of the L lanes of the slot, round-robin) */
    unsigned exp;	/* 2 bits per (sel, j): expect value 0, 1 or 2 */
    unsigned wrapj;	/* the j whose slot is the wrap-around slot (period -1), W if it is not this lane's */
    unsigned rot0;	/* this slot starts its walk over every segment rot0 iterations in, and wraps: periods are
			 * a multiple of the bank count apart in slow modes, so slots walking in step would
			 * hit the same shared-memory banks (0: the periods spread the slots by themselves) */
};

template <int G, int W, int L>
__device__ __forceinline__ LaneWinM<W> lane_windows_multi(const fsk_b200_geom &geo, unsigned g)
{
    constexpr unsigned SLOTS = (unsigned)(W * (G / L));
    const unsigned part = g % L, slot = g / L;
    LaneWinM<W> lw;
    lw.own = 0;
    lw.exp = 0;
    lw.wrapj = W;
#pragma unroll
    for (int j = 0; j < W; j++) {
	const unsigned m = slot * W + j;
	const bool window = m < geo.n_bits, period = m <= geo.n_bits;
	lw.beg[j] = period ? geo.bit_nsamples * m : 0u;
	if (window && part == (unsigned)(j % L))
	    lw.own |= 1u << j;
	const unsigned e0 = window ? geo.expect[0][m] : 2u, e1 = window ? geo.expect[1][m] : 2u;
	lw.exp |= (e0 << (2 * j)) | (e1 << (2 * (j + W)));
	if (m == SLOTS - 1u)
	    lw.wrapj = j;
    }
    {
	/* Bank of this slot's first sample relative to slot 0's: slot * (W * N mod 32).  If two slots of
	 * the group come closer than L banks (each slot's L lanes read L neighbouring samples), the slots
	 * start their walks L samples apart instead: sample loads are then conflict-free inside the
	 * group and the twiddle rows of the slots fall into two bank classes (optimal for G/L * L rows
	 * of 16 bytes).  Where the periods already spread the slots (1200 baud: 24 banks apart) nothing
	 * rotates and all slots share their twiddle loads. */
	constexpr unsigned SPG = (unsigned)(G / L);
	const unsigned stride = (geo.bit_nsamples * (unsigned)W) & 31u;
	bool collide = false;
	for (unsigned a = 0; a < SPG; a++)
	    for (unsigned b = a + 1; b < SPG; b++) {
		const unsigned d = ((b - a) * stride) & 31u;
		collide |= d < (unsigned)L || 32u - d < (unsigned)L;
	    }
	/* iterations: slot s walks s * L samples (banks) ahead; bit 31 = the group rotates at all (uniform) */
	lw.rot0 = collide ? (slot | 0x80000000u) : 0u;
    }
    return lw;
}

/* segment sums of this lane's W periods: one walk over the period, the accumulator set switching
 * at rho1 and rho2.  Inside every segment the walk of a slot that would collide with the other
 * slots' shared-memory banks (LaneWinM.rot0 > 0) starts rot0 iterations in and wraps: the slots
 * then stay rot0 iterations -- L*rot0 banks -- apart for the length of the segment.  (A rotation
 * of the whole period does not survive: the slots re-converge at every segment boundary.)  The
 * loops are unrolled by hand, remainder LAST: the compiler's remainder-first unrolling re-aligns
 * slots whose trip counts differ. */
template <int C, int W, int L>
__device__ __forceinline__ void seg_walk(float (&acc)[W][3][4], const float *const (&ptr)[W], const float4 *tw,
	unsigned n, const unsigned end)
{
#define FSK_SEG_STEP(NN) { \
	const float4 c = tw[NN]; \
	_Pragma("unroll") \
	for (int j = 0; j < W; j++) { \
	    const float x = ptr[j][NN]; \
	    acc[j][C][0] = fmaf(x, c.x, acc[j][C][0]); \
	    acc[j][C][1] = fmaf(x, c.y, acc[j][C][1]); \
	    acc[j][C][2] = fmaf(x, c.z, acc[j][C][2]); \
	    acc[j][C][3] = fmaf(x, c.w, acc[j][C][3]); \
	} }
#pragma unroll 1
    for (; n + 3u * L < end; n += 4u * L) {
	FSK_SEG_STEP(n)
	FSK_SEG_STEP(n + L)
	FSK_SEG_STEP(n + 2u * L)
	FSK_SEG_STEP(n + 3u * L)
    }
#pragma unroll 1
    for (; n < end; n += L)
	FSK_SEG_STEP(n)
#undef FSK_SEG_STEP
}

template <int W, int L>
__device__ __forceinline__ void corr_multi(float (&acc)[W][3][4], const float *const (&p0)[W],
	const float *const (&p1)[W], const float *const (&p2)[W], const float4 *tw, unsigned part,
	unsigned rho1, unsigned rho2, unsigned N, unsigned rot0)
{
    /* first sample of this lane (n = part mod L) at or after a segment start */
    auto first_in = [&](unsigned a) { return a + ((part + (unsigned)L - a % (unsigned)L) % (unsigned)L); };
    const unsigned f0 = part, f1 = first_in(rho1), f2 = first_in(rho2);
    if (rot0 == 0u) {			/* the same for every lane of the group */
	seg_walk<0, W, L>(acc, p0, tw, f0, rho1);
	seg_walk<1, W, L>(acc, p1, tw, f1, rho2);
	seg_walk<2, W, L>(acc, p2, tw, f2, N);
    } else {
	const unsigned r = (rot0 & 0x7fffffffu) * (unsigned)L;
	const unsigned m0 = min(f0 + r, rho1), m1 = min(f1 + r, rho2), m2 = min(f2 + r, N);
	seg_walk<0, W, L>(acc, p0, tw, m0 >= rho1 ? rho1 : f0 + r, rho1);	/* from rot0 iterations in ... */
	seg_walk<0, W, L>(acc, p0, tw, f0, m0 >= rho1 ? rho1 : f0 + r);	/* ... and the ones skipped */
	seg_walk<1, W, L>(acc, p1, tw, m1 >= rho2 ? rho2 : f1 + r, rho2);
	seg_walk<1, W, L>(acc, p1, tw, f1, m1 >= rho2 ? rho2 : f1 + r);
	seg_walk<2, W, L>(acc, p2, tw, m2 >= N ? N : f2 + r, N);
	seg_walk<2, W, L>(acc, p2, tw, f2, m2 >= N ? N : f2 + r);
    }
}

/* (a + ib) * (c + is) added to (x + iy) */
__device__ __forceinline__ void rot_add(float &x, float &y, float a, float b, float c, float s)
{
    x += fmaf(c, a, -(s * b));
    y += fmaf(c, b, s * a);
}

struct FoundN {
    Found f;
    unsigned ncand;		/* candidates analysed by this call */
};

/* One search of the rx loop (src/fsk.c:449-538 as called at src/minimodem.c:1265 / :1373), all of
 * its candidates from shared segment sums.  `skip_first`: the candidate visited first has already
 * been analysed by the caller (the single-candidate fast path of the steady state) and `seed` is
 * the search's best-so-far after it.  A call, not inlined: the 36 segment accumulators then get
 * their own register allocation and the rx loop around the call keeps the one it had. */
template <int G, int W, int L>
__device__ __forceinline__ FoundN find_frame_multi(const Ring rg, unsigned pos_off,
	const fsk_b200_geom &geo, const LaneWinM<W> lw, int sel, unsigned tw_s, unsigned g, unsigned gmask,
	const fsk_b200_mkind &kind, float limit, bool pending, const Found seed, unsigned skip_first)
{
    const float *ring = static_cast<const float *>(__cvta_shared_to_generic(rg.ring_s));
    const float4 *tw = static_cast<const float4 *>(__cvta_shared_to_generic(tw_s));
    const unsigned N = geo.bit_nsamples, R = rg.R;
    const unsigned part = g % L;
    Found best = seed;
    unsigned best_order = 0, ncand = 0;

#pragma unroll 1
    for (unsigned b = 0; b < kind.nbatch; b++) {
	const fsk_b200_mbatch &mb = kind.b[b];
	const unsigned anchor_off = ring_wrap(pos_off + mb.anchor, R);
	/* period pointers; the wrap-around slot reads its segments >= csplit one grid length
	 * (SLOTS periods) earlier, which is the period before the anchor */
	const float *p0[W], *p1[W], *p2[W];
#pragma unroll
	for (int j = 0; j < W; j++) {
	    const float *fwd = ring + ring_wrap(anchor_off + lw.beg[j], R);
	    p0[j] = p1[j] = p2[j] = fwd;
	    if ((unsigned)j == lw.wrapj && mb.csplit < 3u) {
		const float *back = ring + (anchor_off >= N ? anchor_off - N : anchor_off + R - N);
		if (mb.csplit <= 0u) p0[j] = back;
		if (mb.csplit <= 1u) p1[j] = back;
		p2[j] = back;
	    }
	}
	float acc[W][3][4];
#pragma unroll
	for (int j = 0; j < W; j++)
#pragma unroll
	    for (int c = 0; c < 3; c++)
		acc[j][c][0] = acc[j][c][1] = acc[j][c][2] = acc[j][c][3] = 0.f;
	if (pending) {			/* the copies of this iteration: waited for as late as possible */
	    cp_async_wait<0>();
	    __syncwarp(gmask);
	    pending = false;
	}
	corr_multi<W, L>(acc, p0, p1, p2, tw, part, mb.rho1, mb.rho2, N, lw.rot0);

#pragma unroll 1
	for (unsigned i = (b == 0u ? skip_first : 0u); i < mb.ncand; i++) {
	    const unsigned cs = mb.cseg[i];
	    const int shift = mb.shift[i];
	    const unsigned t = mb.t[i];
	    ncand++;
	    /* this lane's partial sums of its W windows */
	    float wp[W][4];
	    if (cs == 0u && shift == 0) {
		/* the windows are whole periods */
#pragma unroll
		for (int j = 0; j < W; j++)
#pragma unroll
		    for (int k = 0; k < 4; k++)
			wp[j][k] = (acc[j][0][k] + acc[j][1][k]) + acc[j][2][k];
	    } else {
		/* tails (segments >= cs) and heads (segments < cs) of every period of this lane */
		float tl[W][4], hd[W][4];
#pragma unroll
		for (int j = 0; j < W; j++)
#pragma unroll
		    for (int k = 0; k < 4; k++) {
			if (cs == 0u) {			/* shift = +1: the whole NEXT period */
			    tl[j][k] = 0.f;
			    hd[j][k] = (acc[j][0][k] + acc[j][1][k]) + acc[j][2][k];
			} else if (cs == 1u) {
			    tl[j][k] = acc[j][1][k] + acc[j][2][k];
			    hd[j][k] = acc[j][0][k];
			} else {
			    tl[j][k] = acc[j][2][k];
			    hd[j][k] = acc[j][0][k] + acc[j][1][k];
			}
		    }
		if (shift >= 0) {
		    /* window j = tail of period j + head of period j+1 (the next lane's first for j = W-1) */
		    float nx[4];
#pragma unroll
		    for (int k = 0; k < 4; k++)
			nx[k] = __shfl_sync(gmask, hd[0][k], (g + L) & (G - 1), G);
#pragma unroll
		    for (int j = 0; j < W; j++) {
			const float h0 = j + 1 < W ? hd[j + 1 < W ? j + 1 : 0][0] : nx[0];
			const float h1 = j + 1 < W ? hd[j + 1 < W ? j + 1 : 0][1] : nx[1];
			const float h2 = j + 1 < W ? hd[j + 1 < W ? j + 1 : 0][2] : nx[2];
			const float h3 = j + 1 < W ? hd[j + 1 < W ? j + 1 : 0][3] : nx[3];
			wp[j][0] = tl[j][0]; wp[j][1] = tl[j][1]; wp[j][2] = tl[j][2]; wp[j][3] = tl[j][3];
			rot_add(wp[j][0], wp[j][1], h0, h1, geo.rot[0], geo.rot[1]);
			rot_add(wp[j][2], wp[j][3], h2, h3, geo.rot[2], geo.rot[3]);
		    }
		} else {
		    /* shift = -1: window j = tail of period j-1 (the previous lane's last for j = 0) + head of period j */
		    float pv[4];
#pragma unroll
		    for (int k = 0; k < 4; k++)
			pv[k] = __shfl_sync(gmask, tl[W - 1][k], (g + G - L) & (G - 1), G);
#pragma unroll
		    for (int j = 0; j < W; j++) {
#pragma unroll
			for (int k = 0; k < 4; k++)
			    wp[j][k] = j > 0 ? tl[j > 0 ? j - 1 : 0][k] : pv[k];
			rot_add(wp[j][0], wp[j][1], hd[j][0], hd[j][1], geo.rot[0], geo.rot[1]);
			rot_add(wp[j][2], wp[j][3], hd[j][2], hd[j][3], geo.rot[2], geo.rot[3]);
		    }
		}
	    }
	    /* first sample of this lane's windows (fp64 re-sum of near-zero bins only) */
	    const float *q[W];
	    const unsigned cand_off = ring_wrap(pos_off + t, R);
#pragma unroll
	    for (int j = 0; j < W; j++)
		q[j] = ring + ring_wrap(cand_off + lw.beg[j], R);
	    unsigned lo, hi;
	    float a;
	    const float c = frame_finish<G, W, L, true>(wp, q, lw.own, lw.exp, geo, tw, sel, g, gmask,
		    lo, hi, a);
	    /* src/fsk.c:492-501 visits the candidates in `order`; a later batch may hold an earlier
	     * candidate, so among equals the earlier one is kept (what `best_c < c` does there) */
	    const unsigned order = mb.order[i];
	    if (best.confidence < c || (best.confidence == c && c > 0.f && order < best_order)) {
		best = Found{ c, a, t, lo, hi };
		best_order = order;
		if (c >= limit && kind.nbatch == 1u)
		    return FoundN{ best, ncand };	/* first to reach the limit wins (:499) */
	    }
	}
    }
    return FoundN{ best, ncand };
}
/* ======================================================================== */
/* PREFIX: chunk-prefix table search (plan: fsk_b200_internal.h, fsk_b200_pfx) */
/* ======================================================================== */
/* One stream per warp.  pfx_build demodulates the search span once per rx-loop iteration; every
 * candidate of the coarse and of the fine search of that iteration is then analysed from the table
 * (pfx_search): a candidate costs a few loads per bit window, independent of bit_nsamples, and
 * 32 / bs candidates are analysed side by side, one lane per window boundary. */

/* what a lane needs to know about its place in a candidate slot, computed once per kernel */
struct PfxLane {
    unsigned cslot;	/* candidate slot of this lane (== cpr: none, the lane idles) */
    unsigned kk;	/* boundary index inside the slot */
    unsigned sbase;	/* first lane of the slot */
    unsigned bb;	/* offset of this lane's boundary inside a candidate (0 for an idle lane) */
    unsigned peer;	/* lane that holds the END boundary of this lane's window */
    unsigned exp;	/* expect value (0, 1, 2) of this lane's window: bits 0-1 data string, bits 2-3 sync string */
    unsigned idx0;	/* rotation-table index of the first piece of this lane's run (table build) */
    bool win;		/* this lane decides a bit window (kk < n_bits) */
};

__device__ __forceinline__ PfxLane pfx_lane(const fsk_b200_geom &geo, const fsk_b200_pfx &pg, unsigned lane)
{
    PfxLane pl;
    const unsigned nb = geo.n_bits, N = geo.bit_nsamples;
    pl.cslot = min(lane / pg.bs, pg.cpr);
    pl.kk = lane - pl.cslot * pg.bs;
    const bool in_slot = pl.cslot < pg.cpr;
    pl.sbase = in_slot ? pl.cslot * pg.bs : 0u;		/* (an idle lane adds up slot 0: sbase + bs stays inside the scratch) */
    pl.win = in_slot && pl.kk < nb;
    if (pl.win)
	pl.bb = geo.bit_begin[pl.kk];
    else if (!in_slot)
	pl.bb = 0u;
    else if (pg.tiles)
	pl.bb = pl.kk == nb ? geo.bit_begin[nb - 1u] + N : 0u;
    else
	pl.bb = pl.kk < 2u * nb ? geo.bit_begin[pl.kk - nb] + N : 0u;
    pl.peer = (lane + (pg.tiles ? 1u : nb)) & 31u;
    const unsigned e0 = pl.win ? geo.expect[0][pl.kk] : 2u, e1 = pl.win ? geo.expect[1][pl.kk] : 2u;
    pl.exp = e0 | (e1 << 2);
    pl.idx0 = (pg.s4 * lane * pg.S) % pg.fp;
    return pl;
}

/* A pair of fp32 lanes: even and odd samples summed side by side.  sm_90 has no paired fp32 FMA, so each
 * half is one FFMA / FMUL with one rounding (round to nearest); the kernel is built with -fmad=false, so
 * the explicit fma is the only contraction. */
struct F2 {
    float lo, hi;
};
__device__ __forceinline__ F2 fma2(const F2 a, const F2 b, const F2 c) { return F2{ fmaf(a.lo, b.lo, c.lo), fmaf(a.hi, b.hi, c.hi) }; }
__device__ __forceinline__ F2 mul2(const F2 a, const F2 b) { return F2{ a.lo * b.lo, a.hi * b.hi }; }

/* eight samples against both tones, phase counted from the first: (re, im) mark, (re, im) space.
 * loc[p][k] = the twiddles exp(-2 pi i b j / fftsize) of the sample pair j = 2p, 2p + 1, component
 * k = (re, im) mark, (re, im) space (j = 0: 1, 0, 1, 0), side by side as the paired sums (fma2) take them.
 * Even and odd samples are summed side by side and added at the end. */
template <class LOC>
__device__ __forceinline__ float4 pfx_local(const float4 a, const float4 b, const LOC &loc)
{
    float4 s;
    float *sp = &s.x;
#pragma unroll
    for (int k = 0; k < 4; k++) {
	F2 acc = mul2(F2{ a.x, a.y }, F2{ loc[0][k][0], loc[0][k][1] });
	acc = fma2(F2{ a.z, a.w }, F2{ loc[1][k][0], loc[1][k][1] }, acc);
	acc = fma2(F2{ b.x, b.y }, F2{ loc[2][k][0], loc[2][k][1] }, acc);
	acc = fma2(F2{ b.z, b.w }, F2{ loc[3][k][0], loc[3][k][1] }, acc);
	sp[k] = acc.lo + acc.hi;
    }
    return s;
}
/* the same for a single piece (the last chunk of a run) */
template <class LOC>
__device__ __forceinline__ float4 pfx_local4(const float4 a, const LOC &loc)
{
    float4 s;
    float *sp = &s.x;
#pragma unroll
    for (int k = 0; k < 4; k++) {
	F2 acc = mul2(F2{ a.x, a.y }, F2{ loc[0][k][0], loc[0][k][1] });
	acc = fma2(F2{ a.z, a.w }, F2{ loc[1][k][0], loc[1][k][1] }, acc);
	sp[k] = acc.lo + acc.hi;
    }
    return s;
}
/* acc += rot * s, tone by tone (complex) */
__device__ __forceinline__ void pfx_rot_acc(float4 &acc, const float4 rt, const float4 s)
{
    acc.x = fmaf(-rt.y, s.y, fmaf(rt.x, s.x, acc.x));
    acc.y = fmaf(rt.y, s.x, fmaf(rt.x, s.y, acc.y));
    acc.z = fmaf(-rt.w, s.w, fmaf(rt.z, s.z, acc.z));
    acc.w = fmaf(rt.w, s.z, fmaf(rt.z, s.w, acc.w));
}

/* The table of one search span.  Piece q = ring floats [base + 4q, base + 4q + 4) (base = ring offset of the
 * 16-byte piece that holds the search position), npieces of them are needed.  Lane g walks the pieces
 * [g * S, (g + 1) * S) two at a time (the last chunk of a run is a single piece: S is odd), stores the sum
 * of the run's EARLIER chunks in pre[g * tstride + c] and the run's total in tot[g].  The head of the ring
 * is mirrored behind its end for the length of a run and the rotation table is staged a run longer than
 * its period, so a run is three linear walks: no wrap tests. */
__device__ __forceinline__ void pfx_build(const float *ring, unsigned R, unsigned base, unsigned npieces,
	float4 *pre, float4 *tot, const float4 *twc, const float4 *loc_s, const fsk_b200_pfx &pg, const PfxLane &pl,
	unsigned lane)
{
    const unsigned S = pg.S, q0 = lane * S;
    const unsigned avail = q0 < npieces ? min(S, npieces - q0) : 0u;	/* pieces of this run that are needed */
    const unsigned nfull = min((avail + 1u) >> 1, (S - 1u) >> 1);	/* (a trailing piece nobody needs rides along) */
    unsigned off = base + 4u * q0;
    if (off >= R)
	off -= R;
    const float4 *xp = reinterpret_cast<const float4 *>(ring + off);
    const float4 *tp = twc + pl.idx0;
    const unsigned step2 = 2u * pg.s4;
    float4 *row = pre + lane * pg.tstride;
    /* the chunk-local twiddles in ordinary registers for the walk, loaded from the block's shared copy
     * through an address the compiler cannot prove uniform.  This layout was chosen for paired fp32
     * instructions, which need register pairs; on sm_90 each half is a plain FFMA that could also read a
     * uniform register, and whether kernel parameters would be faster here has not been measured. */
    float lc[4][4][2];
    {
	const float4 *lp = loc_s + (lane & pg.zero);
#pragma unroll
	for (int p = 0; p < 4; p++)
#pragma unroll
	    for (int k2 = 0; k2 < 2; k2++) {
		const float4 v = lp[p * 2 + k2];
		lc[p][2 * k2][0] = v.x; lc[p][2 * k2][1] = v.y;
		lc[p][2 * k2 + 1][0] = v.z; lc[p][2 * k2 + 1][1] = v.w;
	    }
    }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (unsigned c = 0; c < nfull; c++) {
	const float4 xa = xp[0], xb = xp[1];
	const float4 rt = *tp;
	row[c] = acc;
	pfx_rot_acc(acc, rt, pfx_local(xa, xb, lc));
	xp += 2;
	tp += step2;
    }
    if (avail == S) {				/* the run's last chunk is a single piece */
	const float4 xa = xp[0];
	const float4 rt = *tp;
	row[nfull] = acc;
	pfx_rot_acc(acc, rt, pfx_local4(xa, lc));
    }
    tot[lane] = acc;
}

/* Sums over the lanes of a candidate slot; every lane of the slot ends with the total.  LB > 0: the slot is
 * 1 << LB lanes, aligned: butterflies.  LB == 0: slots of any size (pg.bs) packed back to back; a shuffle
 * tree over such a slot needs a source clamp, a bounds test and a select per value and step, so the lanes
 * leave their terms in the stream's 32-entry scratch `red` and every lane adds up its slot's entries in
 * lane order: 1 store + bs broadcast loads.  (Measured at RTTY: the same instruction count and time as the
 * clamped shuffle tree, 12.06 against 12.12 G instructions per launch; kept for the fixed summation order
 * and the shorter dependency chain.) */
template <int LB>
__device__ __forceinline__ void pfx_slot_sum4(float &a, float &b, float &c, unsigned &d, const fsk_b200_pfx &pg,
	const PfxLane &pl, unsigned lane, float4 *red)
{
    const unsigned FULL = 0xffffffffu;
    if (LB > 0) {
#pragma unroll
	for (int o = (1 << LB) >> 1; o; o >>= 1) {
	    a += __shfl_xor_sync(FULL, a, o);
	    b += __shfl_xor_sync(FULL, b, o);
	    c += __shfl_xor_sync(FULL, c, o);
	    d += __shfl_xor_sync(FULL, d, o);
	}
    } else {
	red[lane] = make_float4(a, b, c, __uint_as_float(d));
	__syncwarp();
	const float4 *rp = red + pl.sbase;
	a = b = c = 0.f;
	d = 0u;
	for (unsigned k = 0; k < pg.bs; k++) {
	    const float4 v = rp[k];
	    a += v.x;
	    b += v.y;
	    c += v.z;
	    d += __float_as_uint(v.w);
	}
	__syncwarp();			/* the scratch is written again right away (pfx_slot_sum1) */
    }
}
template <int LB>
__device__ __forceinline__ float pfx_slot_sum1(float a, const fsk_b200_pfx &pg, const PfxLane &pl, unsigned lane,
	float4 *red)
{
    const unsigned FULL = 0xffffffffu;
    if (LB > 0) {
#pragma unroll
	for (int o = (1 << LB) >> 1; o; o >>= 1)
	    a += __shfl_xor_sync(FULL, a, o);
	return a;
    }
    float *rf = reinterpret_cast<float *>(red);
    rf[lane] = a;
    __syncwarp();
    const float *rp = rf + pl.sbase;
    a = 0.f;
    for (unsigned k = 0; k < pg.bs; k++)
	a += rp[k];
    __syncwarp();
    return a;
}

/* One round: the candidates `t` of the cpr slots (valid or not, per slot), every window of every one
 * of them from the table.  All 32 lanes take part (full-mask shuffles).  Returns this slot's
 * confidence (0 for an invalid slot or a rejected candidate); all lanes of a slot hold the same values. */
template <int LB>
__device__ __forceinline__ float pfx_round(const float *ring, unsigned R, unsigned base, unsigned r0, unsigned t,
	bool valid, const float4 *pre, const float4 *tot, const float4 *twc, const float4 *__restrict__ tw_sample,
	const fsk_b200_pfx &pg, const fsk_b200_geom &geo, const PfxLane &pl, int sel, unsigned lane, float4 *red,
	unsigned &bits_lo_out, unsigned &bits_hi_out, float &ampl_out, float2 *bit_mags = nullptr)
{
    const unsigned FULL = 0xffffffffu;
    const unsigned N = geo.bit_nsamples, nb = geo.n_bits;
    /* this lane's boundary: sample i of the span, in piece q = run l_b, piece o4 of the run; r samples of
     * the boundary's chunk (pieces qa, qa + 1) precede it */
    const unsigned i = r0 + (valid ? t : 0u) + pl.bb;
    const unsigned q = i >> 2;
    const unsigned l_b = (unsigned)(((float)q + 0.5f) * pg.inv_S);
    const unsigned o4 = q - l_b * pg.S;
    const unsigned r = ((o4 & 1u) << 2) | (i & 3u);
    const unsigned qa = q - (o4 & 1u);
    unsigned offa = base + 4u * qa;
    if (offa >= R)
	offa -= R;
    const float4 xa = *reinterpret_cast<const float4 *>(ring + offa);
    const float4 xb = *reinterpret_cast<const float4 *>(ring + offa + 4u);	/* (the mirror covers a read across the end) */
    const unsigned sm = pg.s4 * qa;
    const unsigned idx = sm - (unsigned)(((float)sm + 0.5f) * pg.inv_fp) * pg.fp;
    const float4 rt = twc[idx];
    float4 P = pre[l_b * pg.tstride + (o4 >> 1)];
    /* (pieces past the requested samples, or of the next run, are only ever met with r too small to use them) */
    pfx_rot_acc(P, rt, pfx_local(
	    make_float4(r > 0u ? xa.x : 0.f, r > 1u ? xa.y : 0.f, r > 2u ? xa.z : 0.f, r > 3u ? xa.w : 0.f),
	    make_float4(r > 4u ? xb.x : 0.f, r > 5u ? xb.y : 0.f, r > 6u ? xb.z : 0.f, 0.f), pg.loc));
    /* the end of this lane's window is another lane's boundary */
    float4 S;
    S.x = __shfl_sync(FULL, P.x, pl.peer) - P.x;
    S.y = __shfl_sync(FULL, P.y, pl.peer) - P.y;
    S.z = __shfl_sync(FULL, P.z, pl.peer) - P.z;
    S.w = __shfl_sync(FULL, P.w, pl.peer) - P.w;
    const unsigned l_e = __shfl_sync(FULL, l_b, pl.peer);
    const bool own = pl.win && valid;
    if (own) {
#pragma unroll 1
	for (unsigned l = l_b; l < l_e; l++) {		/* the lane-runs the window crosses: a few */
	    const float4 tl = tot[l];
	    S.x += tl.x; S.y += tl.y; S.z += tl.z; S.w += tl.w;
	}
    }
    /* per-window decision (src/fsk.c:158-169) and this lane's share of the sums (:271-289); magnitudes stay
     * unscaled as in frame_finish */
    const float eps_u = geo.eps_unscaled;
    float mag_mark = fast_sqrt(S.x * S.x + S.y * S.y);
    float mag_space = fast_sqrt(S.z * S.z + S.w * S.w);
    const float mag_hi = fmaxf(mag_mark, mag_space);
    /* The window is a difference of prefix values, so its fp32 error is a few ulp of the prefix at its
     * boundary, not of the window.  A loud sample earlier in the lane-run (a click) leaves the prefix far above
     * the window, and the difference cancels: past 16x the error exceeds the 2e-6 budget of needs_resum, and
     * far past it the window reads as silence.  A NaN or inf there makes the difference NaN (the unordered
     * test below).  Either way the window does not hold the sample, and the raw samples give it exactly. */
    const float pmax = fmaxf(fmaxf(fabsf(P.x), fabsf(P.y)), fmaxf(fabsf(P.z), fabsf(P.w)));
    if (own && (pmax > 16.f * mag_hi
		|| (mag_hi != 0.f && !(fminf(mag_mark, mag_space) >= eps_u + 2e-6f * mag_hi)))) {
	/* too close to the :279 threshold for fp32 sums (see needs_resum), cancelled or not finite: the window
	 * again, in fp64, phase counted from its first sample (the per-sample table, from global memory: rare) */
	double drm = 0., dim = 0., drs = 0., dis = 0.;
	unsigned qq = base + i;
	if (qq >= R)
	    qq -= R;
#pragma unroll 1
	for (unsigned n = 0; n < N; n++) {
	    const double xs = (double)ring[qq];
	    const float4 c = __ldg(tw_sample + n);
	    drm = fma(xs, (double)c.x, drm);
	    dim = fma(xs, (double)c.y, dim);
	    drs = fma(xs, (double)c.z, drs);
	    dis = fma(xs, (double)c.w, dis);
	    if (++qq == R)
		qq = 0u;
	}
	const float frm = (float)drm, fim = (float)dim, frs = (float)drs, fis = (float)dis;
	mag_mark = sqrtf(frm * frm + fim * fim);
	mag_space = sqrtf(frs * frs + fis * fis);
    }
    const bool one = mag_mark > mag_space;			/* strict: tie -> space */
    const float sig = own ? (one ? mag_mark : mag_space) : 0.f;
    const float noise = one ? mag_space : mag_mark;
    const unsigned e = (pl.exp >> (sel ? 2 : 0)) & 3u;		/* (2 for a lane without a window) */
    if (bit_mags && own)
	bit_mags[pl.kk] = make_float2(sig * geo.mag_scalar, noise * geo.mag_scalar);
    float tn = (own && noise > eps_u) ? noise : 0.f;		/* :279 */
    if (own && e != 2u && e != (one ? 1u : 0u))			/* pass 1, :211: poisons the noise sum */
	tn = INFINITY;
    const bool mark = own && one;
    float am = mark ? sig : 0.f, as = mark ? 0.f : sig;
    unsigned nm, blo = mark && pl.kk < 32u ? 1u << (pl.kk & 31u) : 0u, bhi = mark && pl.kk >= 32u ? 1u << (pl.kk & 31u) : 0u;
    /* the frame sums over the lanes of the slot (src/fsk.c:271-289); the mark count rides above the bits
     * (disjoint bit positions: OR == ADD) when the frame is short enough */
    if (nb <= 24u) {
	unsigned packed = blo | (mark ? 1u << 24 : 0u);
	pfx_slot_sum4<LB>(tn, am, as, packed, pg, pl, lane, red);
	blo = packed & 0xffffffu;
	nm = packed >> 24;
    } else {
	float z0 = 0.f, z1 = 0.f, z2 = 0.f;
	nm = mark ? 1u : 0u;
	pfx_slot_sum4<LB>(tn, am, as, nm, pg, pl, lane, red);
	/* bit positions are disjoint, so the words add like they OR */
	pfx_slot_sum4<LB>(z0, z1, z2, blo, pg, pl, lane, red);
	pfx_slot_sum4<LB>(z0, z1, z2, bhi, pg, pl, lane, red);
    }
    const float ts = am + as;
    const unsigned n_space = nb - nm;
    const float snr = fast_div(ts, tn);					/* :292, may be +inf */
    const float avg_bit_sig = ts * geo.inv_n_bits * geo.mag_scalar;	/* :295, with the 2/N of :132 */
    if (nm)
	am = fast_div(am, (float)nm);					/* :298-301 */
    if (n_space)
	as = fast_div(as, (float)n_space);
    const float other = one ? am : as;					/* :305-311 */
    float dv = own ? fast_div(fabsf(sig - other), other) : 0.f;
    dv = pfx_slot_sum1<LB>(dv, pg, pl, lane, red);
    const float divergence = dv * 2.f * geo.inv_n_bits;		/* :312-313 */
    if (!valid || tn == INFINITY) {					/* pass 1 reject, :211-212 */
	bits_lo_out = bits_hi_out = 0u;
	ampl_out = 0.f;
	return 0.f;
    }
    bits_lo_out = blo;
    bits_hi_out = bhi;
    ampl_out = avg_bit_sig;						/* :342 */
    return snr * (1.0f - divergence);					/* :336 */
}

/* fsk_find_frame (src/fsk.c:449-538) over the table: the candidates in the reference's visiting order
 * (first, +1, -1, +2, -2, ... steps; the scan ends at the first upward step that reaches try_max, and
 * downward steps below 0 are skipped: fsk_b200_pfx_kind), cpr of them per round.  The reference returns
 * the first candidate in that order whose confidence reaches `limit` (everything before it was below the
 * limit, so it is also the best so far), else the largest confidence, the earliest among equals (:492 is
 * strict). */
template <int LB>
__device__ __forceinline__ Found pfx_search(const float *ring, unsigned R, unsigned base, unsigned r0,
	const float4 *pre, const float4 *tot, const float4 *twc, const float4 *__restrict__ tw_sample,
	const fsk_b200_pfx &pg, const fsk_b200_geom &geo, const PfxLane &pl, int sel, unsigned try_first,
	const fsk_b200_pfx_kind &kd, float limit, unsigned lane, float4 *red, unsigned &ncand)
{
    const unsigned FULL = 0xffffffffu;
    const unsigned cpr = pg.cpr, k_dn = kd.k_dn, ncands = kd.ncands, step = kd.step;
    Found best = { 0.f, 0.f, 0u, 0u, 0u };
#pragma unroll 1
    for (unsigned o0 = 0; o0 < ncands; o0 += cpr) {
	const unsigned o = o0 + pl.cslot;
	const bool valid = pl.cslot < cpr && o < ncands;
	/* the o-th candidate of the visiting order */
	unsigned t = try_first;
	if (o > 2u * k_dn)
	    t = try_first + (o - k_dn) * step;
	else if (o & 1u)
	    t = try_first + ((o + 1u) >> 1) * step;
	else
	    t = try_first - (o >> 1) * step;
	unsigned lo, hi;
	float a;
	float c = pfx_round<LB>(ring, R, base, r0, t, valid, pre, tot, twc, tw_sample, pg, geo, pl, sel, lane, red, lo, hi, a);
	if (!(c > 0.f))
	    c = 0.f;					/* NaN and negatives never win (:492) */
	ncand += min(cpr, ncands - o0);
	/* the round's winner: the earliest slot that reaches the limit, else the largest confidence
	 * (the earliest among equals); slots are in visiting order */
	const unsigned reach = __ballot_sync(FULL, c >= limit);
	unsigned src;
	if (reach)
	    src = (unsigned)__ffs((int)reach) - 1u;
	else {
	    /* (c >= 0: floats order like their bit patterns; one REDUX instead of a five-stage butterfly) */
	    const unsigned cm = __reduce_max_sync(FULL, __float_as_uint(c));
	    src = (unsigned)__ffs((int)__ballot_sync(FULL, __float_as_uint(c) == cm)) - 1u;
	}
	const float cw = __shfl_sync(FULL, c, src);
	if (best.confidence < cw) {
	    best.confidence = cw;
	    best.amplitude = __shfl_sync(FULL, a, src);
	    best.start = __shfl_sync(FULL, t, src);
	    best.bits_lo = __shfl_sync(FULL, lo, src);
	    best.bits_hi = __shfl_sync(FULL, hi, src);
	    if (cw >= limit)
		break;					/* :499 */
	}
    }
    return best;
}

/* ------------------------------------------------------------------------ */
/* asynchronous ring fill: HBM -> shared memory, 16 bytes per cp.async,     */
/* every sample fetched once; bytes at or past the valid length arrive as 0 */
/* ------------------------------------------------------------------------ */


#ifndef FSK_EMU	/* inline PTX, see tests/emu */
__device__ __forceinline__ void ldgsts16(unsigned dst, const float *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void ldgsts16_zfill(unsigned dst, const float *src, unsigned valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" :: "r"(dst), "l"(src), "r"(valid) : "memory");
}
#endif

/* one linear run of `count` floats (multiple of 4): lanes take 16-byte chunks round-robin */
template <int G>
__device__ __forceinline__ void ring_run(unsigned dst, const float *__restrict__ src, unsigned count,
	unsigned g)
{
    dst += 16u * g;
    src += 4u * g;
#pragma unroll 4
    for (unsigned c = 4u * g; c < count; c += 4u * G, dst += 16u * G, src += 4 * G)
	ldgsts16(dst, src);
}

/* copies absolute indices [from, to) (multiples of 4) of stream x (valid length n)
 * into the ring and its mirror; `pos`/`pos_off` anchor the mapping
 * (to - (pos & ~3) <= R).  Bytes at or past n arrive as zeros. */
template <int G>
__device__ __forceinline__ void ring_issue(const Ring rg, const float *__restrict__ x, unsigned n,
	unsigned pos, unsigned pos_off, unsigned from, unsigned to, unsigned g)
{
    if (to <= from)
	return;
    int off0 = (int)pos_off + (int)(from - pos);	/* from - pos >= -3 */
    if (off0 < 0)
	off0 += (int)rg.R;
    unsigned off = (unsigned)off0;
    if (off >= rg.R)
	off -= rg.R;
    const unsigned ring_s = rg.ring_s;
    if (to <= n) {
	/* whole range valid: at most two linear runs plus their mirrored heads */
	const unsigned len = to - from;
	const unsigned run1 = min(len, rg.R - off), run2 = len - run1;
	ring_run<G>(ring_s + off * 4u, x + from, run1, g);
	if (run2)
	    ring_run<G>(ring_s, x + from + run1, run2, g);
	if (off < rg.pad)
	    ring_run<G>(ring_s + (rg.R + off) * 4u, x + from, min(run1, rg.pad - off), g);
	if (run2)
	    ring_run<G>(ring_s + rg.R * 4u, x + from + run1, min(run2, rg.pad), g);
	return;
    }
    /* end of the stream: per-chunk validity, zero fill */
    unsigned i = from + 4u * g;
    off += 4u * g;
    if (off >= rg.R)
	off -= rg.R;
    for (; i < to; i += 4u * G) {
	const unsigned valid = i + 4u <= n ? 16u : (i < n ? (n - i) * 4u : 0u);
	const float *s = valid ? x + i : x;
	ldgsts16_zfill(ring_s + off * 4u, s, valid);
	if (off < rg.pad)
	    ldgsts16_zfill(ring_s + (rg.R + off) * 4u, s, valid);
	off += 4u * G;
	if (off >= rg.R)
	    off -= rg.R;
    }
}


/* Block-granular fill: the ring is filled in blocks of RING_BLOCK floats that never
 * wrap (R % RING_BLOCK == 0 and blocks start at multiples of RING_BLOCK from the ring
 * origin), so every lane issues exactly 32/G 16-byte copies per block with immediate
 * offsets -- no per-chunk address arithmetic, no remainder loops. */
#ifdef FSK_RING_BLOCK
#define RING_BLOCK FSK_RING_BLOCK
#else
#define RING_BLOCK 128u
#endif

/* one whole block, all of it valid, with the lane's addresses carried by the caller: dst/src = this
 * lane's first chunk of the block, mlim = shared address below which a chunk belongs to the mirrored
 * head of the ring (copied behind its end as well) */
template <int G>
__device__ __forceinline__ void ring_block_at(unsigned dst, const float *__restrict__ src,
	unsigned mlim, unsigned R)
{
    constexpr int CPL = (int)(RING_BLOCK / 4u) / G;	/* copies per lane */
#pragma unroll
    for (int k = 0; k < CPL; k++)
	ldgsts16(dst + (unsigned)k * 16u * G, src + k * 4 * G);
    if (dst < mlim) {
#pragma unroll
	for (int k = 0; k < CPL; k++)
	    if (dst + (unsigned)k * 16u * G < mlim)
		ldgsts16(dst + R * 4u + (unsigned)k * 16u * G, src + k * 4 * G);
    }
}

/* a block that reaches past the valid length n: bytes at or past n arrive as zeros.  `first` is 64-bit:
 * the ring holds zeros past the end of a row, and a row may end just below 2^32 */
template <int G>
__device__ __forceinline__ void ring_block_tail(const Ring rg, unsigned ring_s, unsigned foff,
	const float *__restrict__ x, unsigned n, unsigned long long first, unsigned g)
{
    constexpr int CPL = (int)(RING_BLOCK / 4u) / G;
#pragma unroll
    for (int k = 0; k < CPL; k++) {
	const unsigned c = 4u * (g + (unsigned)k * G);
	const unsigned long long i = first + c;
	const unsigned valid = i + 4u <= n ? 16u : (i < n ? (n - (unsigned)i) * 4u : 0u);
	const float *sp = valid ? x + i : x;
	ldgsts16_zfill(ring_s + (foff + c) * 4u, sp, valid);
	if (foff + c < rg.pad)
	    ldgsts16_zfill(ring_s + (rg.R + foff + c) * 4u, sp, valid);
    }
}

/* ------------------------------------------------------------------------ */
/* ring fill through the TMA engine: cp.async.bulk (global -> shared, 1-D),  */
/* completion counted in bytes on a per-stream mbarrier                      */
/* ------------------------------------------------------------------------ */

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

#ifndef FSK_EMU	/* inline PTX, see tests/emu */
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity)
{
    unsigned ok;
    asm volatile("{\n.reg .pred p;\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
	    "selp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
#endif
/* bounded spin: a byte-count bug must end in a trapped kernel, never a hung GPU */
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    for (unsigned spin = 0; !mbar_try_wait(bar, parity); spin++)
	if (spin > (1u << 24))
	    __trap();
}
#ifndef FSK_EMU	/* inline PTX, see tests/emu */
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void *src, unsigned bytes, unsigned bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
	    :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
#endif

/* Lane 0 of the group copies absolute indices [from, to) (multiples of 4, to <= the
 * 4-rounded valid length, to - (pos & ~3) <= R) into the ring and its mirror with at
 * most four bulk copies (the range may wrap the ring once; the part that falls into
 * the first `pad` floats is copied to the mirror as well) and arms `bar` with the
 * byte count.  Called exactly once per barrier phase, possibly with an empty range. */
__device__ __forceinline__ void ring_issue_bulk(const Ring rg, const float *__restrict__ x,
	unsigned pos, unsigned pos_off, unsigned from, unsigned to, unsigned bar)
{
    const unsigned len = to > from ? to - from : 0u;
    const unsigned ring_s = rg.ring_s;
    int off0 = (int)pos_off + (int)(from - pos);
    if (off0 < 0)
	off0 += (int)rg.R;
    unsigned off = (unsigned)off0;
    if (off >= rg.R)
	off -= rg.R;
    /* main copy: up to two runs */
    const unsigned run1 = min(len, rg.R - off), run2 = len - run1;
    /* mirror: the parts of the runs below `pad` */
    const unsigned m1 = off < rg.pad ? min(run1, rg.pad - off) : 0u;	/* run1 starts at off */
    const unsigned m2 = min(run2, rg.pad);				/* run2 starts at 0 */
    mbar_arrive_expect_tx(bar, (run1 + run2 + m1 + m2) * 4u);
    if (run1)
	bulk_g2s(ring_s + off * 4u, x + from, run1 * 4u, bar);
    if (run2)
	bulk_g2s(ring_s, x + from + run1, run2 * 4u, bar);
    if (m1)
	bulk_g2s(ring_s + (rg.R + off) * 4u, x + from, m1 * 4u, bar);
    if (m2)
	bulk_g2s(ring_s + rg.R * 4u, x + from + run1, m2 * 4u, bar);
}

/* ------------------------------------------------------------------------ */
/* int16 PCM ingest fused into the fill (N2): a block's 128 samples arrive as 256  */
/* bytes of int16 in the UPPER half of the block's own 512 bytes of ring, and are   */
/* widened in place (x / 32768, exact) once they have landed                        */
/* ------------------------------------------------------------------------ */
/* the copies of one block: 16 chunks of 8 samples, chunk c -> bytes [256 + 16c, 272 + 16c) of the block */
template <int G>
__device__ __forceinline__ void ring_block16(unsigned ring_s, unsigned foff, const int16_t *__restrict__ src,
	unsigned g)
{
#pragma unroll
    for (int c0 = 0; c0 < 16; c0 += G) {
	const unsigned c = (unsigned)c0 + g;
	if (G <= 16 || c < 16u)
	    ldgsts16(ring_s + foff * 4u + 256u + 16u * c, reinterpret_cast<const float *>(src + 8u * c));
    }
}
/* the same for a block that reaches past the valid length n: bytes at or past n arrive as zeros */
template <int G>
__device__ __forceinline__ void ring_block16_tail(unsigned ring_s, unsigned foff, const int16_t *__restrict__ x,
	unsigned n, unsigned long long first, unsigned g)
{
#pragma unroll
    for (int c0 = 0; c0 < 16; c0 += G) {
	const unsigned c = (unsigned)c0 + g;
	if (G <= 16 || c < 16u) {
	    const unsigned long long i = first + 8u * c;
	    const unsigned valid = i + 8u <= n ? 16u : (i < n ? (n - (unsigned)i) * 2u : 0u);
	    ldgsts16_zfill(ring_s + foff * 4u + 256u + 16u * c,
		    reinterpret_cast<const float *>(valid ? x + i : x), valid);
	}
    }
}
/* widen a landed block in place: every lane reads its chunks (8 samples each), the group
 * synchronises (a chunk's 32 bytes of floats may cover another chunk's 16 bytes of int16), then
 * writes the floats, into the mirror behind the ring's end as well for the head of the ring */
template <int G>
__device__ __forceinline__ void ring_widen16(const Ring rg, unsigned foff, unsigned g, unsigned gmask)
{
    constexpr int CPL = G >= 16 ? 1 : 16 / G;
    char *blk = static_cast<char *>(__cvta_shared_to_generic(rg.ring_s)) + (size_t)foff * 4u;
    int4 v[CPL];
#pragma unroll
    for (int k = 0; k < CPL; k++) {
	const unsigned c = (unsigned)(k * G) + g;
	if (G <= 16 || c < 16u)
	    v[k] = *reinterpret_cast<const int4 *>(blk + 256u + 16u * c);
    }
    __syncwarp(gmask);
#pragma unroll
    for (int k = 0; k < CPL; k++) {
	const unsigned c = (unsigned)(k * G) + g;
	if (G <= 16 || c < 16u) {
	    const float q = 1.0f / 32768.0f;		/* a power of two: the scaling is exact */
	    float4 a, b;
	    a.x = (float)(short)(v[k].x & 0xffff) * q;  a.y = (float)(short)(v[k].x >> 16) * q;
	    a.z = (float)(short)(v[k].y & 0xffff) * q;  a.w = (float)(short)(v[k].y >> 16) * q;
	    b.x = (float)(short)(v[k].z & 0xffff) * q;  b.y = (float)(short)(v[k].z >> 16) * q;
	    b.z = (float)(short)(v[k].w & 0xffff) * q;  b.w = (float)(short)(v[k].w >> 16) * q;
	    float4 *d = reinterpret_cast<float4 *>(blk + 32u * c);
	    d[0] = a;
	    d[1] = b;
	    if (foff + 8u * c < rg.pad) {		/* pad % 4 == 0: a float4 is mirrored whole or not at all */
		float4 *m = reinterpret_cast<float4 *>(blk + (size_t)rg.R * 4u + 32u * c);
		m[0] = a;
		if (foff + 8u * c + 4u < rg.pad)
		    m[1] = b;
	    }
	}
    }
    __syncwarp(gmask);
}

/* int16 streams straight from global memory (generic path) */
struct GlobalSrc16 {
    const int16_t *x;
    unsigned n;
    __device__ __forceinline__ float operator()(unsigned i) const
    {
	return i < n ? (float)__ldg(x + i) * (1.0f / 32768.0f) : 0.0f;
    }
};

/* plain zero fill of absolute indices [from, to) (any alignment) by the group; 64-bit, as the zeros past
 * the end of a row may lie beyond 2^32 */
template <int G>
__device__ __forceinline__ void ring_zero(const Ring rg, unsigned pos, unsigned pos_off,
	unsigned long long from, unsigned long long to, unsigned g)
{
    for (unsigned long long i = from + g; i < to; i += G) {
	int off0 = (int)pos_off + (int)(i - pos);	/* i - pos >= -3, below two ring lengths */
	if (off0 < 0)
	    off0 += (int)rg.R;
	unsigned off = (unsigned)off0;
	if (off >= rg.R)
	    off -= rg.R;
	if (off >= rg.R)		/* (an early request for the NEXT window reaches up to two ring lengths ahead of pos) */
	    off -= rg.R;
	float *ring = static_cast<float *>(__cvta_shared_to_generic(rg.ring_s));
	ring[off] = 0.f;
	if (off < rg.pad)
	    ring[rg.R + off] = 0.f;
    }
}

/* a row's samples and the generic path's reader of them: float32 (SRC 0) or int16 PCM (SRC 1) */
template <int SRC> struct RowOf { typedef float T; typedef GlobalSrc Src; };
template <> struct RowOf<1> { typedef int16_t T; typedef GlobalSrc16 Src; };

/* One stream's ring fill in the rx loop.  FILL 0: cp.async blocks by all lanes of the group (int16 rows land
 * in the upper half of each block and are widened in place by `ready`); FILL 1: cp.async.bulk by lane 0,
 * completion on two mbarriers used in turn.  The caller keeps `pos`; the searches read `pos_off`. */
template <int G, int FILL, int SRC>
struct StreamRing {
    typedef typename RowOf<SRC>::T T;
    static constexpr unsigned AL = SRC ? 7u : 3u;	/* 16-byte source chunks: 4 floats, or 8 int16 */
    const Ring rg;
    const T *const x;
    const unsigned n, n4;		/* rows are readable up to a multiple of 4 (n <= 2^32 - 4) */
    const unsigned need_max, span;	/* need_max: the samples past `pos` an iteration reads at most */
    const unsigned g, gmask, bar0, bar1;
    const unsigned dst0;		/* this lane's first 16-byte chunk of the ring */
    unsigned pos_off;			/* the ring offset of `pos` */
    /* the absolute index up to which the ring content has been REQUESTED (copies issued or zeros stored): 64-bit,
     * as the requests run past the end of the row (zeros), which may lie just below 2^32 (pos < n stays 32-bit) */
    unsigned long long filled;
    unsigned long long conv;		/* SRC 1: blocks up to `conv` (ring offset coff) are widened */
    unsigned coff;
    unsigned fdst;			/* block fill: this lane's first 16-byte chunk of the block at `filled`, */
    const T *fsrc;			/* in the ring and in the row, carried instead of recomputed */
    unsigned kphase = 0;		/* bulk fill: number of barrier phases armed */
    bool tail_fix = false;		/* bulk fill: [n, n4) holds row padding, not zeros */

    __device__ __forceinline__ StreamRing(const Ring &r, unsigned bars, const T *row, unsigned len, unsigned pos,
	    unsigned need, unsigned sp, unsigned lane_g, unsigned mask)
	: rg(r), x(row), n(len), n4((len + 3u) & ~3u), need_max(need), span(sp), g(lane_g), gmask(mask),
	  bar0(bars), bar1(bars + 8u), dst0(r.ring_s + 16u * lane_g) { start(pos); }

    /* the request limit of an iteration at p: its largest window `extra` samples further on, and no more
     * than the ring holds */
    __device__ __forceinline__ unsigned long long reach(unsigned p, unsigned extra) const
    {
	return min(((unsigned long long)p + extra + need_max + 3u) & ~3ull, (unsigned long long)(p & ~AL) + rg.R);
    }

    /* the barriers (bulk fill) and the first request */
    __device__ __forceinline__ void open(unsigned pos)
    {
	if (FILL == 1 && g == 0) {
	    mbar_init(bar0, 1);
	    mbar_init(bar1, 1);
	    mbar_fence_init();
	}
	__syncwarp(gmask);
	request(reach(pos, 0u), pos);
    }

    /* FILL 0: whole blocks while they start below `to` and still fit in a ring whose oldest live sample
     * is `base` */
    __device__ __forceinline__ void request_at(unsigned long long to, unsigned base)
    {
	const unsigned long long lim = min(to, (unsigned long long)(base & ~AL) + rg.R - (RING_BLOCK - 1u));
	while (filled < lim) {
	    if constexpr (SRC) {		/* int16 rows: landing zone = upper half of the block */
		if (filled + RING_BLOCK <= n)
		    ring_block16<G>(rg.ring_s, (fdst - dst0) >> 2, x + filled, g);
		else
		    ring_block16_tail<G>(rg.ring_s, (fdst - dst0) >> 2, x, n, filled, g);
	    } else if (filled + RING_BLOCK <= n)	/* the common case: all of it valid */
		ring_block_at<G>(fdst, fsrc, rg.ring_s + rg.pad * 4u, rg.R);
	    else				/* end of the stream: zero fill */
		ring_block_tail<G>(rg, rg.ring_s, (fdst - dst0) >> 2, x, n, filled, g);
	    filled += RING_BLOCK;
	    fsrc += RING_BLOCK;
	    fdst += RING_BLOCK * 4u;
	    if (fdst == dst0 + rg.R * 4u)
		fdst = dst0;
	}
	cp_async_commit();
    }

    /* request the ring content up to absolute index `to` (rounded up to whole blocks) */
    __device__ __forceinline__ void request(unsigned long long to, unsigned pos)
    {
	if constexpr (FILL == 0)
	    request_at(to, pos);
	else {
	    static_assert(SRC == 0, "bulk fill: float rows only");
	    const unsigned to_b = (unsigned)min(to, (unsigned long long)n4);
	    const unsigned from_b = (unsigned)min(filled, (unsigned long long)to_b);
	    if (g == 0)
		ring_issue_bulk(rg, x, pos, pos_off, from_b, to_b, (kphase & 1u) ? bar1 : bar0);
	    if (n < n4 && from_b < n4 && to_b == n4 && to_b > from_b)
		tail_fix = true;
	    kphase++;
	    if (to > max(filled, (unsigned long long)n4))	/* past the end of the stream: zeros */
		ring_zero<G>(rg, pos, pos_off, max(filled, (unsigned long long)n4), to, g);
	    if (to > filled)
		filled = to;
	}
    }

    /* The top of the iteration at `pos`.  Its samples were normally requested an iteration ago (request_next);
     * what is missing -- a launch's first iteration, a restarted ring, the bulk fill -- is requested here with
     * what the next iteration can need (it starts at most `ahead` samples further).  Returns whether copies
     * are pending: the search waits for float cp.async itself; int16 rows are widened, the bulk fill settles. */
    __device__ __forceinline__ bool ready(unsigned pos, unsigned try_max, unsigned ahead)
    {
	const unsigned long long need_now = ((unsigned long long)pos + try_max - 1u + span + 3u) & ~3ull;
	const bool late = filled < need_now;	/* part of this window is only now requested */
	if (FILL != 0 || late)
	    request(reach(pos, ahead), pos);
	if (SRC) {
	    cp_async_wait<0>();
	    __syncwarp(gmask);
	    for (; conv < filled; conv += RING_BLOCK) {
		ring_widen16<G>(rg, coff, g, gmask);
		coff += RING_BLOCK;
		if (coff == rg.R)
		    coff = 0;
	    }
	    return false;
	}
	if (FILL == 0)
	    return true;
	settle(late || tail_fix);
	if (tail_fix) {
	    __syncwarp(gmask);
	    if (n >= (pos & ~3u))
		ring_zero<G>(rg, pos, pos_off, n, n4, g);
	    tail_fix = false;
	}
	__syncwarp(gmask);
	return false;
    }

    /* FILL 0, once the searches are over: the samples before the next start `npos` are dead, so ask for the
     * next iteration's now (unless the advance skips past everything requested: filled < (npos & ~AL)) */
    __device__ __forceinline__ void request_next(unsigned npos, unsigned ahead)
    {
	__syncwarp(gmask);	/* every read of this window precedes the copies */
	request_at(reach(npos, ahead), npos);
    }

    /* wait until nothing is in flight into this ring */
    __device__ __forceinline__ void drain()
    {
	if (FILL == 0)
	    cp_async_wait<0>();
	else
	    settle(true);
	__syncwarp(gmask);
    }

    /* restart the ring at `pos`, as a resumed stream starts it */
    __device__ __forceinline__ void restart(unsigned pos)
    {
	drain();
	start(pos);
    }

    /* `pos` has just moved `adv` samples on (adv < R by construction) */
    __device__ __forceinline__ void advance(unsigned pos, unsigned adv)
    {
	pos_off = ring_wrap(pos_off + adv, rg.R);
	if (filled < (pos & ~AL))		/* skipped past everything requested so far */
	    restart(pos);
	__syncwarp(gmask);	/* every read of this window precedes the next copies */
    }

private:
    __device__ __forceinline__ void start(unsigned pos)
    {
	filled = pos & ~AL;
	pos_off = pos & AL;
	fdst = dst0;
	fsrc = x + filled + 4u * g;
	conv = filled;
	coff = 0;
    }

    /* bulk fill: wait for everything requested before the latest request (all of it if `all`) */
    __device__ __forceinline__ void settle(bool all) const
    {
	if (kphase >= 2u)
	    wait_phase(kphase - 2u);
	if (all && kphase >= 1u)
	    wait_phase(kphase - 1u);
    }

    /* phase k (0-based) lives on barrier k&1 with parity (k>>1)&1 */
    __device__ __forceinline__ void wait_phase(unsigned k) const { mbar_wait((k & 1u) ? bar1 : bar0, (k >> 1) & 1u); }
};

__device__ __forceinline__ void store_frame(fsk_b200_frame *f, unsigned long long bits, float conf,
	float ampl, unsigned start)
{
    uint32_t *p = reinterpret_cast<uint32_t *>(f);
    p[0] = (uint32_t)bits;
    p[1] = (uint32_t)(bits >> 32);
    p[2] = __float_as_uint(conf);
    p[3] = __float_as_uint(ampl);
    p[4] = start;
}

#endif /* FSK_B200_DEVICE_CUH */
