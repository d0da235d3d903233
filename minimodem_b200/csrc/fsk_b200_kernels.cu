/*
 * fsk_b200_kernels.cu -- CUDA side of the FSK engine (sm_90a, H100): the kernels and
 * their host-side launch logic.  The device functions are in fsk_b200_device.cuh.
 *
 * Work decomposition (DESIGN.md has the derivation and the measurements):
 *   - one GROUP of G lanes (4, 8, 16 or 32) owns one audio stream; a warp runs 32/G
 *     streams side by side; a block of `wpb` warps is the unit the hardware scheduler
 *     hands out, so streams of different length or difficulty balance by themselves;
 *   - the stream's samples live in a per-stream shared-memory RING (whole 128-float
 *     blocks, the first bit-window length mirrored behind its end); every input sample
 *     is fetched from HBM exactly once with 16-byte cp.async copies (MODE 3: by default
 *     cp.async.bulk through the TMA engine) issued one loop iteration ahead of its use;
 *   - inside a frame candidate the lanes of a group split the bit windows and, L lanes
 *     per window, the samples of a window, and correlate each window against the mark
 *     and space tones at the FFT-bin centre frequencies (exp(-2 pi i k n / fftsize),
 *     k = b_mark, b_space) -- the two bins the reference reads out of a full FFT
 *     (src/fsk.c:157-159);
 *   - the frame statistic (src/fsk.c:271-342), the zig-zag search with early-out
 *     (src/fsk.c:477-502) and the rx-loop state machine (src/minimodem.c:1229-1407)
 *     run per group in registers.
 *
 *   - MODE 2 (shared segments) correlates every sample once per batch of up to three candidates;
 *     MODE 3 (chunk-prefix table, the default for bit periods >= 128 samples) runs one stream per
 *     warp, demodulates the whole search span ONCE per loop iteration into per-chunk prefix sums
 *     (paired fp32 sums, bank-conflict-free odd lane-runs, TMA bulk fill) and analyses every candidate of the
 *     coarse and the fine search from that table, two or three candidates side by side.
 *
 * k_rx<G,W,L,MODE,FILL,SRC> the whole rx loop per stream: MODE 0 per candidate (the headline kernel at
 *                         1200 baud), 1 generic (global memory, IEEE, serial order), 2 shared segments,
 *                         3 prefix table (G = 32; W codes the candidate slot); FILL 0 cp.async, 1 TMA bulk
 *                         copies (MODE 3 only); SRC 0 float32 rows, 1 int16 PCM rows widened inside the fill
 * k_find_frame<G,W,L,MODE> batched fsk_find_frame
 * k_tx_synth<T,VEC,LUT>   the transmitter: text (or data words) -> int16 / float32 samples
 * k_band_mags, k_detect_carrier, k_s16_to_f32, k_decode<KIND>   the "next" rows (DESIGN.md 0)
 *
 * Compiled with -fmad=false: every a*b+c below is either an explicit fmaf() (the
 * correlation sums) or two separately rounded operations, as in the reference's
 * x86-64 build.  The generic path also keeps IEEE division and square root and the
 * reference's serial summation order; the fast path uses approximate (<= 2 ulp)
 * division/sqrt and a fixed tree order for the frame statistic.
 */
#include <cuda_runtime.h>
#include <errno.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "fsk_b200_internal.h"
#include "fsk_b200_device.cuh"
#include "fsk_b200_decode_core.h"

static unsigned long long g_launches;

/* Kernel launch and dynamic shared memory go through two macros so that the test harness
 * (tests/emu: the same source compiled for the host under a SIMT emulator) can substitute its
 * own; the product build is plain CUDA. */
#ifndef FSK_EMU
#define FSK_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define FSK_DYN_SMEM(name) extern __shared__ float4 name[]
#endif

#define CUDA_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    fsk_b200_set_error("%s: %s", #call, cudaGetErrorString(e_)); return -EIO; } } while (0)


/* ------------------------------------------------------------------------ */
/* shared memory carve-up                                                   */
/* ------------------------------------------------------------------------ */
/* [twiddles: N float4 (optional)] [rings: slots x (ring_floats + pad)] [scratch: slots x n_bits float2]
 * [mbarriers: slots x 2 x u64] */
struct Smem {
    const float4 *tw;
    float *ring;
    float2 *scr;
    unsigned long long *bars;	/* two mbarriers per stream (bulk fill) */
    float4 *pre, *tot;		/* MODE 3: the stream's chunk-prefix table and its 32 lane-run totals */
    const float4 *loc;		/* MODE 3: the block's copy of fsk_b200_pfx.loc (8 float4) */
    float4 *red;		/* MODE 3, packed candidate slots: 32 entries of reduction scratch per stream */
};

/* pad: floats of the ring's head mirrored behind its end (0: no mirror); pfx_chunks: MODE 3 table entries
 * per stream (0: none) */
template <int G>
__device__ __forceinline__ Smem carve(float4 *smem, const fsk_b200_geom &geo,
	const float4 *__restrict__ tw_global, unsigned tw_in_smem, unsigned ring_floats, unsigned pad,
	unsigned pfx_chunks = 0, const float *pfx_loc = nullptr, unsigned pfx_red = 0)
{
    const unsigned N = geo.tw_entries, wpb = blockDim.x >> 5;	/* table entries staged (>= bit_nsamples) */
    Smem s;
    float4 *p = smem;
    if (tw_in_smem) {
	for (unsigned i = threadIdx.x; i < N; i += blockDim.x)
	    p[i] = tw_global[i];
	s.tw = p;
	p += N;
    } else {
	s.tw = tw_global;
    }
    const unsigned spw = 32 / G;
    const unsigned slot = (threadIdx.x >> 5) * spw + (threadIdx.x & 31) / G;
    float *rings = reinterpret_cast<float *>(p);
    if (!ring_floats)
	pad = 0u;
    s.ring = rings + (size_t)slot * (ring_floats + pad);
    float2 *scrs = reinterpret_cast<float2 *>(rings + (size_t)wpb * spw * (ring_floats + pad));
    s.scr = scrs + (size_t)slot * geo.n_bits;
    /* (an even number of float2 in all, so that what follows stays 16-byte aligned) */
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(scrs + (((size_t)wpb * spw * geo.n_bits + 1u) & ~(size_t)1u));
    s.bars = bars + 2 * slot;
    float4 *pfx = reinterpret_cast<float4 *>(bars + 2 * (size_t)wpb * spw);
    s.loc = pfx;
    if (pfx_chunks) {
	if (threadIdx.x < 32u)
	    reinterpret_cast<float *>(pfx)[threadIdx.x] = pfx_loc[threadIdx.x];
	pfx += 8;
    }
    s.pre = pfx + (size_t)slot * (pfx_chunks + 32u + pfx_red);
    s.tot = s.pre + pfx_chunks;
    s.red = s.tot + 32u;
    __syncthreads();
    return s;
}

#define GROUP_VARS \
    const unsigned lane = threadIdx.x & 31, g = lane % G, sidx = lane / G, spw = 32 / G; \
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (sidx * G)); \
    const unsigned wpb = blockDim.x >> 5, warp = threadIdx.x >> 5; \
    (void)lane

/* per-call arguments of the batched search */
struct FindArgs {
    const float *samples;
    unsigned nstreams;
    size_t stride;
    const uint32_t *offset, *nvalid, *try_first, *try_max, *try_step;
    const float *limit;
    const uint8_t *expect_sel;
    fsk_b200_frame *frames;
    float2 *bit_mags;		/* optional diagnostics: [nstreams][n_bits] (signal, noise) of the winning candidate */
};

struct RxArgs {
    const float *samples;
    const int16_t *samples16;	/* SRC 1: the same rows as int16 PCM (x / 32768), `samples` unused */
    unsigned nstreams;
    size_t stride;
    const uint32_t *nsamples;
    uint32_t nsamples_all;
    fsk_b200_frame *frames;
    uint32_t max_frames;
    fsk_b200_stream_state *states;
};

__device__ __forceinline__ float sample_at(const float *__restrict__ x, unsigned n) { return x[n]; }
/* int16 PCM rows: the reference's float = short / 32768 (exact) */
__device__ __forceinline__ float sample_at(const int16_t *__restrict__ x, unsigned n)
{
    return (float)x[n] * (1.0f / 32768.0f);
}

/* magnitude of band k over the first nsamples of x, zero-padded to fftsize (src/fsk.c:549-553) */
template <class T>
__device__ __forceinline__ float band_mag(const T *__restrict__ x, unsigned nsamples, unsigned F, unsigned k)
{
    double re = 0., im = 0.;
    unsigned r = 0;				/* (k*n) mod F, kept exact in integers */
    for (unsigned n = 0; n < nsamples; n++) {
	float sn, cs;
	sincospif(2.0f * (float)r / (float)F, &sn, &cs);
	const float xn = sample_at(x, n);
	re += (double)(xn * cs);
	im += (double)(xn * sn);
	r += k;
	if (r >= F)
	    r -= F;
    }
    const float magscalar = 1.0f / ((float)nsamples / 2.0f);	/* src/fsk.c:553 */
    const float fr = (float)re, fi = (float)im;
    return sqrtf(fr * fr + fi * fi) * magscalar;
}

/* --auto-carrier (src/minimodem.c:1179-1220) in the per-candidate rx kernel (AUTO = 1) */
struct AutoArgs {
    fsk_b200_auto_state *states;
    uint32_t *rec_band;		/* optional: [nstreams][max_frames], the mark band of every record */
    const float2 *unit;		/* (cos, -sin)(2 pi r / fftsize), r = 0 .. fftsize-1, as fsk_b200_cuda_set_table rounds them */
    float threshold;		/* carrier_autodetect_threshold */
    float scan_n;		/* nsamples_per_scan = min(nsamples_per_bit, fftsize), a float as in the reference */
    int b_shift;		/* :1200-1203, negated under --inverted */
    unsigned fftsize, nbands;
    unsigned half_ring;		/* samplebuf_size / 2: the refill of the virtual ring count */
    unsigned expect_nsamples;	/* the loop's own stop rule; lc.expect_nsamples above it is a live stream's holdback */
};

/* fsk_detect_carrier (src/fsk.c:543-581) on one window, by the G lanes of a group: lane g takes the
 * bands 1 + g, 1 + g + G, ...; the rule of k_detect_carrier picks the first strictly largest
 * magnitude at or above the threshold.  Returns the band or -1. */
template <int G, class T>
__device__ __forceinline__ int detect_group(const T *__restrict__ x, unsigned nsamples, const AutoArgs &au,
	unsigned g, unsigned gmask)
{
    float max_mag = 0.0f;
    int best = -1;
    for (unsigned k = 1 + g; k < au.nbands; k += G) {
	const float m = band_mag(x, nsamples, au.fftsize, k);
	if (m < au.threshold)
	    continue;
	if (max_mag < m) {
	    max_mag = m;
	    best = (int)k;
	}
    }
    for (int o = G / 2; o; o >>= 1) {
	const float om = __shfl_xor_sync(gmask, max_mag, o);
	const int ob = __shfl_xor_sync(gmask, best, o);
	if (ob >= 0 && (best < 0 || max_mag < om || (max_mag == om && ob < best))) {
	    max_mag = om;
	    best = ob;
	}
    }
    return best;
}

/* ------------------------------------------------------------------------ */
/* K1: batched fsk_find_frame (src/fsk.c:449-538), one search per stream     */
/* ------------------------------------------------------------------------ */

/* MODE 0: fast (ring + compile-time split), 1: generic from global memory */
template <int G, int W, int L, int MODE>
__global__ void __launch_bounds__(256)
k_find_frame(const __grid_constant__ fsk_b200_geom geo, const float4 *__restrict__ tw_global,
	unsigned tw_in_smem, unsigned ring_floats, const __grid_constant__ FindArgs a)
{
    FSK_DYN_SMEM(smem4);
    const Smem sm = carve<G>(smem4, geo, tw_global, tw_in_smem, ring_floats, (geo.bit_nsamples + 3u) & ~3u);
    GROUP_VARS;
    const Ring rg = { smem_u32(sm.ring), ring_floats, (geo.bit_nsamples + 3u) & ~3u };
    const unsigned tw_s = tw_in_smem ? smem_u32(sm.tw) : 0u;	/* the fast path requires the table in shared memory */
    const LaneWin<W> lw = lane_windows<G, W, L>(geo, g);

    for (unsigned s = (blockIdx.x * wpb + warp) * spw + sidx; s < a.nstreams;
	    s += gridDim.x * wpb * spw) {
	const float *x = a.samples + (size_t)s * a.stride;
	const unsigned off = a.offset ? a.offset[s] : 0u;
	const unsigned n = a.nvalid[s];
	const unsigned tmax = a.try_max[s];
	unsigned tstep = a.try_step[s];
	if (tstep == 0)
	    tstep = 1;
	const int sel = a.expect_sel ? (a.expect_sel[s] ? 1 : 0) : 0;
	unsigned long long bits = 0;
	float ampl = 0.f, conf = 0.f;
	unsigned start = 0;
	if (tmax) {
	    const unsigned from = off & ~3u;
	    const unsigned to = (off + tmax - 1u + geo.span + 3u) & ~3u;
	    if (MODE == 0 && to - from <= ring_floats) {
		__syncwarp(gmask);
		ring_issue<G>(rg, x, n, off, off & 3u, from, to, g);
		cp_async_commit();
		cp_async_wait<0>();
		__syncwarp(gmask);
		/* the search inlined, as k_rx has it: built as a separate __noinline__ call taking the LaneWin by
		 * value, the sm_90a code returned wrong bits for the first window of every lane at W = 4, L = 1
		 * (magnitudes, decisions and confidence right; tests/test_gpu_instantiations.py) */
		unsigned ncand = 0;
		const Found f = find_frame_fast_body<G, W, L>(rg, off & 3u, geo, lw, sel, tw_s, g, gmask,
			a.try_first[s], tmax, tstep, a.limit[s], false, ncand);
		conf = f.confidence;
		ampl = f.amplitude;
		start = f.start;
		bits = ((unsigned long long)f.bits_hi << 32) | f.bits_lo;
		if (a.bit_mags) {		/* analyse the winner once more, exporting its per-bit magnitudes */
		    unsigned lo, hi;
		    float am;
		    bool nopend = false;
		    __syncwarp(gmask);
		    (void)frame_analyze_fast<G, W, L>(rg, ring_wrap((off & 3u) + f.start, rg.R), geo, lw, sel, tw_s,
			    g, gmask, lo, hi, am, nopend, a.bit_mags + (size_t)s * geo.n_bits);
		}
	    } else {
		const GlobalSrc src = { x, n };
		conf = find_frame<G, GlobalSrc>(src, off, geo, sel, sm.tw, sm.scr, g, gmask,
			a.try_first[s], tmax, tstep, a.limit[s], bits, ampl, start);
		if (a.bit_mags) {
		    unsigned long long b2;
		    float am;
		    (void)frame_analyze<G, GlobalSrc>(src, off + start, geo, sel, sm.tw, sm.scr, g, gmask, b2, am,
			    a.bit_mags + (size_t)s * geo.n_bits);
		}
	    }
	}
	if (g == 0)
	    store_frame(a.frames + s, bits, conf, ampl, start);
    }
}

/* ------------------------------------------------------------------------ */
/* K2: the rx loop (src/minimodem.c:1137-1463) for whole streams            */
/* ------------------------------------------------------------------------ */

/* FILL 0: cp.async (LDGSTS) by all lanes of the group, the next iteration's samples asked for as
 * soon as the searches of this one are over rather than at the top of the next iteration;
 * FILL 1 (MODE 3): cp.async.bulk (TMA engine) issued by lane 0 with mbarrier completion. */
/* 128 threads x 4 blocks caps the kernel at 128 registers per thread: 8 blocks of 64 threads per
 * SM, which is also what the shared-memory rings allow */
#ifndef FSK_MINBLOCKS
#define FSK_MINBLOCKS 4
#endif
#ifndef FSK_MAXTHREADS
#define FSK_MAXTHREADS 128
#endif
/* MODE 3 runs one stream per warp and shares one rotation table per block, so its blocks are large
 * (up to 16 streams): 512 threads x 1 block caps it at 128 registers per thread */
#ifndef FSK_PFX_MAXTHREADS
#define FSK_PFX_MAXTHREADS 512
#endif
/* SRC 0: float32 rows; SRC 1: int16 PCM rows (N2, src/simpleaudio-sndfile.c:43-57), widened to the
 * reference's float = short / 32768 inside the ring fill: 2 bytes per sample of HBM traffic.
 * AUTO 1 (MODE 0, FILL 0 only): --auto-carrier.  Each stream has its own tone table in shared memory
 * behind the mbarriers (geo.tw_entries float4 per slot, filled from au.unit when a band is accepted),
 * and scans for a carrier band over its virtual ring count while it has none (DESIGN.md 5). */
template <int G, int W, int L, int MODE, int FILL, int SRC = 0, int AUTO = 0>
__global__ void __launch_bounds__(MODE == 3 ? FSK_PFX_MAXTHREADS : FSK_MAXTHREADS,
	MODE == 3 ? 1 : (MODE == 2 && G >= 16) ? 3 : FSK_MINBLOCKS)
k_rx(const __grid_constant__ fsk_b200_geom geo, const __grid_constant__ fsk_b200_loopc lc,
	const float4 *__restrict__ tw_global, unsigned tw_in_smem, unsigned ring_floats,
	unsigned lookahead, const __grid_constant__ RxArgs a, const __grid_constant__ fsk_b200_mplan mp,
	const float4 *__restrict__ tw_sample, const __grid_constant__ fsk_b200_pfx pg,
	const __grid_constant__ AutoArgs au)
{
    static_assert(FILL == 0 || MODE == 3, "bulk fill: prefix-table kernel only");
    static_assert(!AUTO || (MODE == 0 && FILL == 0), "auto-carrier: per-candidate kernel, cp.async fill");
    FSK_DYN_SMEM(smem4);
    /* MODE 3 (chunk-prefix table): the ring's mirror covers one lane-run of the table build (not a bit window);
     * the staged table (tw_global) is the chunk-rotation table, the per-sample one stays in global memory
     * (tw_sample) */
    const unsigned ring_pad = MODE == 3 ? 4u * pg.S + 8u : (geo.bit_nsamples + 3u) & ~3u;
    constexpr int LB = W == 1 ? 0 : W;		/* MODE 3: log2 of the candidate slot (0: packed slots of any size) */
    const Smem sm = carve<G>(smem4, geo, tw_global, tw_in_smem, ring_floats, ring_pad, MODE == 3 ? 32u * pg.tstride : 0u,
	    &pg.loc[0][0][0], (MODE == 3 && LB == 0) ? 32u : 0u);
    GROUP_VARS;
    const Ring rg = { smem_u32(sm.ring), ring_floats, ring_pad };
    /* the fast path requires the table in shared memory; AUTO: this slot's own table */
    float4 *const tw_auto = AUTO ? reinterpret_cast<float4 *>(sm.bars - 2u * (warp * spw + sidx) + 2u * wpb * spw)
	    + (size_t)(warp * spw + sidx) * geo.tw_entries : nullptr;
    const unsigned tw_s = AUTO ? smem_u32(tw_auto) : tw_in_smem ? smem_u32(sm.tw) : 0u;
    /* MODE 2 (shared-segment search) owns CONSECUTIVE bit periods per lane, MODE 0 interleaved windows */
    const LaneWin<W> lw = lane_windows<G, W, L>(geo, g);
    const LaneWinM<W> lwm = lane_windows_multi<G, W, L>(geo, g);
    const PfxLane pfl = MODE == 3 ? pfx_lane(geo, pg, lane) : PfxLane();
    const unsigned pre_s = smem_u32(sm.pre), tot_s = smem_u32(sm.tot), loc_s = smem_u32(sm.loc), red_s = smem_u32(sm.red);
    const unsigned R = ring_floats;

    for (unsigned s = (blockIdx.x * wpb + warp) * spw + sidx; s < a.nstreams;
	    s += gridDim.x * wpb * spw) {
	fsk_b200_stream_state st = a.states[s];
	if (st.done)
	    continue;
	const float *x = SRC ? (const float *)nullptr : a.samples + (size_t)s * a.stride;
	const int16_t *x16 = SRC ? a.samples16 + (size_t)s * a.stride : (const int16_t *)nullptr;
	/* a row never extends past its stride (per-stream lengths are caller data) */
	const unsigned n = (unsigned)min((size_t)(a.nsamples ? a.nsamples[s] : a.nsamples_all), a.stride);
	fsk_b200_frame *out = a.frames + (size_t)s * a.max_frames;
	/* 16-byte chunks of the source line up with 16-byte chunks of the ring: 4 floats, or 8 int16 */
	constexpr unsigned AL = SRC ? 7u : 3u;

	unsigned pos = (unsigned)st.pos;
	unsigned nframes = st.nframes;
	unsigned carrier = st.carrier, noconfidence = st.noconfidence;
	float track_amplitude = st.track_amplitude, peak_confidence = st.peak_confidence;
	unsigned long long carrier_nsamples = st.carrier_nsamples;
	float confidence_total = st.confidence_total, amplitude_total = st.amplitude_total;
	unsigned nframes_decoded = st.nframes_decoded;
	unsigned done = 0;
	unsigned ncand = 0, nsearch = 0;	/* statistics: candidates analysed, searches run */
	bool mhint = st.reserved != 0u;		/* MODE 2: the latest coarse search needed more than its first candidate */
	/* AUTO: the accepted mark band (0: none, :1180) and the virtual ring count */
	unsigned band = AUTO ? au.states[s].carrier_band : 0u, vring = AUTO ? au.states[s].v : 0u;
	/* fsk_set_tones_by_bandshift (src/fsk.c:585-598) for this stream's table: entry e of the tone b is
	 * the unit-circle entry (b * e) mod fftsize, the value fsk_b200_cuda_set_table computes for it */
	auto set_tones = [&](unsigned bm) {
	    const unsigned bsp = (unsigned)((int)bm + au.b_shift);
	    __syncwarp(gmask);
	    for (unsigned e = g; e < geo.tw_entries; e += G) {
		const float2 um = au.unit[(unsigned)(((unsigned long long)bm * e) % au.fftsize)];
		const float2 us = au.unit[(unsigned)(((unsigned long long)bsp * e) % au.fftsize)];
		tw_auto[e] = make_float4(um.x, um.y, us.x, us.y);
	    }
	    __syncwarp(gmask);
	};
	if (AUTO && band)
	    set_tones(band);

	/* ring bookkeeping (MODE 0): ring offset of `pos`, and the absolute index up to
	 * which the ring content has been REQUESTED (copies issued or zeros stored) */
	unsigned pos_off = pos & AL;
	unsigned filled = pos & ~AL;
	unsigned conv = filled, coff = 0;		/* SRC 1: blocks up to `conv` (ring offset coff) are widened */
	const unsigned need_max = lc.try_max_nocarrier - 1u + geo.span;
	const unsigned n4 = (n + 3u) & ~3u;		/* rows are readable up to a multiple of 4 */
	const unsigned bar0 = smem_u32(sm.bars), bar1 = bar0 + 8u;
	unsigned kphase = 0;				/* bulk fill: number of barrier phases armed */
	bool tail_fix = false;				/* bulk fill: [n, n4) holds row padding, not zeros */

	const unsigned ring_s = rg.ring_s;
	/* block fill: this lane's running source and destination (its first 16-byte chunk of
	 * the block that starts at absolute index `filled`), carried instead of recomputed */
	const unsigned dst0 = ring_s + 16u * g, dst_end = dst0 + R * 4u;
	const unsigned mlim = ring_s + rg.pad * 4u;	/* chunks below this are mirrored behind the end */
	unsigned fdst = dst0;
	const float *fsrc = SRC ? x : x + filled + 4u * g;
	/* request the ring content up to absolute index `to` (rounded up to whole blocks) */
	auto request_at = [&](unsigned to, unsigned base) {
	    /* FILL 0 only: whole blocks while they start below `to` and still fit in a ring
	     * whose oldest live sample is `base` */
	    const unsigned lim = min(to, (base & ~AL) + R - (RING_BLOCK - 1u));
	    while (filled < lim) {
		if (SRC) {				/* int16 rows: landing zone = upper half of the block */
		    if (filled + RING_BLOCK <= n)
			ring_block16<G>(ring_s, (fdst - dst0) >> 2, x16 + filled, g);
		    else
			ring_block16_tail<G>(ring_s, (fdst - dst0) >> 2, x16, n, filled, g);
		} else if (filled + RING_BLOCK <= n)	/* the common case: all of it valid */
		    ring_block_at<G>(fdst, fsrc, mlim, R);
		else					/* end of the stream: zero fill */
		    ring_block_tail<G>(rg, ring_s, (fdst - dst0) >> 2, x, n, filled, g);
		filled += RING_BLOCK;
		fsrc += RING_BLOCK;
		fdst += RING_BLOCK * 4u;
		if (fdst == dst_end)
		    fdst = dst0;
	    }
	    cp_async_commit();
	};
	auto request = [&](unsigned to) {
	    if (FILL == 0) {
		request_at(to, pos);
	    } else {
		const unsigned to_b = min(to, n4);
		const unsigned from_b = min(filled, to_b);
		if (g == 0)
		    ring_issue_bulk(rg, x, pos, pos_off, from_b, to_b, (kphase & 1u) ? bar1 : bar0);
		if (n < n4 && from_b < n4 && to_b == n4 && to_b > from_b)
		    tail_fix = true;
		kphase++;
		if (to > max(filled, n4))		/* past the end of the stream: zeros */
		    ring_zero<G>(rg, pos, pos_off, max(filled, n4), to, g);
		if (to > filled)
		    filled = to;
	    }
	};
	/* bulk fill: wait for everything requested before the latest request (all of it if `all`) */
	auto settle = [&](bool all) {
	    /* phase k (0-based) lives on barrier k&1 with parity (k>>1)&1 */
	    if (kphase >= 2u) {
		const unsigned k = kphase - 2u;
		mbar_wait((k & 1u) ? bar1 : bar0, (k >> 1) & 1u);
	    }
	    if ((all || tail_fix) && kphase >= 1u) {
		const unsigned k = kphase - 1u;
		mbar_wait((k & 1u) ? bar1 : bar0, (k >> 1) & 1u);
	    }
	    if (tail_fix) {
		__syncwarp(gmask);
		if (n >= (pos & ~3u))
		    ring_zero<G>(rg, pos, pos_off, n, n4, g);
		tail_fix = false;
	    }
	    __syncwarp(gmask);
	};
	/* wait until nothing is in flight into this ring */
	auto drain = [&]() {
	    if (FILL == 0) {
		cp_async_wait<0>();
	    } else {
		if (kphase >= 2u) {
		    const unsigned k = kphase - 2u;
		    mbar_wait((k & 1u) ? bar1 : bar0, (k >> 1) & 1u);
		}
		if (kphase >= 1u) {
		    const unsigned k = kphase - 1u;
		    mbar_wait((k & 1u) ? bar1 : bar0, (k >> 1) & 1u);
		}
	    }
	    __syncwarp(gmask);
	};
	if (MODE != 1) {
	    if (FILL == 1) {
		if (g == 0) {
		    mbar_init(bar0, 1);
		    mbar_init(bar1, 1);
		    mbar_fence_init();
		}
	    }
	    __syncwarp(gmask);
	    request(min((pos + need_max + 3u) & ~3u, (pos & ~AL) + R));
	}

	for (;;) {
	    if (pos >= n) { done = 1; break; }			/* :1176 */
	    const unsigned remaining = n - pos;
	    if (AUTO) {
		/* a live stream's holdback (lc.expect_nsamples raised above the loop's own rule) stops the
		 * loop before the scan: the refill below must not see where the stream was cut */
		if (lc.expect_nsamples > au.expect_nsamples && remaining < lc.expect_nsamples) { done = 1; break; }
		if (vring > remaining)				/* (a state that does not fit this row) */
		    vring = remaining;
		if (vring < au.half_ring)			/* :1158-1174, the refill */
		    vring += min(remaining - vring, au.half_ring);
		if (band == 0) {				/* :1181-1220 */
		    const float sf = au.scan_n;
		    const unsigned sn = (unsigned)sf;
		    unsigned i = 0;
		    int found = -1;
		    for (; (float)i + sf <= (float)vring; i = (unsigned)((float)i + sf)) {
			if (SRC)
			    found = detect_group<G>(x16 + pos + i, sn, au, g, gmask);
			else
			    found = detect_group<G>(x + pos + i, sn, au, g, gmask);
			if (found >= 0)
			    break;
		    }
		    const int b_space = found + au.b_shift;
		    if (found >= 0 && b_space >= 1 && b_space < (int)au.nbands) {
			band = (unsigned)found;
			set_tones(band);			/* and search at the ring start */
		    } else {
			const unsigned adv = min((unsigned)((float)i + sf), vring);
			pos += adv;
			vring -= adv;
			/* restart the ring at the new position, as a resumed stream starts it */
			drain();
			filled = pos & ~AL;
			pos_off = pos & AL;
			fdst = dst0;
			fsrc = SRC ? x : x + filled + 4u * g;
			conv = filled;
			coff = 0;
			__syncwarp(gmask);
			continue;
		    }
		}
	    }
	    if (remaining < lc.expect_nsamples) { done = 1; break; }	/* :1229 */
	    if (nframes >= a.max_frames)
		break;						/* output full: resumable */

	    unsigned try_max = carrier ? lc.try_max_carrier : lc.try_max_nocarrier;	/* :1236-1241 */
	    unsigned try_step = try_max / 3u;			/* :1248-1251 */
	    if (try_step == 0)
		try_step = 1;
	    const unsigned try_first = carrier ? lc.nsamples_overscan : 0u;	/* :1263 */
	    const int sel = carrier ? 0 : 1;			/* :1270 data / sync string */

	    bool pending = false;
	    if (MODE != 1) {
		/* The samples of this iteration were normally requested an iteration ago (FILL 0,
		 * below); whatever is missing -- first iteration of a launch, a restarted ring, the
		 * bulk fill -- is requested here together with what the next iteration can need
		 * (it starts at most `lookahead` samples further) */
		const unsigned need_now = (pos + try_max - 1u + geo.span + 3u) & ~3u;
		const bool late = filled < need_now;	/* part of this window is only now requested */
		if (FILL != 0 || late)
		    request(min((pos + lookahead + need_max + 3u) & ~3u, (pos & ~AL) + R));
		if (SRC) {
		    /* int16 rows: everything requested so far has to land and be widened in place
		     * before the search reads it (the float fill lets the search itself wait) */
		    cp_async_wait<0>();
		    __syncwarp(gmask);
		    while (conv < filled) {
			ring_widen16<G>(rg, coff, g, gmask);
			conv += RING_BLOCK;
			coff += RING_BLOCK;
			if (coff == R)
			    coff = 0;
		    }
		    pending = false;
		} else if (FILL == 0) {
		    /* the search waits for all copies itself, right before its first correlation */
		    pending = true;
		} else
		    settle(late);
	    }
	    const GlobalSrc gsrc = { x, n };
	    const GlobalSrc16 gsrc16 = { x16, n };

	    unsigned long long bits;
	    float amplitude, confidence;
	    unsigned frame_start;
	    Found refined = { 0.f, 0.f, 0u, 0u, 0u };
	    if (MODE != 1) {
		/* one (inlined) search site, taken a second time for the refinement of :1357-1389: whether
		 * that happens is a pure function of the first result and the loop state, so it is
		 * decided here and the state machine below only merges the outcome */
		Found first = { 0.f, 0.f, 0u, 0u, 0u };
		unsigned step = try_step;
		float limit = lc.confidence_search_limit;
		int which = sel;
		for (int pass = 0;; pass++) {
		    nsearch++;
		    Found f;
		    if (MODE == 3) {
			/* :1265, :1378 from the chunk-prefix table of this iteration's search span, built once
			 * (before the coarse search) for both */
			/* (shared-window addresses turned back into pointers here, so that the loads stay LDS/STS) */
			const float *ringp = static_cast<const float *>(__cvta_shared_to_generic(rg.ring_s));
			float4 *pre = static_cast<float4 *>(__cvta_shared_to_generic(pre_s));
			float4 *tot = static_cast<float4 *>(__cvta_shared_to_generic(tot_s));
			const float4 *twc = static_cast<const float4 *>(__cvta_shared_to_generic(tw_s));
			const float4 *locp = static_cast<const float4 *>(__cvta_shared_to_generic(loc_s));
			float4 *redp = static_cast<float4 *>(__cvta_shared_to_generic(red_s));
			const unsigned base = pos_off & ~3u;
			if (pass == 0) {
			    if (pending) {
				cp_async_wait<0>();
				__syncwarp(gmask);
				pending = false;
			    }
			    pfx_build(ringp, R, base, ((pos_off & 3u) + try_max - 1u + geo.span) / 4u + 1u, pre, tot,
				    twc, locp, pg, pfl, lane);
			    __syncwarp(gmask);
			}
			f = pfx_search<LB>(ringp, R, base, pos_off & 3u, pre, tot, twc, tw_sample, pg, geo, pfl, which,
				try_first, pg.kind[(carrier ? 1 : 0) + (pass ? 2 : 0)], limit, lane, redp, ncand);
		    } else if (MODE == 2) {
			/* :1265, :1378 from shared segment sums.  Which plan: the window is the one chosen at the
			 * top of the iteration (carrier then), coarse or fine.  A coarse search in the steady
			 * state ends at its first candidate (:499), and one candidate alone is cheapest analysed
			 * by itself: that is tried first unless the previous coarse search of this stream needed
			 * more than one (mhint); the fine search visits all of its candidates anyway. */
			const fsk_b200_mkind &kind = mp.kind[(carrier ? 1 : 0) + (pass ? 2 : 0)];
			Found seed = { 0.f, 0.f, 0u, 0u, 0u };
			unsigned skip = 0;
			bool decided = false;
			if (pass == 0 && !mhint && !mp.always) {
			    unsigned lo, hi;
			    float am;
			    const float c = frame_analyze_fast<G, W, L, true, LaneWinM<W> >(rg,
				    ring_wrap(pos_off + try_first, R), geo, lwm, which, tw_s, g, gmask, lo, hi, am,
				    pending);
			    ncand++;
			    if (0.f < c) {					/* src/fsk.c:492 */
				seed = Found{ c, am, try_first, lo, hi };
				decided = c >= limit;			/* :499 */
			    }
			    skip = 1;
			    mhint = !decided;
			}
			if (decided)
			    f = seed;
			else {
			    const FoundN r = find_frame_multi<G, W, L>(rg, pos_off, geo, lwm, which, tw_s, g, gmask,
				    kind, limit, pending, seed, skip);
			    f = r.f;
			    ncand += r.ncand;
			    if (pass == 0 && !skip)
				mhint = r.ncand > 1u;
			}
		    } else if (MODE == 0 && pass == 1 && lc.slide)
			/* :1373, the fine search: its candidates in ascending order, each from the one before */
			f = find_frame_slide<G, W, L>(rg, pos_off, geo, lw, which, tw_s, g, gmask, try_first, try_max,
				step, ncand);
		    else
			f = find_frame_fast_body<G, W, L>(rg, pos_off, geo, lw, which, tw_s, g,
				gmask, try_first, try_max, step, limit, pending, ncand);
		    if (pass) {
			refined = f;
			break;
		    }
		    first = f;
		    float c = f.confidence;
		    const bool below_peak = c < peak_confidence * 0.75f;	/* :1278 */
		    if (f.amplitude < track_amplitude * 0.25f)		/* :1286 */
			c = 0.f;
		    if (!(c > lc.confidence_threshold) || !(below_peak || !carrier) || !(c < INFINITY)
			    || try_step <= 1u)
			break;
		    step = try_max / 8u;
		    if (step == 0)
			step = 1;
		    limit = INFINITY;
		    which = 0;
		    pending = false;
		}
		confidence = first.confidence;
		amplitude = first.amplitude;
		frame_start = first.start;
		bits = ((unsigned long long)first.bits_hi << 32) | first.bits_lo;
		if (FILL == 0) {
		    /* The searches are over, so the samples before the next start are dead: ask for
		     * the next iteration's samples now, ahead of the bookkeeping below, instead of
		     * right before they are needed.  `adv` restates the advance of :1318/:1407;
		     * should it ever be short, the top of the loop asks for the rest. */
		    float c = first.confidence;
		    if (first.amplitude < track_amplitude * 0.25f)
			c = 0.f;
		    const unsigned fs = refined.confidence > first.confidence ? refined.start : first.start;
		    const unsigned adv = c <= lc.confidence_threshold ? try_max
			    : fs + lc.frame_nsamples - lc.nsamples_overscan;
		    const unsigned npos = pos + adv;
		    if (adv <= remaining && filled >= (npos & ~AL)) {
			__syncwarp(gmask);	/* every read of this window precedes the copies */
			request_at(min((npos + lookahead + need_max + 3u) & ~3u, (npos & ~AL) + R), npos);
		    }
		    /* (The bulk fill of MODE 3 asks at the top of the next iteration.  Asking here as well
		     * costs one more barrier phase per iteration, and the state machine below is too short
		     * to hide a copy; the other warps of the SM do that already.) */
		}
	    } else if (SRC)
		confidence = find_frame<G, GlobalSrc16>(gsrc16, pos, geo, sel, sm.tw, sm.scr, g, gmask,
			try_first, try_max, try_step, lc.confidence_search_limit,
			bits, amplitude, frame_start);
	    else
		confidence = find_frame<G, GlobalSrc>(gsrc, pos, geo, sel, sm.tw, sm.scr, g, gmask,
			try_first, try_max, try_step, lc.confidence_search_limit,
			bits, amplitude, frame_start);

	    bool want_refine = false;
	    if (confidence < peak_confidence * 0.75f) {		/* :1278-1282 */
		want_refine = true;
		peak_confidence = 0.f;
	    }
	    if (amplitude < track_amplitude * 0.25f)		/* :1286 */
		confidence = 0.f;

	    unsigned advance;
	    if (confidence <= lc.confidence_threshold) {	/* :1292 */
		if (++noconfidence > 20u) {			/* :1295 */
		    if (carrier) {
			/* report_no_carrier(), :1299-1302, as a record */
			if (g == 0)
			    store_frame(out + nframes, carrier_nsamples, confidence_total,
				    amplitude_total, FSK_B200_FRAME_REPORT);
			if (AUTO && g == 0 && au.rec_band)
			    au.rec_band[(size_t)s * a.max_frames + nframes] = band;
			nframes++;
			carrier = 0;				/* :1303-1308 */
			carrier_nsamples = 0;
			confidence_total = 0.f;
			amplitude_total = 0.f;
			nframes_decoded = 0;
			track_amplitude = 0.f;
		    }
		    if (AUTO)
			band = 0;				/* :1297 */
		}
		advance = try_max;				/* :1318 */
	    } else {
		unsigned acquired = 0;
		carrier_nsamples += lc.frame_nsamples;		/* :1324 */
		if (carrier) {
		    carrier_nsamples += frame_start;		/* :1329-1330: the COARSE start */
		    carrier_nsamples -= lc.nsamples_overscan;
		} else {					/* :1332-1355 */
		    carrier = 1;
		    acquired = FSK_B200_FRAME_ACQUIRED;
		    want_refine = true;
		}
		if (want_refine && confidence < INFINITY && try_step > 1u) {	/* :1357-1389 */
		    try_step = try_max / 8u;
		    if (try_step == 0)
			try_step = 1;
		    unsigned long long bits2;
		    float amplitude2, confidence2;
		    unsigned frame_start2;
		    /* `carrier` is 1 by now, so the data string is searched (:1378) */
		    if (MODE != 1) {
			confidence2 = refined.confidence;	/* searched above */
			amplitude2 = refined.amplitude;
			frame_start2 = refined.start;
			bits2 = ((unsigned long long)refined.bits_hi << 32) | refined.bits_lo;
		    } else if (SRC)
			confidence2 = find_frame<G, GlobalSrc16>(gsrc16, pos, geo, 0, sm.tw, sm.scr, g,
				gmask, try_first, try_max, try_step, INFINITY,
				bits2, amplitude2, frame_start2);
		    else
			confidence2 = find_frame<G, GlobalSrc>(gsrc, pos, geo, 0, sm.tw, sm.scr, g,
				gmask, try_first, try_max, try_step, INFINITY,
				bits2, amplitude2, frame_start2);
		    if (confidence2 > confidence) {
			bits = bits2;
			amplitude = amplitude2;
			frame_start = frame_start2;
		    }
		}
		track_amplitude = (track_amplitude + amplitude) / 2.f;	/* :1391 */
		if (peak_confidence < confidence)
		    peak_confidence = confidence;
		confidence_total += confidence;			/* :1397-1400 */
		amplitude_total += amplitude;
		nframes_decoded++;
		noconfidence = 0;
		if (g == 0)
		    store_frame(out + nframes, bits, confidence, amplitude, frame_start | acquired);
		if (AUTO && g == 0 && au.rec_band)
		    au.rec_band[(size_t)s * a.max_frames + nframes] = band;
		nframes++;
		advance = frame_start + lc.frame_nsamples - lc.nsamples_overscan;	/* :1407 */
	    }
	    if (advance > remaining) { done = 1; break; }	/* :1151 */
	    pos += advance;
	    if (AUTO)
		vring = advance >= vring ? 0u : vring - advance;
	    if (MODE != 1) {
		pos_off = ring_wrap(pos_off + advance, R);	/* advance < R by construction */
		if (filled < (pos & ~AL)) {
		    /* skipped past everything requested so far: restart the ring here */
		    drain();
		    filled = pos & ~AL;
		    pos_off = pos & AL;
		    fdst = dst0;
		    fsrc = SRC ? x : x + filled + 4u * g;
		    conv = filled;
		    coff = 0;
		}
		__syncwarp(gmask);	/* every read of this window precedes the next copies */
	    }
	}
	if (MODE != 1)
	    drain();	/* before the slot is reused or the block exits */

	if (g == 0) {
	    st.pos = pos;
	    st.nframes = nframes;
	    st.carrier = carrier;
	    st.noconfidence = noconfidence;
	    st.track_amplitude = track_amplitude;
	    st.peak_confidence = peak_confidence;
	    st.carrier_nsamples = carrier_nsamples;
	    st.confidence_total = confidence_total;
	    st.amplitude_total = amplitude_total;
	    st.nframes_decoded = nframes_decoded;
	    st.done = done;
	    st.stat_candidates += ncand;
	    st.stat_searches += nsearch;
	    st.reserved = mhint ? 1u : 0u;
	    a.states[s] = st;
	    if (AUTO) {
		au.states[s].carrier_band = band;
		au.states[s].v = vring;
	    }
	}
	__syncwarp(gmask);
    }
}


/* ------------------------------------------------------------------------ */
/* full-spectrum magnitudes for fsk_detect_carrier (src/fsk.c:543-581)      */
/* ------------------------------------------------------------------------ */

__global__ void k_band_mags(const float *__restrict__ x, unsigned nsamples, int fftsize,
	unsigned nbands, float *__restrict__ mags)
{
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nbands)
	return;
    mags[k] = band_mag(x, nsamples, (unsigned)fftsize, k);
}

/* N3, batched: fsk_detect_carrier (src/fsk.c:543-581) for one stream per warp.  The lanes take
 * the bands 1, 2, ... round-robin; each keeps the first strictly largest magnitude at or above
 * the threshold among its own (ascending) bands, and the warp then keeps the largest, the
 * lowest band on a tie -- which is what the reference's single ascending scan picks. */
__global__ void k_detect_carrier(const float *__restrict__ samples, unsigned nstreams, size_t stride,
	const uint32_t *__restrict__ offset, unsigned nsamples, int fftsize, unsigned nbands,
	float min_mag_threshold, int32_t *__restrict__ out_band)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (s >= nstreams)
	return;						/* whole warps leave together */
    const float *x = samples + (size_t)s * stride + (offset ? offset[s] : 0u);
    float max_mag = 0.0f;
    int best = -1;
    for (unsigned k = 1 + lane; k < nbands; k += 32) {
	const float m = band_mag(x, nsamples, (unsigned)fftsize, k);
	if (m < min_mag_threshold)			/* :566 */
	    continue;
	if (max_mag < m) {				/* :570: strict, so the first of equals stays */
	    max_mag = m;
	    best = (int)k;
	}
    }
    for (int o = 16; o; o >>= 1) {
	const float om = __shfl_xor_sync(0xffffffffu, max_mag, o);
	const int ob = __shfl_xor_sync(0xffffffffu, best, o);
	if (ob >= 0 && (best < 0 || max_mag < om || (max_mag == om && ob < best))) {
	    max_mag = om;
	    best = ob;
	}
    }
    if (lane == 0)
	out_band[s] = best;
}

/* ------------------------------------------------------------------------ */
/* transmitter: bytes -> data words -> tones -> samples, one warp per stream */
/* (src/minimodem.c:81-250, src/simple-tone-generator.c:107-175)            */
/* ------------------------------------------------------------------------ */
/* A stream's signal is a sequence of TONES (frequency, duration): optional silence (the lead-in of
 * fsk_b200_tx_batch), leader, sync-byte preamble, the frames of the data words, the idle tone,
 * the trailer.  The warp makes them 32 at a time, lane j tone j of the batch: its duration, the
 * start sample (a warp scan of the durations) and its starting phase (the reference's serial
 * cphase chain, one add and one fractional part per tone) go into a ring of the last 64 tones in
 * shared memory.  Then the lanes write the samples up to the end of the batch, lane j the VEC
 * consecutive samples of vector j, j + 32, ... whatever tone they fall in: a bit of 40 samples
 * does not leave lanes idle, and each lane stores 16 bytes at a time when the row alignment
 * allows it.  The words come from the stream's bytes 32 at a time, encoded by the lanes side by
 * side; Baudot's charset (the only state an encoder has) is carried across the lanes by a warp
 * scan of the three-state transition maps. */

#define TX_WARPS 4			/* warps (streams) per block */
#define TX_RING 64			/* tones kept per warp: the batch being written and the one before */
#define TX_WRING 128			/* data words kept per warp */

/* fmodf(x, 1.0f) for x >= 0, exactly: the fractional part of a float is representable, so
 * x - trunc(x) is computed without rounding -- the same value the reference's fmodf returns
 * (src/simple-tone-generator.c:162-163), for a third of the instructions on the serial chain */
__device__ __forceinline__ float tx_frac(float x)
{
    return x - truncf(x);
}

/* sin(x) in double precision for 0 <= x < 2^22 (x = 2 pi turns; a tone of up to ~667 000 cycles):
 * a two-constant reduction by pi/2 with exact fma products, then the Taylor series of sin or cos
 * on |r| <= pi/4 (truncation below 1e-19).  Rounded to float it equals (float)sin((double)x) of
 * glibc on every float of that range (checked exhaustively on the CPU); unlike CUDA's sin() it
 * has no slow-path call, whose register saves spill in this kernel. */
__device__ __forceinline__ double tx_sin(float xf)
{
    const double x = (double)xf;
    const double q = rint(x * 0.63661977236758134308);
    double r = fma(-q, 0x1.921fb54442d18p0, x);
    r = fma(-q, 0x1.1a62633145c07p-54, r);
    const double z = r * r;
    const double sn = r + r * z * (-1.0 / 6 + z * (1.0 / 120 + z * (-1.0 / 5040 + z * (1.0 / 362880
	    + z * (-1.0 / 39916800 + z * (1.0 / 6227020800.0 + z * (-1.0 / 1307674368000.0
	    + z * (1.0 / 355687428096000.0))))))));
    const double cs = 1.0 + z * (-0.5 + z * (1.0 / 24 + z * (-1.0 / 720 + z * (1.0 / 40320
	    + z * (-1.0 / 3628800 + z * (1.0 / 479001600.0 + z * (-1.0 / 87178291200.0
	    + z * (1.0 / 20922789888000.0 + z * (-1.0 / 6402373705728000.0)))))))));
    const int k = (int)q & 3;
    return k == 0 ? sn : k == 1 ? cs : k == 2 ? -sn : -cs;
}

/* warp-inclusive sum */
__device__ __forceinline__ unsigned tx_scan_add(unsigned v, unsigned lane)
{
    for (unsigned o = 1; o < 32; o <<= 1) {
	const unsigned u = __shfl_sync(0xffffffffu, v, lane >= o ? lane - o : lane);
	if (lane >= o)
	    v += u;
    }
    return v;
}

/* Baudot charset transition maps: 2 bits per incoming charset (0, 1, 2) */
#define TX_MAP_ID (0u | 1u << 2 | 2u << 4)
__device__ __forceinline__ unsigned tx_map_apply(unsigned m, unsigned cs) { return (m >> (2 * cs)) & 3u; }
__device__ __forceinline__ unsigned tx_map_then(unsigned first, unsigned second)
{
    unsigned r = 0;
    for (unsigned cs = 0; cs < 3; cs++)
	r |= tx_map_apply(second, tx_map_apply(first, cs)) << (2 * cs);
    return r;
}

/* the sample at i samples into a tone (wave == 0: silence) */
template <typename T, bool LUT>
__device__ __forceinline__ T tx_sample(const fsk_b200_tx_plan &P, const T *lut, unsigned i, float wave,
	float cph)
{
    if (wave == 0.0f)
	return (T)0;
    const float turns = (float)i / wave + cph;				/* :121 */
    if constexpr (LUT) {
	int t = (int)((float)P.lut_len * turns + 0.5f);			/* :77-84, :89-96 */
	t = (P.lut_len & (P.lut_len - 1u)) ? t % (int)P.lut_len : t & (int)(P.lut_len - 1u);
	return lut[t];
    }
    /* :133-134, :151-152, with the sine in double precision for glibc's sinf (DESIGN.md 5) */
    const float s = (float)tx_sin((float)M_PI * 2 * turns);
    if constexpr (sizeof(T) == 4)
	return (T)(P.mag * s);
    else
	return (T)lroundf(P.mag_s * s);
}

template <typename T, int VEC>
__device__ __forceinline__ void tx_store(T *row, unsigned q0, unsigned end, const T (&v)[VEC])
{
    if constexpr (VEC > 1) {
	if (q0 + VEC <= end) {
	    if constexpr (sizeof(T) == 4) {
		*reinterpret_cast<float4 *>(row + q0) = make_float4(v[0], v[1], v[2], v[3]);
	    } else {
		int4 w;
		w.x = (int)((uint16_t)v[0] | (unsigned)(uint16_t)v[1] << 16);
		w.y = (int)((uint16_t)v[2] | (unsigned)(uint16_t)v[3] << 16);
		w.z = (int)((uint16_t)v[4] | (unsigned)(uint16_t)v[5] << 16);
		w.w = (int)((uint16_t)v[6] | (unsigned)(uint16_t)v[7] << 16);
		*reinterpret_cast<int4 *>(row + q0) = w;
	    }
	    return;
	}
    }
    for (int e = 0; e < VEC; e++)
	if (q0 + e < end)
	    row[q0 + e] = v[e];
}

/* samples [from, to) of the row (from a multiple of VEC): the tones [lo, hi) are in the ring,
 * tones end at sample `sig_end`, zeros follow */
template <typename T, int VEC, bool LUT>
__device__ __forceinline__ void tx_write(const fsk_b200_tx_plan &P, const T *lut, const float4 *ring,
	unsigned lo, unsigned hi, unsigned sig_end, T *row, unsigned from, unsigned to, unsigned lane)
{
    for (unsigned q0 = from + lane * VEC; q0 < to; q0 += 32 * VEC) {
	T v[VEC];
	unsigned idx = lo, next = 0xffffffffu;
	float wave = 0.0f, cph = 0.0f;
	unsigned start = 0;
	if (q0 < sig_end) {
	    unsigned a = lo, b = hi;				/* the last tone that starts at or before q0 */
	    while (b - a > 1) {
		const unsigned m = (a + b) >> 1;
		if (__float_as_uint(ring[m % TX_RING].x) <= q0)
		    a = m;
		else
		    b = m;
	    }
	    idx = a;
	    const float4 r = ring[idx % TX_RING];
	    start = __float_as_uint(r.x), wave = r.y, cph = r.z;
	    next = idx + 1 < hi ? __float_as_uint(ring[(idx + 1) % TX_RING].x) : 0xffffffffu;
	}
#pragma unroll
	for (int e = 0; e < VEC; e++) {
	    const unsigned q = q0 + e;
	    if (q >= sig_end) {
		v[e] = (T)0;
		continue;
	    }
	    while (q >= next) {					/* the next tone(s) begin inside this vector */
		idx++;
		const float4 r = ring[idx % TX_RING];
		start = __float_as_uint(r.x), wave = r.y, cph = r.z;
		next = idx + 1 < hi ? __float_as_uint(ring[(idx + 1) % TX_RING].x) : 0xffffffffu;
	    }
	    v[e] = tx_sample<T, LUT>(P, lut, q - start, wave, cph);
	}
	tx_store<T, VEC>(row, q0, to, v);
    }
}

template <typename T, int VEC, bool LUT>
__global__ void __launch_bounds__(TX_WARPS * 32, 8) k_tx_synth(const __grid_constant__ fsk_b200_tx_plan P,
	const __grid_constant__ fsk_b200_tx_io io, const T *__restrict__ lut_global, unsigned lut_in_smem)
{
    FSK_DYN_SMEM(smem);
    T *lut_s = reinterpret_cast<T *>(smem);
    const unsigned lut_bytes = lut_in_smem ? ((P.lut_len * (unsigned)sizeof(T) + 15u) & ~15u) : 0u;
    unsigned *btab = reinterpret_cast<unsigned *>(reinterpret_cast<unsigned char *>(smem) + lut_bytes);
    float4 *rings = reinterpret_cast<float4 *>(btab + 96);
    unsigned *wrings = reinterpret_cast<unsigned *>(rings + TX_WARPS * TX_RING);
    if (lut_in_smem)
	for (unsigned i = threadIdx.x; i < P.lut_len; i += blockDim.x)
	    lut_s[i] = lut_global[i];
    if (P.encoder == FSK_B200_ENCODE_BAUDOT)
	for (unsigned i = threadIdx.x; i < 96; i += blockDim.x)
	    btab[i] = fsk_enc_baudot_entry((int)i);
    __syncthreads();
    const T *lut = lut_in_smem ? lut_s : lut_global;

    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t s = (size_t)blockIdx.x * TX_WARPS + warp;
    if (s >= io.nstreams)
	return;						/* whole warps leave together */
    float4 *ring = rings + warp * TX_RING;
    unsigned *wring = wrings + warp * TX_WRING;
    T *row = reinterpret_cast<T *>(io.out) + s * io.out_stride;

    fsk_b200_tx_state st = { 0.0f, 0u, 0u, 0u };
    if (io.states)
	st = io.states[s];
    const unsigned flags = io.states ? io.flags : FSK_B200_TX_FINAL;
    const unsigned tpf = P.tones_per_frame;
    const unsigned n_in = P.encoder == FSK_B200_ENCODE_WORDS ? io.nwords
	    : io.text_len[s] < io.text_stride ? io.text_len[s] : (unsigned)io.text_stride;
    const unsigned lead = io.lead_in ? min(io.lead_in[s], io.cap) : 0u;

    /* the tone sequence, src/minimodem.c:202-237, :246-247, :60-66 */
    const unsigned nS = lead ? 1u : 0u;
    const unsigned nL = n_in && st.transmitting == 0 ? P.leader : 0u;
    const unsigned nP = n_in && st.transmitting < 2 ? P.nsync * tpf : 0u;
    const unsigned nI = !n_in && (flags & FSK_B200_TX_IDLE_IF_EMPTY) ? 1u : 0u;
    const unsigned tx_after = n_in ? 2u : nI ? 1u : st.transmitting;
    const unsigned nT = (flags & FSK_B200_TX_FINAL) && tx_after ? P.trailer : 0u;
    const unsigned d0 = nS + nL + nP;			/* the first tone of the data frames */
    const float mark_idle = P.invert_start_stop ? P.f_space : P.f_mark;

    unsigned nread = 0, nenc = 0, charset = st.baudot_charset;
    float cphase = st.cphase;
    unsigned sig_end = 0, written = 0, G = 0, nb = 0;
    const unsigned cap = io.cap;
    for (;; G += 32) {
	/* encode until the words of this batch's data tones are there */
	if (G + 31 >= d0) {
	    const unsigned w_hi = (G + 31 - d0) / tpf;
	    while (nread < n_in && nenc <= w_hi) {
		const unsigned take = min(32u, n_in - nread);
		unsigned w0 = 0, w1 = 0, cnt = 0;
		if (P.encoder == FSK_B200_ENCODE_WORDS) {
		    if (lane < take) {
			w0 = io.words[s * io.nwords + nread + lane];
			cnt = 1;
		    }
		} else {
		    const unsigned byte = lane < take ? io.text[s * io.text_stride + nread + lane] : 0u;
		    if (P.encoder == FSK_B200_ENCODE_ASCII8) {
			w0 = fsk_enc_ascii8(byte);
			cnt = lane < take ? 1u : 0u;
		    } else {
			const int c = fsk_enc_toupper((int)(int8_t)(uint8_t)byte);
			const unsigned entry = c >= 0 && c < 0x60 ? btab[c] : 0u;
			uint32_t w[2];
			unsigned map = TX_MAP_ID;
			if (lane < take) {
			    map = 0;
			    for (unsigned cs = 0; cs < 3; cs++) {
				uint32_t t = cs;
				fsk_enc_baudot_with(&t, c, entry, w);
				map |= t << (2 * cs);
			    }
			}
			unsigned incl = map;			/* charset map of bytes 0..lane */
			for (unsigned o = 1; o < 32; o <<= 1) {
			    const unsigned u = __shfl_sync(0xffffffffu, incl, lane >= o ? lane - o : lane);
			    if (lane >= o)
				incl = tx_map_then(u, incl);
			}
			const unsigned excl = __shfl_sync(0xffffffffu, incl, lane ? lane - 1 : 0);
			uint32_t cs_in = tx_map_apply(lane ? excl : TX_MAP_ID, charset);
			if (lane < take) {
			    cnt = fsk_enc_baudot_with(&cs_in, c, entry, w);
			    w0 = w[0];
			    w1 = w[1];
			}
			charset = tx_map_apply(__shfl_sync(0xffffffffu, incl, 31), charset);
		    }
		}
		const unsigned end = tx_scan_add(cnt, lane);
		const unsigned at = nenc + end - cnt;
		if (cnt > 0)
		    wring[at % TX_WRING] = w0;
		if (cnt > 1)
		    wring[(at + 1) % TX_WRING] = w1;
		nenc += __shfl_sync(0xffffffffu, end, 31);
		nread += take;
		__syncwarp();
	    }
	}
	const unsigned nD = nread == n_in ? nenc * tpf : 0xffffffffu;
	const unsigned total = nread == n_in ? d0 + nD + nI + nT : 0xffffffffu;
	if (G >= total)
	    break;
	nb = min(32u, total - G);

	/* lane j: tone G + j */
	float freq = 0.0f;
	unsigned dur = 0;
	if (lane < nb) {
	    unsigned k = G + lane;
	    if (k < nS) {
		dur = lead;					/* silence */
	    } else if ((k -= nS) < nL) {
		freq = mark_idle, dur = P.bit;			/* leader, :211-212 */
	    } else if ((k -= nL) < nP || k - nP < nD) {
		/* a frame, fsk_transmit_frame :81-112: the sync byte (LSB first, :218-221) or a data word */
		const bool sync = k < nP;
		unsigned b = (sync ? k : k - nP) % tpf;
		const unsigned word = sync ? P.sync_byte : wring[((k - nP) / tpf) % TX_WRING];
		const int msb = sync ? 0 : P.msb_first;
		if (P.has_start && b-- == 0) {
		    freq = P.invert_start_stop ? P.f_mark : P.f_space, dur = P.start;
		} else if (b < P.n_data_bits) {
		    const unsigned bit = msb ? (word >> (P.n_data_bits - b - 1)) & 1u : (word >> b) & 1u;
		    freq = bit ? P.f_mark : P.f_space, dur = P.bit;
		} else {
		    freq = P.invert_start_stop ? P.f_space : P.f_mark, dur = P.stop;
		}
	    } else if ((k -= nP + nD) < nI) {
		freq = mark_idle, dur = P.idle;			/* idle tone, :233-236 */
	    } else {
		freq = P.f_mark, dur = P.bit;			/* trailer, :65-66 */
	    }
	}
	const unsigned end = tx_scan_add(dur, lane);
	const unsigned start = sig_end + end - dur;
	sig_end += __shfl_sync(0xffffffffu, end, 31);
	/* the phase chain (src/simple-tone-generator.c:116, :162-163; a tone of frequency 0 is
	 * silence and restarts the phase, :166-169) */
	const float wave = freq != 0.0f ? (float)P.rate / freq : 0.0f;
	const float step = freq != 0.0f ? (float)dur / wave : 0.0f;
	float my_cph = 0.0f;
	for (unsigned i = 0; i < nb; i++) {
	    const float si = __shfl_sync(0xffffffffu, step, i);
	    const float wi = __shfl_sync(0xffffffffu, wave, i);
	    if (lane == i)
		my_cph = cphase;
	    cphase = wi != 0.0f ? tx_frac(cphase + si) : 0.0f;
	}
	if (lane < nb)
	    ring[(G + lane) % TX_RING] = make_float4(__uint_as_float(start), wave, my_cph, 0.0f);
	__syncwarp();
	const bool last = G + nb >= total;
	unsigned to = last ? (cap ? cap : sig_end) : sig_end / VEC * VEC;
	if (cap)
	    to = min(to, cap);
	const unsigned hi = G + nb;
	tx_write<T, VEC, LUT>(P, lut, ring, hi > TX_RING ? hi - TX_RING : 0u, hi, sig_end, row, written, to, lane);
	written = max(written, to);
	__syncwarp();
	if (last || (cap && written >= cap))
	    break;
    }
    if (cap && written < cap)				/* no tones at all: a silent row */
	tx_write<T, VEC, LUT>(P, lut, ring, 0u, 0u, 0u, row, written, cap, lane);
    if (io.states && lane == 0) {
	st.cphase = cphase;
	st.baudot_charset = charset;
	st.transmitting = flags & FSK_B200_TX_FINAL ? 0u : tx_after;	/* :71 */
	io.states[s] = st;
	io.out_len[s] = sig_end;
    }
}
/* ------------------------------------------------------------------------ */
/* N2: int16 PCM -> float32 (x / 32768, exact), 8 samples per thread        */
/* ------------------------------------------------------------------------ */
__global__ void k_s16_to_f32(const int4 *__restrict__ src, float4 *__restrict__ dst, size_t n8)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8)
	return;
    const int4 v = __ldg(src + i);
    const float k = 1.0f / 32768.0f;
    float4 a, b;
    a.x = (float)(short)(v.x & 0xffff) * k;  a.y = (float)(short)(v.x >> 16) * k;
    a.z = (float)(short)(v.y & 0xffff) * k;  a.w = (float)(short)(v.y >> 16) * k;
    b.x = (float)(short)(v.z & 0xffff) * k;  b.y = (float)(short)(v.z >> 16) * k;
    b.z = (float)(short)(v.w & 0xffff) * k;  b.w = (float)(short)(v.w >> 16) * k;
    dst[2 * i] = a;
    dst[2 * i + 1] = b;
}

/* generic tail / unaligned variant: one sample per thread */
__global__ void k_s16_to_f32_scalar(const short *__restrict__ src, float *__restrict__ dst, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
	dst[i] = (float)src[i] * (1.0f / 32768.0f);
}

/* ------------------------------------------------------------------------ */
/* live streams: between two rx launches, each stream's unconsumed tail moves to */
/* the front of its row and the new samples are appended (one warp per stream)   */
/* ------------------------------------------------------------------------ */
__global__ void k_stream_push(float *__restrict__ samples, unsigned nstreams, size_t stride,
	uint32_t *__restrict__ fill, fsk_b200_stream_state *__restrict__ states,
	const float *__restrict__ chunk, size_t chunk_stride, const uint32_t *__restrict__ chunk_len,
	uint32_t chunk_len_all, uint32_t *__restrict__ dropped)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (s >= nstreams)
	return;						/* whole warps leave together */
    float *row = samples + (size_t)s * stride;
    const unsigned have = fill[s];
    unsigned long long pos64 = states[s].pos;
    const unsigned pos = pos64 < have ? (unsigned)pos64 : have;
    const unsigned tail = have - pos;
    /* forward move in tiles of 32: a tile is read completely before it is written, and the
     * destination of tile k ends below the source of tile k+1 (dst = src - pos, pos >= 0) */
    if (pos)
	for (unsigned k = 0; k < tail; k += 32) {
	    const float v = k + lane < tail ? row[pos + k + lane] : 0.f;
	    __syncwarp();
	    if (k + lane < tail)
		row[k + lane] = v;
	    __syncwarp();
	}
    unsigned len = chunk_len ? chunk_len[s] : chunk_len_all;
    const unsigned room = (unsigned)min((size_t)0xffffffffu, stride) - tail;
    const unsigned drop = len > room ? len - room : 0u;
    len -= drop;
    const float *src = chunk + (size_t)s * chunk_stride;
    for (unsigned i = lane; i < len; i += 32)
	row[tail + i] = src[i];
    __syncwarp();		/* every lane has read fill[s] and states[s] before lane 0 rewrites them */
    if (lane == 0) {
	fill[s] = tail + len;
	states[s].pos = 0;
	states[s].nframes = 0;				/* the record buffer starts over */
	states[s].done = 0;
	if (dropped)
	    dropped[s] = drop;
    }
}

/* ------------------------------------------------------------------------ */
/* N1: frame records -> bytes through one of the reference's databits decoders  */
/* (fsk_b200_decode_core.h) behind the bit chop of src/minimodem.c:1415-1446;   */
/* one thread per stream, the decoder state of the stream in registers/local    */
/* ------------------------------------------------------------------------ */
template <int KIND>
__global__ void k_decode(unsigned shift, unsigned n_data_bits, int msb_first, int do_rx_sync,
	unsigned long long sync_byte, const fsk_b200_frame *__restrict__ frames,
	const fsk_b200_stream_state *__restrict__ states, unsigned nstreams, uint32_t max_frames,
	fsk_b200_decoder_state *__restrict__ dstates,
	uint8_t *__restrict__ out, uint32_t out_stride, uint32_t *__restrict__ out_count)
{
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nstreams)
	return;
    const unsigned nrec = min(states[s].nframes, max_frames);
    const uint32_t *rec = reinterpret_cast<const uint32_t *>(frames + (size_t)s * max_frames);
    fsk_dec_sink sink = { out + (size_t)s * out_stride, out_stride, 0u };
    /* Caller-ID collects into the stream's own state block in global memory (256 bytes per
     * stream do not belong in registers); the others carry a few words */
    fsk_b200_decoder_state local;
    fsk_b200_decoder_state *st = &local;
    if (KIND == FSK_B200_DECODE_CALLERID && dstates)
	st = dstates + s;
    else if (KIND == FSK_B200_DECODE_CALLERID) {
	local.cid_msgtype = local.cid_ndata = 0;
	for (int i = 0; i < 256; i++)
	    local.cid_buf[i] = 0;
    } else
	local.baudot_charset = dstates ? dstates[s].baudot_charset : 0u;
    for (unsigned i = 0; i < nrec; i++, rec += 5)
	fsk_dec_record(KIND, shift, n_data_bits, msb_first, do_rx_sync, sync_byte, st, rec, &sink);
    if (KIND == FSK_B200_DECODE_BAUDOT && dstates)
	dstates[s].baudot_charset = local.baudot_charset;
    out_count[s] = min(sink.n, out_stride);
}

/* ======================================================================== */
/* host side of the CUDA translation unit                                   */
/* ======================================================================== */

struct CudaEngine {
    int device;
    int sm_count;
    int smem_optin;
    /* twiddle table */
    float4 *d_tw;
    unsigned tw_cap, tw_n;
    int tw_fftsize;
    unsigned tw_bm, tw_bs;
    /* tuning (0 = automatic) */
    int lanes, wpb, ring, split;
    char last_kernel[160];	/* what the latest rx / find_frame launch ran (diagnostics) */
    int multi;			/* 1 (default): shared-segment search where the mode allows it; 0: always per candidate */
    int pfx_fill;		/* mode 3, float rows: 1 (default) TMA bulk fill, 0 cp.async fill */
    int prefix;			/* chunk-prefix table search (mode 3): -1 (default) where it pays, 0 never, 1 wherever it fits */
    float4 *d_twc;		/* mode 3: chunk-rotation table, twc_n = fftsize / gcd(4, fftsize) entries (0: not built) */
    unsigned twc_n, twc_cap;
    /* single-stream staging */
    float *d_one;
    size_t d_one_cap;
    uint32_t *d_args;		/* offset, nvalid, first, max, step, limit(as float) */
    fsk_b200_frame *d_frame;
    float *d_mags;
    size_t d_mags_cap;
    /* host-batch slabs */
    float *d_slab[2];			/* float32 copy of an int16 slab (only when the widening is a separate pass) */
    void *d_slab_in[2];			/* the slab as it came over the wire: float32 or int16 */
    size_t slab_in_bytes, slab_f32_floats;
    fsk_b200_frame *d_slab_frames[2];
    fsk_b200_stream_state *d_slab_states[2];
    size_t slab_streams, slab_stride, slab_max_frames;
    size_t slab_bytes;			/* host-buffer path: sample bytes per slab (FSK_B200_SLAB_BYTES) */
    cudaStream_t st[2];
    float2 *d_unit;			/* --auto-carrier: unit-circle table of unit_f entries (AutoArgs.unit) */
    int unit_f;
};

extern "C" unsigned long long fsk_b200_cuda_launch_count(void) { return g_launches; }

extern "C" int fsk_b200_cuda_device_ok(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
	(void)cudaGetLastError();
	return 0;
    }
    return 1;
}

extern "C" void *fsk_b200_cuda_engine_new(void)
{
    CudaEngine *ce = (CudaEngine *)calloc(1, sizeof(CudaEngine));
    if (!ce)
	return NULL;
    if (cudaGetDevice(&ce->device) != cudaSuccess
	    || cudaDeviceGetAttribute(&ce->sm_count, cudaDevAttrMultiProcessorCount, ce->device) != cudaSuccess
	    || cudaDeviceGetAttribute(&ce->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ce->device) != cudaSuccess) {
	fsk_b200_set_error("cuda engine: %s", cudaGetErrorString(cudaGetLastError()));
	free(ce);
	return NULL;
    }
    const char *e;
    if ((e = getenv("FSK_B200_LANES"))) ce->lanes = atoi(e);
    if ((e = getenv("FSK_B200_WPB"))) ce->wpb = atoi(e);
    if ((e = getenv("FSK_B200_RING"))) ce->ring = atoi(e);
    if ((e = getenv("FSK_B200_SPLIT"))) ce->split = atoi(e);
    /* shared-segment search: -1 (default) = modes with long bit periods, every coarse search through
     * the shared segments (at short periods the per-candidate kernel is used); 0 never; 1 everywhere it
     * fits, with the single-candidate fast path; 2 everywhere it fits, always */
    ce->multi = -1;
    if ((e = getenv("FSK_B200_MULTI"))) ce->multi = atoi(e);
    /* chunk-prefix table search: -1 (default) for bit periods of FSK_PREFIX_MIN_N samples and more, 0 never,
     * 1 wherever the mode fits it */
    ce->prefix = -1;
    if ((e = getenv("FSK_B200_PREFIX"))) ce->prefix = atoi(e);
    ce->pfx_fill = 1;
    if ((e = getenv("FSK_B200_PFX_FILL"))) ce->pfx_fill = atoi(e) ? 1 : 0;
#ifdef FSK_EMU
    ce->pfx_fill = 0;		/* the host emulation of the test harness does not model cp.async.bulk / mbarrier */
#endif
    /* 256 MiB of samples ON THE WIRE per slab, two slabs in flight, so that the copies keep PCIe busy
     * while the previous slab is demodulated.  int16 slabs carry the same number of bytes, i.e. twice
     * the streams: with the same stream count, the fixed cost per slab (conversion and launch) is
     * spread over half the bytes. */
    ce->slab_bytes = (size_t)256 << 20;
    if ((e = getenv("FSK_B200_SLAB_BYTES")) && atoll(e) > 0) ce->slab_bytes = (size_t)atoll(e);
    return ce;
}

/* an engine belongs to the device that was current when it was created: its buffers and the
 * caller's device pointers must live there, and launches go to the CURRENT device */
static int engine_device_check(const CudaEngine *ce, const char *what)
{
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != ce->device) {
	fsk_b200_set_error("%s: engine was created on CUDA device %d but device %d is current", what,
		ce->device, cur);
	return -EINVAL;
    }
    return 0;
}

extern "C" void fsk_b200_cuda_engine_destroy(void *p)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (!ce)
	return;
    cudaFree(ce->d_tw);
    cudaFree(ce->d_twc);
    cudaFree(ce->d_unit);
    cudaFree(ce->d_one);
    cudaFree(ce->d_args);
    cudaFree(ce->d_frame);
    cudaFree(ce->d_mags);
    for (int i = 0; i < 2; i++) {
	cudaFree(ce->d_slab[i]);
	cudaFree(ce->d_slab_in[i]);
	cudaFree(ce->d_slab_frames[i]);
	cudaFree(ce->d_slab_states[i]);
	if (ce->st[i])
	    cudaStreamDestroy(ce->st[i]);
    }
    free(ce);
}

extern "C" const char *fsk_b200_cuda_last_kernel(void *p) { return ((CudaEngine *)p)->last_kernel; }

extern "C" int fsk_b200_cuda_tune(void *p, int lanes, int wpb, int ring)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (lanes && (lanes < 4 || lanes > 32 || (lanes & (lanes - 1)))) {
	fsk_b200_set_error("lanes per stream must be 4, 8, 16 or 32");
	return -EINVAL;
    }
    if (ring && ring < 128) {
	fsk_b200_set_error("ring size must be at least 128 floats (it is rounded up to whole 128-float blocks)");
	return -EINVAL;
    }
    if (wpb < 0 || wpb > 4) {
	fsk_b200_set_error("warps per block must be 1..4");
	return -EINVAL;
    }
    ce->lanes = lanes;
    ce->wpb = wpb;
    ce->ring = ring;
    return 0;
}

#define FSK_PFX_MAX_TABLE_BYTES (16u * 1024u)
#define FSK_PFX_TABLE_EXTRA 2056u	/* rotation-table entries past one period (a lane-run of up to 512 pieces, s4 <= 4) */
#ifndef FSK_PREFIX_MIN_N
#define FSK_PREFIX_MIN_N 128u	/* shortest bit period (samples) for which mode 3 is the default: Bell103 (160) and RTTY @8 kHz
				 * (176) take it, SAME (92) and Bell202 (40) stay on the per-candidate kernel */
#endif

/* exp(-2 pi i k n / fftsize) for k = b_mark, b_space; the argument is reduced
 * exactly in integers and evaluated in double before rounding to float */
extern "C" int fsk_b200_cuda_set_table(void *p, int fftsize, unsigned b_mark, unsigned b_space,
	unsigned bit_nsamples)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (ce->d_tw && ce->tw_fftsize == fftsize && ce->tw_bm == b_mark && ce->tw_bs == b_space
	    && ce->tw_n >= bit_nsamples)
	return 0;
    if (fftsize <= 0 || bit_nsamples == 0) {
	fsk_b200_set_error("set_table: bad size");
	return -EINVAL;
    }
    float4 *h = (float4 *)malloc(sizeof(float4) * bit_nsamples);
    if (!h)
	return -ENOMEM;
    const unsigned long long F = (unsigned long long)fftsize;
    for (unsigned n = 0; n < bit_nsamples; n++) {
	const double am = 2.0 * M_PI * (double)(((unsigned long long)b_mark * n) % F) / (double)F;
	const double as = 2.0 * M_PI * (double)(((unsigned long long)b_space * n) % F) / (double)F;
	h[n].x = (float)cos(am);
	h[n].y = (float)-sin(am);
	h[n].z = (float)cos(as);
	h[n].w = (float)-sin(as);
    }
    if (ce->tw_cap < bit_nsamples) {
	cudaFree(ce->d_tw);
	ce->d_tw = NULL;
	ce->tw_cap = 0;
	if (cudaMalloc(&ce->d_tw, sizeof(float4) * bit_nsamples) != cudaSuccess) {
	    fsk_b200_set_error("set_table: %s", cudaGetErrorString(cudaGetLastError()));
	    free(h);
	    return -ENOMEM;
	}
	ce->tw_cap = bit_nsamples;
    }
    /* synchronous copy from pageable memory, then a device-wide synchronise: the library's own
     * streams and the caller's may be cudaStreamNonBlocking, which the legacy stream does not order */
    cudaError_t err = cudaMemcpy(ce->d_tw, h, sizeof(float4) * bit_nsamples, cudaMemcpyHostToDevice);
    if (err == cudaSuccess)
	err = cudaDeviceSynchronize();
    free(h);
    if (err != cudaSuccess) {
	fsk_b200_set_error("set_table: %s", cudaGetErrorString(err));
	return -EIO;
    }
    ce->tw_n = bit_nsamples;
    ce->tw_fftsize = fftsize;
    ce->tw_bm = b_mark;
    ce->tw_bs = b_space;
    /* mode 3: the phase of chunk m (4 samples) relative to chunk 0 is b * 4m / fftsize turns; 4m mod fftsize
     * only takes multiples of gcd(4, fftsize), so the table has fftsize / gcd entries, entry e for the
     * sample index e * gcd.  Kept only while it is small enough to be staged per block. */
    ce->twc_n = 0;
    {
	const unsigned g4 = (fftsize % 4 == 0) ? 4u : (fftsize % 2 == 0) ? 2u : 1u;
	const unsigned fp = (unsigned)fftsize / g4;
	if ((size_t)fp * sizeof(float4) <= FSK_PFX_MAX_TABLE_BYTES) {
	    /* (FSK_PFX_TABLE_EXTRA entries more than one period: a lane-run of the table build walks it
	     * linearly from anywhere inside the period) */
	    const unsigned fp1 = fp, fpx = fp + FSK_PFX_TABLE_EXTRA;
	    float4 *hc = (float4 *)malloc(sizeof(float4) * fpx);
	    if (!hc)
		return -ENOMEM;
	    for (unsigned i = 0; i < fpx; i++) {
		const unsigned long long n = (unsigned long long)(i % fp1) * g4;
		const double am = 2.0 * M_PI * (double)(((unsigned long long)b_mark * n) % F) / (double)F;
		const double as = 2.0 * M_PI * (double)(((unsigned long long)b_space * n) % F) / (double)F;
		hc[i].x = (float)cos(am);
		hc[i].y = (float)-sin(am);
		hc[i].z = (float)cos(as);
		hc[i].w = (float)-sin(as);
	    }
	    if (ce->twc_cap < fpx) {
		cudaFree(ce->d_twc);
		ce->d_twc = NULL;
		ce->twc_cap = 0;
		if (cudaMalloc(&ce->d_twc, sizeof(float4) * fpx) != cudaSuccess) {
		    (void)cudaGetLastError();
		    free(hc);
		    return 0;			/* mode 3 is simply not offered */
		}
		ce->twc_cap = fpx;
	    }
	    cudaError_t err2 = cudaMemcpy(ce->d_twc, hc, sizeof(float4) * fpx, cudaMemcpyHostToDevice);
	    if (err2 == cudaSuccess)
		err2 = cudaDeviceSynchronize();
	    free(hc);
	    if (err2 != cudaSuccess) {
		fsk_b200_set_error("set_table: %s", cudaGetErrorString(err2));
		return -EIO;
	    }
	    ce->twc_n = fp;
	}
    }
    return 0;
}

/* launch shape shared by K1 and K2 */
struct Shape {
    int G, W, L, mode, wpb, blocks;
    unsigned ring, tw_in_smem, lookahead;
    size_t smem;
    fsk_b200_geom geo;
    fsk_b200_mplan mplan;	/* mode 2 */
    fsk_b200_pfx pfx;		/* mode 3 */
    unsigned pfx_tw_stage;	/* mode 3: rotation-table entries staged per block */
    unsigned slide;		/* mode 0: fine searches by sliding (extended twiddle table staged) */
};

/* (G, W, L) combinations that are instantiated for the fast path: G lanes per
 * stream, L lanes per bit window, W windows per lane (W * G/L >= n_bits) */
#define FAST_COMBOS(X) \
    X(4, 1, 1) X(4, 2, 1) X(4, 3, 1) X(4, 4, 1) X(4, 2, 2) X(4, 4, 2) \
    X(8, 1, 1) X(8, 2, 1) X(8, 3, 1) X(8, 4, 1) X(8, 1, 2) X(8, 2, 2) X(8, 3, 2) X(8, 4, 2) X(8, 4, 4) \
    X(16, 1, 1) X(16, 2, 1) X(16, 3, 1) X(16, 4, 1) X(16, 1, 2) X(16, 2, 2) X(16, 3, 2) X(16, 4, 2) \
    X(16, 1, 4) X(16, 2, 4) X(16, 3, 4) X(16, 4, 4) \
    X(32, 1, 1) X(32, 2, 1) X(32, 1, 2) X(32, 2, 2) X(32, 3, 2) X(32, 4, 2) X(32, 1, 4) X(32, 2, 4) X(32, 3, 4) X(32, 4, 4)

#ifndef FSK_MULTI_MIN_N
#define FSK_MULTI_MIN_N 96u	/* shortest bit period (samples) for which mode 2 is the default */
#endif
/* (G, W, L) of the shared-segment rx kernel (mode 2): W * G/L period slots >= n_bits + 1 */
#define MULTI_COMBOS(X) \
    X(8, 2, 2) X(8, 3, 2) X(8, 4, 2) X(16, 2, 2) X(16, 3, 2) X(16, 4, 2) X(16, 2, 4) X(16, 3, 4) X(16, 4, 4) \
    X(32, 2, 4) X(32, 3, 4) X(32, 4, 4)

/* mode 3: the W of k_rx<32, W, 1, 3> codes the candidate slot: 1 = packed slots of nbnd lanes, 3 / 4 / 5 = aligned
 * slots of 8 / 16 / 32 lanes */
#define PFX_SLOTS(X) X(1) X(3) X(4) X(5)

/* per-candidate shapes that are also built for int16 rows (SRC 1); every MULTI_COMBOS shape is */
#define S16_FAST_COMBOS(X) \
    X(8, 1, 1) X(8, 2, 1) X(8, 3, 1) X(8, 2, 2) X(8, 3, 2) X(8, 4, 2) X(8, 4, 4) \
    X(16, 1, 2) X(16, 2, 2) X(16, 2, 4) X(16, 3, 4) X(16, 4, 4) X(32, 2, 4)

static bool fast_combo(int G, int W, int L)
{
#define X(GG, WW, LL) if (G == GG && W == WW && L == LL) return true;
    FAST_COMBOS(X)
#undef X
    return false;
}

/* mode 2: the (W, L) of MULTI_COMBOS with the fewest idle period slots for `periods` bit periods */
static bool split_for_multi(int G, unsigned periods, int *W, int *L)
{
    unsigned best = ~0u;
#define X(GG, WW, LL) if (G == GG && (unsigned)(WW * (GG / LL)) >= periods && (unsigned)(WW * (GG / LL)) <= best) { \
	best = (unsigned)(WW * (GG / LL)); *W = WW; *L = LL; }
    MULTI_COMBOS(X)
#undef X
    return best != ~0u;
}

/* best (W, L) for a group of G lanes: highest lane utilisation n_bits / (W * G/L);
 * ties go to the larger L (neighbouring lanes then read neighbouring samples, which
 * spreads the shared-memory banks) */
static bool split_for(int G, unsigned n_bits, int force_L, int *W, int *L)
{
    double best = -1.0;
    for (int l = 1; l <= 4 && l <= G; l *= 2) {
	if (force_L && l != force_L)
	    continue;
	const unsigned wpp = (unsigned)(G / l);
	const unsigned w = (n_bits + wpp - 1) / wpp;
	if (w > 4 || !fast_combo(G, (int)w, l))
	    continue;
	const double util = (double)n_bits / (double)(w * wpp);
	if (util >= best - 1e-9) {
	    best = util;
	    *W = (int)w;
	    *L = l;
	}
    }
    return best > 0.0;
}

/* per_stream_tw (--auto-carrier): the per-candidate kernel only, with a tone table per stream instead of
 * one per block */
static int pick_shape(const CudaEngine *ce, const fsk_b200_geom *g, unsigned need_floats,
	unsigned max_advance, size_t nstreams, Shape *sh, const fsk_b200_loopc *lc = NULL, bool per_stream_tw = false)
{
    sh->geo = *g;
    memset(&sh->mplan, 0, sizeof(sh->mplan));
    const size_t smem_max = (size_t)ce->smem_optin;
    const size_t tw_bytes = (size_t)g->bit_nsamples * sizeof(float4);	/* the sliding search's extension is added at the end */
    sh->tw_in_smem = tw_bytes <= 24 * 1024;
    const size_t fixed = sh->tw_in_smem && !per_stream_tw ? tw_bytes : 0;
    const size_t pad_bytes = (size_t)((g->bit_nsamples + 3u) & ~3u) * 4;
    /* per stream, besides the ring: scratch, mirror, 2 mbarriers (and its tone table) */
    const size_t scr_bytes = (size_t)g->n_bits * sizeof(float2) + pad_bytes + 16 + (per_stream_tw ? tw_bytes : 0);

    /* ring: the widest search window plus (ideally) one full advance of look-ahead */
    /* whole blocks; room for the widest window starting anywhere inside a block */
    const unsigned ring_min = (need_floats + 8u + 2u * RING_BLOCK - 1u) / RING_BLOCK * RING_BLOCK;
    (void)max_advance;
    /* default: the minimum, which already leaves 1..2 blocks of look-ahead; a deeper ring means
     * fewer resident streams */
    unsigned ring = ce->ring ? ((unsigned)ce->ring + RING_BLOCK - 1u) / RING_BLOCK * RING_BLOCK : ring_min;
    if (ring < ring_min)
	ring = ring_min;
    /* keep at least ~24 streams per SM resident if that is possible at all */
    if (!ce->ring) {
	while (ring > ring_min && (smem_max - fixed) / ((size_t)ring * 4 + scr_bytes) < 24)
	    ring -= RING_BLOCK;
    }

    int G = ce->lanes;
    if (!G) {
	const size_t per_stream = (size_t)ring * 4 + scr_bytes;
	size_t streams_per_sm = (smem_max > fixed ? smem_max - fixed : 0) / (per_stream ? per_stream : 1);
	if (streams_per_sm < 1)
	    streams_per_sm = 1;
	G = 8;
	while (G < 32 && streams_per_sm * (size_t)G < 256)
	    G <<= 1;
    }
    int W = 1, L = 1;
    bool fast = split_for(G, g->n_bits, ce->split, &W, &L);
    while (!fast && G < 32) {			/* e.g. 47-bit frames need G >= 16 */
	G <<= 1;
	fast = split_for(G, g->n_bits, ce->split, &W, &L);
    }
    if (g->bit_nsamples > FAST_MAX_N * (unsigned)L || !sh->tw_in_smem)
	fast = false;

    int wpb = ce->wpb ? ce->wpb : 2;
    for (;;) {
	const size_t spw = 32 / G;
	const size_t smem = (fixed + (size_t)wpb * spw * ((size_t)ring * 4 + scr_bytes) + 15) & ~(size_t)15;
	if (smem <= smem_max) {
	    sh->smem = smem;
	    break;
	}
	if (wpb > 1) { wpb--; continue; }
	if (G < 32) {
	    G <<= 1;
	    fast = split_for(G, g->n_bits, ce->split, &W, &L) && g->bit_nsamples <= FAST_MAX_N * (unsigned)L && sh->tw_in_smem;
	    continue;
	}
	if (ring) { ring = 0; fast = false; continue; }	/* not even one ring fits: read global memory */
	sh->tw_in_smem = 0;
	sh->smem = ((size_t)g->n_bits * sizeof(float2) + 16 + 15) & ~(size_t)15;
	break;
    }
    if (!fast) {
	/* generic kernels are instantiated for G = 32 only and do not use a ring */
	G = 32;
	ring = 0;
	L = 1;
	while ((unsigned)(L * 2) * g->n_bits <= 32u)
	    L *= 2;
	W = (int)((g->n_bits + 32 / L - 1) / (32 / L));
	const size_t fixed2 = sh->tw_in_smem ? tw_bytes : 0;
	const size_t scr_only = (size_t)g->n_bits * sizeof(float2) + 16;
	wpb = ce->wpb ? ce->wpb : 4;
	sh->smem = (fixed2 + (size_t)wpb * scr_only + 15) & ~(size_t)15;
	if (sh->smem > smem_max) {
	    sh->tw_in_smem = 0;
	    sh->smem = ((size_t)wpb * scr_only + 15) & ~(size_t)15;
	}
    }
    sh->mode = fast ? 0 : 1;
    if (fast && lc && !per_stream_tw && ce->multi && (ce->multi > 0 || g->bit_nsamples >= FSK_MULTI_MIN_N)) {
	/* the rx loop's searches from shared segment sums, if this mode's windows tile and all of its
	 * searches fit the period slots of a (W, L) split of this group size */
	int W2 = 0, L2 = 0;
	if (split_for_multi(G, g->n_bits + 1u, &W2, &L2) && g->bit_nsamples <= FAST_MAX_N * (unsigned)L2
		&& fsk_b200_mplan_build(g, lc, (unsigned)(W2 * (G / L2)), &sh->mplan) == 0) {
	    sh->mode = 2;
	    sh->mplan.always = ce->multi >= 2 || ce->multi < 0;
	    W = W2;
	    L = L2;
	}
    }
    memset(&sh->pfx, 0, sizeof(sh->pfx));
    if (lc && !per_stream_tw && ce->prefix && ce->twc_n && ring_min >= 128u
	    && (ce->prefix > 0 || g->bit_nsamples >= FSK_PREFIX_MIN_N)) {
	/* the rx loop's searches from a chunk-prefix table (mode 3): one stream per warp, one lane per
	 * window boundary of a candidate, the ring without its mirror plus the table per stream */
	fsk_b200_pfx &pf = sh->pfx;
	const unsigned nb = g->n_bits, N = g->bit_nsamples;
	pf.tiles = 1;
	for (unsigned w = 0; w + 1 < nb; w++)
	    if (g->bit_begin[w + 1] != g->bit_begin[w] + N)
		pf.tiles = 0;
	pf.nbnd = pf.tiles ? nb + 1u : 2u * nb;
	/* candidate slots: aligned power-of-two slots reduce by butterflies; slots of exactly nbnd lanes packed
	 * back to back are used only where they hold more candidates per round (9 boundaries: 3 instead of 2) */
	unsigned bs2 = 8;
	int lb = 3;
	while (bs2 < pf.nbnd) {
	    bs2 <<= 1;
	    lb++;
	}
	if (pf.nbnd <= 32u && 32u / bs2 == 32u / pf.nbnd) {
	    pf.bs = bs2;
	    pf.pow2 = 1;
	} else {
	    pf.bs = pf.nbnd;
	    pf.pow2 = 0;
	    lb = 1;			/* the kernel's template code for packed slots */
	}
	pf.cpr = pf.bs ? 32u / pf.bs : 0u;
	/* 16-byte pieces of the widest search span (it may start up to 3 samples into its first piece), dealt
	 * to the 32 lanes in runs of S pieces.  S odd: the lanes walk their runs in step, S pieces apart, and
	 * only an odd stride spreads a quarter-warp's 16-byte accesses over all banks; the same for the table
	 * rows (tstride) */
	const unsigned npieces = (3u + need_floats) / 4u + 1u;
	pf.S = ((npieces + 31u) / 32u) | 1u;
	pf.inv_S = 1.0f / (float)pf.S;
	pf.tstride = ((pf.S + 1u) / 2u) | 1u;
	const unsigned F = (unsigned)ce->tw_fftsize;
	const unsigned g4 = (F % 4u == 0) ? 4u : (F % 2u == 0) ? 2u : 1u;
	pf.fp = F / g4;
	pf.s4 = 4u / g4;
	pf.inv_fp = 1.0f / (float)pf.fp;
	for (unsigned j = 0; j <= 7; j++) {
	    const double am = 2.0 * M_PI * (double)(((unsigned long long)ce->tw_bm * j) % F) / (double)F;
	    const double as = 2.0 * M_PI * (double)(((unsigned long long)ce->tw_bs * j) % F) / (double)F;
	    pf.loc[j >> 1][0][j & 1u] = j ? (float)cos(am) : 1.0f;
	    pf.loc[j >> 1][1][j & 1u] = j ? (float)-sin(am) : 0.0f;
	    pf.loc[j >> 1][2][j & 1u] = j ? (float)cos(as) : 1.0f;
	    pf.loc[j >> 1][3][j & 1u] = j ? (float)-sin(as) : 0.0f;
	}
	for (unsigned k = 0; k < 4; k++) {		/* the rx loop's four searches, src/minimodem.c:1236-1263, :1357-1368 */
	    const unsigned carrier = k & 1u, fine = k >> 1;
	    const unsigned tmax_k = carrier ? lc->try_max_carrier : lc->try_max_nocarrier;
	    const unsigned first = carrier ? lc->nsamples_overscan : 0u;
	    unsigned step = tmax_k / (fine ? 8u : 3u);
	    if (step == 0)
		step = 1;
	    fsk_b200_pfx_kind &kd = pf.kind[k];
	    kd.step = step;
	    kd.k_up = tmax_k > first ? (tmax_k - 1u - first) / step : 0u;
	    kd.k_dn = first / step < kd.k_up ? first / step : kd.k_up;
	    kd.ncands = tmax_k > first ? 1u + kd.k_up + kd.k_dn : 0u;
	}
	const unsigned ring3 = ce->ring ? ring : ring_min;
	const unsigned tw_stage = pf.fp + (pf.S + 2u) * pf.s4;	/* one period and a lane-run */
	const size_t table = (size_t)tw_stage * sizeof(float4);
	const size_t per_stream = ((size_t)ring3 + 4u * pf.S + 8u) * 4 + (size_t)nb * sizeof(float2) + 16
	    + (32u * (size_t)pf.tstride + 32u + (pf.pow2 ? 0u : 32u)) * sizeof(float4);	/* ring + mirror, scratch, barriers, table + totals (+ slot-sum scratch) */
	/* warps (= streams) per block: the most resident streams per SM (each block pays the table and 1 KiB) */
	const size_t sm_total = (size_t)ce->smem_optin + 1024;
	int best_wpb = 0;
	size_t best_streams = 0;
	for (int w = 1; w <= FSK_PFX_MAXTHREADS / 32; w++) {
	    const size_t blk = ((table + (size_t)w * per_stream + 16 + 128 + 15) & ~(size_t)15);
	    if (blk > smem_max)
		break;
	    size_t nblk = sm_total / (blk + 1024);
	    if (nblk > 32)
		nblk = 32;
	    size_t streams = nblk * (size_t)w;
	    if (streams > 64)
		streams = 64;
	    if (streams > best_streams) {
		best_streams = streams;
		best_wpb = w;
	    }
	}
	if (ce->wpb && ce->prefix > 0) {
	    const size_t blk = ((table + (size_t)ce->wpb * per_stream + 16 + 128 + 15) & ~(size_t)15);
	    if (blk <= smem_max)
		best_wpb = ce->wpb;
	}
	if (pf.nbnd <= 32u && best_wpb > 0 && pf.S <= 512u && g->bit_nsamples <= ring3 && ce->twc_n) {
	    sh->mode = 3;
	    G = 32;
	    W = lb;
	    L = 1;
	    sh->pfx_tw_stage = tw_stage;
	    wpb = best_wpb;
	    ring = ring3;
	    sh->tw_in_smem = 1;
	    sh->smem = ((table + (size_t)wpb * per_stream + 16 + 128 + 15) & ~(size_t)15);
	}
    }
    /* the table as staged: the window-relative entries, or (per-candidate kernel with the sliding fine
     * search) the absolute-index extension the host layer prepared, if it still fits */
    sh->geo.tw_entries = sh->mode == 3 ? sh->pfx_tw_stage : g->bit_nsamples;
    sh->slide = 0;
    if (sh->mode == 0 && lc && lc->slide && g->tw_entries > g->bit_nsamples && sh->tw_in_smem) {
	const size_t extra = (size_t)(g->tw_entries - g->bit_nsamples) * sizeof(float4)
	    * (per_stream_tw ? (size_t)wpb * (32 / G) : 1u);
	if (sh->smem + extra <= smem_max) {
	    sh->smem += extra;
	    sh->geo.tw_entries = g->tw_entries;
	    sh->slide = 1;
	}
    }
    sh->G = G;
    sh->W = W;
    sh->L = L;
    sh->wpb = wpb;
    sh->ring = ring;
    {
	const unsigned base_need = need_floats + 8u + RING_BLOCK;
	const unsigned slack = ring > base_need ? ring - base_need : 0u;
	sh->lookahead = slack < max_advance ? slack : max_advance;
    }
    sh->geo.lanes_per_window = (unsigned)L;
    /* one block per wpb*(32/G) streams: the hardware block scheduler hands out
     * streams as SM resources free up (streams differ in length and work) */
    const size_t streams_per_block = (size_t)wpb * (32 / G);
    size_t blocks = (nstreams + streams_per_block - 1) / streams_per_block;
    if (blocks > 0x7fffffff)
	blocks = 0x7fffffff;
    sh->blocks = (int)(blocks ? blocks : 1);
    return 0;
}

template <int G, int W, int L, int MODE>
static cudaError_t launch_find_t(const Shape &sh, const CudaEngine *ce, const FindArgs &a, cudaStream_t st)
{
    cudaError_t e = cudaFuncSetAttribute(k_find_frame<G, W, L, MODE>,
	    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh.smem);
    if (e != cudaSuccess)
	return e;
    FSK_LAUNCH((k_find_frame<G, W, L, MODE>), sh.blocks, sh.wpb * 32, sh.smem, st, sh.geo, ce->d_tw,
	    sh.tw_in_smem, sh.ring, a);
    g_launches++;
    return cudaGetLastError();
}

extern "C" int fsk_b200_cuda_find_frame_batch(void *p, const fsk_b200_geom *g, const float *samples,
	size_t nstreams, size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel, fsk_b200_frame *frames, float *bit_mags, void *stream)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (!ce->d_tw || ce->tw_n < g->tw_entries) {
	fsk_b200_set_error("find_frame_batch: twiddle table not set");
	return -EINVAL;
    }
    if (engine_device_check(ce, "find_frame_batch"))
	return -EINVAL;
    Shape sh;
    /* the ring is sized for the widest search of the rx loop: 1.5 bits + span */
    pick_shape(ce, g, g->span + 2u * g->bit_nsamples + 8u, 0, nstreams, &sh);
    const FindArgs a = { samples, (unsigned)nstreams, stride, offset, nvalid, try_first, try_max,
	try_step, limit, expect_sel, frames, reinterpret_cast<float2 *>(bit_mags) };
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaErrorInvalidValue;
    if (sh.mode == 0) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) e = launch_find_t<GG, WW, LL, 0>(sh, ce, a, st);
	FAST_COMBOS(X)
#undef X
    } else {
	e = launch_find_t<32, 1, 1, 1>(sh, ce, a, st);
    }
    snprintf(ce->last_kernel, sizeof(ce->last_kernel),
	    "k_find_frame<G=%d,W=%d,L=%d,mode=%d(%s)> threads=%d ring=%u smem=%zu blocks=%d", sh.G, sh.W, sh.L, sh.mode,
	    sh.mode == 0 ? "per-candidate" : "generic", sh.wpb * 32, sh.ring, sh.smem, sh.blocks);
    if (e != cudaSuccess) {
	fsk_b200_set_error("find_frame_batch launch (G=%d W=%d L=%d mode=%d smem=%zu): %s", sh.G, sh.W,
		sh.L, sh.mode, sh.smem, cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

template <int G, int W, int L, int MODE, int FILL, int SRC = 0, int AUTO = 0>
static cudaError_t launch_rx_t(const Shape &sh, const CudaEngine *ce, const fsk_b200_loopc *lc,
	const RxArgs &a, cudaStream_t st, const AutoArgs &au = AutoArgs())
{
    cudaError_t e = cudaFuncSetAttribute(k_rx<G, W, L, MODE, FILL, SRC, AUTO>,
	    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh.smem);
    if (e != cudaSuccess)
	return e;
    /* AUTO: no block-wide table is staged (tw_in_smem 0); every stream fills its own */
    FSK_LAUNCH((k_rx<G, W, L, MODE, FILL, SRC, AUTO>), sh.blocks, sh.wpb * 32, sh.smem, st, sh.geo, *lc,
	    MODE == 3 ? ce->d_twc : ce->d_tw, AUTO ? 0u : sh.tw_in_smem, sh.ring, sh.lookahead, a, sh.mplan, ce->d_tw, sh.pfx,
	    au);
    g_launches++;
    return cudaGetLastError();
}

/* elem 4: float32 rows; elem 2: int16 PCM rows, widened inside the kernel's ring fill.  -ENOTSUP when
 * the launch shape of this mode has no int16 build (the caller widens with fsk_b200_cuda_s16_to_f32). */
static int rx_batch_any(CudaEngine *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const void *samples, int elem, size_t nstreams, size_t stride, const uint32_t *nsamples,
	uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream)
{
    if (!ce->d_tw || ce->tw_n < g->tw_entries) {
	fsk_b200_set_error("rx_batch: twiddle table not set");
	return -EINVAL;
    }
    if (engine_device_check(ce, "rx_batch"))
	return -EINVAL;
    Shape sh;
    const unsigned tmax = lc->try_max_nocarrier > lc->try_max_carrier
	? lc->try_max_nocarrier : lc->try_max_carrier;
    const unsigned max_advance = tmax - 1u + lc->frame_nsamples;	/* :1407, overscan >= 0 */
    pick_shape(ce, g, tmax - 1u + g->span, max_advance, nstreams, &sh, lc);
    fsk_b200_loopc lc_launch = *lc;
    lc_launch.slide = sh.slide;
    lc = &lc_launch;
    const RxArgs a = { elem == 4 ? (const float *)samples : NULL, elem == 2 ? (const int16_t *)samples : NULL,
	(unsigned)nstreams, stride, nsamples, nsamples_all, frames, max_frames, states };
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaErrorInvalidValue;
    bool launched = false;
    if (elem == 2) {
	if (sh.mode == 3) {
#define X(WW) if (sh.W == WW) { e = launch_rx_t<32, WW, 1, 3, 0, 1>(sh, ce, lc, a, st); launched = true; }
	    PFX_SLOTS(X)
#undef X
	} else if (sh.mode == 2) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) { e = launch_rx_t<GG, WW, LL, 2, 0, 1>(sh, ce, lc, a, st); launched = true; }
	    MULTI_COMBOS(X)
#undef X
	} else if (sh.mode == 0) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) { e = launch_rx_t<GG, WW, LL, 0, 0, 1>(sh, ce, lc, a, st); launched = true; }
	    S16_FAST_COMBOS(X)
#undef X
	} else {
	    e = launch_rx_t<32, 1, 1, 1, 0, 1>(sh, ce, lc, a, st);
	    launched = true;
	}
	if (!launched)
	    return -ENOTSUP;
    } else if (sh.mode == 3) {
	/* one stream per warp: the ring is filled by bulk copies of the TMA engine (one elected lane, two to
	 * four copies per iteration) unless FSK_B200_PFX_FILL=0 asks for the per-lane cp.async fill */
	if (ce->pfx_fill) {
#define X(WW) if (sh.W == WW) e = launch_rx_t<32, WW, 1, 3, 1>(sh, ce, lc, a, st);
	    PFX_SLOTS(X)
#undef X
	} else {
#define X(WW) if (sh.W == WW) e = launch_rx_t<32, WW, 1, 3, 0>(sh, ce, lc, a, st);
	    PFX_SLOTS(X)
#undef X
	}
    } else if (sh.mode == 2) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) e = launch_rx_t<GG, WW, LL, 2, 0>(sh, ce, lc, a, st);
	MULTI_COMBOS(X)
#undef X
    } else if (sh.mode == 0) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) e = launch_rx_t<GG, WW, LL, 0, 0>(sh, ce, lc, a, st);
	FAST_COMBOS(X)
#undef X
    } else {
	e = launch_rx_t<32, 1, 1, 1, 0>(sh, ce, lc, a, st);
    }
    snprintf(ce->last_kernel, sizeof(ce->last_kernel),
	    "k_rx<G=%d,W=%d,L=%d,mode=%d(%s),fill=%d,src=%s> threads=%d ring=%u smem=%zu blocks=%d", sh.G, sh.W, sh.L,
	    sh.mode, sh.mode == 3 ? "prefix-table" : sh.mode == 2 ? "shared-segment" : sh.mode == 0 ? "per-candidate" : "generic",
	    (sh.mode == 3 && elem == 4) ? ce->pfx_fill : 0, elem == 2 ? (sh.slide ? "s16,slide" : "s16") : (sh.slide ? "f32,slide" : "f32"),
	    sh.wpb * 32, sh.ring, sh.smem, sh.blocks);
    if (e != cudaSuccess) {
	fsk_b200_set_error("rx_batch launch (G=%d W=%d L=%d mode=%d ring=%u smem=%zu): %s", sh.G, sh.W,
		sh.L, sh.mode, sh.ring, sh.smem, cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

extern "C" int fsk_b200_cuda_rx_batch(void *p, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const float *samples, size_t nstreams, size_t stride, const uint32_t *nsamples,
	uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream)
{
    return rx_batch_any((CudaEngine *)p, g, lc, samples, 4, nstreams, stride, nsamples, nsamples_all, frames,
	    max_frames, states, stream);
}

extern "C" int fsk_b200_cuda_rx_batch_s16(void *p, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const int16_t *samples, size_t nstreams, size_t stride, const uint32_t *nsamples,
	uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream)
{
    return rx_batch_any((CudaEngine *)p, g, lc, samples, 2, nstreams, stride, nsamples, nsamples_all, frames,
	    max_frames, states, stream);
}

/* --auto-carrier: the shapes of the per-candidate kernel with a tone table per stream (AUTO 1), in float
 * and int16 builds -- what pick_shape chooses for the presets of fsk_b200_rx_config_for_mode at 8 and 48 kHz */
#define AUTO_COMBOS(X) \
    X(8, 3, 2) X(16, 2, 4) X(16, 3, 4) X(16, 3, 1) X(32, 1, 4) X(32, 2, 4) X(32, 3, 2)

/* (cos, -sin)(2 pi r / fftsize): the expression of fsk_b200_cuda_set_table with r = (b * n) mod fftsize, so
 * every per-stream table entry is bit-identical to the one a fixed-tone engine builds */
extern "C" int fsk_b200_cuda_set_unit_table(void *p, int fftsize)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (ce->d_unit && ce->unit_f == fftsize)
	return 0;
    if (fftsize <= 0)
	return -EINVAL;
    float2 *h = (float2 *)malloc(sizeof(float2) * (size_t)fftsize);
    if (!h)
	return -ENOMEM;
    const double F = (double)fftsize;
    for (int r = 0; r < fftsize; r++) {
	const double a = 2.0 * M_PI * (double)r / F;
	h[r].x = (float)cos(a);
	h[r].y = (float)-sin(a);
    }
    cudaFree(ce->d_unit);
    ce->d_unit = NULL;
    ce->unit_f = 0;
    cudaError_t err = cudaMalloc(&ce->d_unit, sizeof(float2) * (size_t)fftsize);
    if (err == cudaSuccess)
	err = cudaMemcpy(ce->d_unit, h, sizeof(float2) * (size_t)fftsize, cudaMemcpyHostToDevice);
    if (err == cudaSuccess)
	err = cudaDeviceSynchronize();
    free(h);
    if (err != cudaSuccess) {
	fsk_b200_set_error("set_unit_table: %s", cudaGetErrorString(err));
	return -EIO;
    }
    ce->unit_f = fftsize;
    return 0;
}

/* elem 4: float32 rows, elem 2: int16 rows.  -ENOTSUP (nothing launched) where the per-candidate kernel
 * cannot take the mode or the shape has no auto build. */
extern "C" int fsk_b200_cuda_rx_batch_auto(void *p, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const fsk_b200_auto_args *aa, const void *samples, int elem, size_t nstreams, size_t stride,
	const uint32_t *nsamples, uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, fsk_b200_auto_state *auto_states, uint32_t *rec_band, void *stream)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (!ce->d_unit || ce->unit_f != aa->fftsize) {
	fsk_b200_set_error("rx_batch_auto: auto-carrier not set");
	return -EINVAL;
    }
    if (engine_device_check(ce, "rx_batch_auto"))
	return -EINVAL;
    Shape sh;
    const unsigned tmax = lc->try_max_nocarrier > lc->try_max_carrier ? lc->try_max_nocarrier : lc->try_max_carrier;
    const unsigned max_advance = tmax - 1u + lc->frame_nsamples;
    pick_shape(ce, g, tmax - 1u + g->span, max_advance, nstreams, &sh, lc, true);
    fsk_b200_loopc lc_launch = *lc;
    lc_launch.slide = sh.slide;
    bool launched = false;
    cudaError_t e = cudaErrorInvalidValue;
    if (sh.mode == 0) {
	const RxArgs a = { elem == 4 ? (const float *)samples : NULL, elem == 2 ? (const int16_t *)samples : NULL,
	    (unsigned)nstreams, stride, nsamples, nsamples_all, frames, max_frames, states };
	const AutoArgs au = { auto_states, rec_band, ce->d_unit, aa->threshold, aa->scan_n, aa->b_shift,
	    (unsigned)aa->fftsize, aa->nbands, aa->half_ring, aa->expect_nsamples };
	cudaStream_t st = (cudaStream_t)stream;
	if (elem == 2) {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) { e = launch_rx_t<GG, WW, LL, 0, 0, 1, 1>(sh, ce, &lc_launch, a, st, au); launched = true; }
	    AUTO_COMBOS(X)
#undef X
	} else {
#define X(GG, WW, LL) if (sh.G == GG && sh.W == WW && sh.L == LL) { e = launch_rx_t<GG, WW, LL, 0, 0, 0, 1>(sh, ce, &lc_launch, a, st, au); launched = true; }
	    AUTO_COMBOS(X)
#undef X
	}
    }
    if (!launched) {
	fsk_b200_set_error("rx_batch_auto: no auto-carrier build of the per-candidate kernel for this mode "
		"(launch shape G=%d W=%d L=%d mode=%d)", sh.G, sh.W, sh.L, sh.mode);
	return -ENOTSUP;
    }
    snprintf(ce->last_kernel, sizeof(ce->last_kernel),
	    "k_rx_auto<G=%d,W=%d,L=%d,mode=0(per-candidate),fill=0,src=%s> threads=%d ring=%u smem=%zu blocks=%d",
	    sh.G, sh.W, sh.L, elem == 2 ? (sh.slide ? "s16,slide" : "s16") : (sh.slide ? "f32,slide" : "f32"),
	    sh.wpb * 32, sh.ring, sh.smem, sh.blocks);
    if (e != cudaSuccess) {
	fsk_b200_set_error("rx_batch_auto launch (G=%d W=%d L=%d ring=%u smem=%zu): %s", sh.G, sh.W, sh.L, sh.ring,
		sh.smem, cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

/* host buffers in, host results out: slabs of streams, copy/compute overlap on two streams.
 * elem = 4: float32 samples; elem = 2: int16 PCM samples, which stay int16 in HBM and are widened
 * inside the rx kernel's ring fill (rows 16-byte aligned, i.e. stride % 8 == 0, and a launch shape
 * with an int16 build; otherwise a separate widening pass runs first).
 * FSK_B200_TRACE=1 prints, per call, where the time went (CUDA events around every step). */
static int rx_batch_host_common(CudaEngine *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const void *host_samples, int elem, size_t nstreams, size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames, fsk_b200_stream_state *host_states)
{
    if (engine_device_check(ce, "rx_batch_host"))
	return -EINVAL;
    /* slab = as many streams as make slab_bytes on the wire (two slabs in flight) */
    size_t slab = ce->slab_bytes / (stride * (size_t)elem);
    if (slab < 1) slab = 1;
    if (slab > nstreams) slab = nstreams;
    bool fused = elem == 2 && (stride & 7) == 0;
    int rc = 0;
#define HOST_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	fsk_b200_set_error("%s: %s", #call, cudaGetErrorString(e_)); rc = -EIO; goto fail; } } while (0)
    {
	const size_t need_bytes = slab * stride * (size_t)elem;
	if (ce->slab_streams < slab || ce->slab_stride != stride || ce->slab_max_frames < max_frames
		|| ce->slab_in_bytes < need_bytes) {
	    /* forget the old shape first: a failed allocation below must not leave it looking valid */
	    ce->slab_streams = ce->slab_stride = ce->slab_max_frames = 0;
	    ce->slab_in_bytes = ce->slab_f32_floats = 0;
	    for (int i = 0; i < 2; i++) {
		cudaFree(ce->d_slab[i]); ce->d_slab[i] = NULL;
		cudaFree(ce->d_slab_in[i]); ce->d_slab_in[i] = NULL;
		cudaFree(ce->d_slab_frames[i]); ce->d_slab_frames[i] = NULL;
		cudaFree(ce->d_slab_states[i]); ce->d_slab_states[i] = NULL;
		HOST_TRY(cudaMalloc(&ce->d_slab_in[i], need_bytes));
		HOST_TRY(cudaMalloc(&ce->d_slab_frames[i], slab * (size_t)max_frames * sizeof(fsk_b200_frame)));
		HOST_TRY(cudaMalloc(&ce->d_slab_states[i], slab * sizeof(fsk_b200_stream_state)));
		if (!ce->st[i])
		    HOST_TRY(cudaStreamCreateWithFlags(&ce->st[i], cudaStreamNonBlocking));
	    }
	    ce->slab_streams = slab;
	    ce->slab_stride = stride;
	    ce->slab_max_frames = max_frames;
	    ce->slab_in_bytes = need_bytes;
	}
    }
    {
	const bool trace = getenv("FSK_B200_TRACE") != NULL;
	const size_t nslabs = (nstreams + slab - 1) / slab;
	cudaEvent_t *ev = NULL;		/* per slab: start, after H2D, after kernel, after D2H */
	if (trace) {
	    ev = (cudaEvent_t *)calloc(nslabs * 4, sizeof(cudaEvent_t));
	    for (size_t i = 0; ev && i < nslabs * 4; i++)
		cudaEventCreate(&ev[i]);
	}
	int k = 0;
	size_t si = 0;
	for (size_t s0 = 0; s0 < nstreams; s0 += slab, k ^= 1, si++) {
	    const size_t ns = nstreams - s0 < slab ? nstreams - s0 : slab;
	    cudaStream_t st = ce->st[k];
	    if (ev) cudaEventRecord(ev[4 * si], st);
	    HOST_TRY(cudaMemcpyAsync(ce->d_slab_in[k], (const char *)host_samples + s0 * stride * (size_t)elem,
			ns * stride * (size_t)elem, cudaMemcpyHostToDevice, st));
	    HOST_TRY(cudaMemcpyAsync(ce->d_slab_states[k], host_states + s0, ns * sizeof(fsk_b200_stream_state),
			cudaMemcpyHostToDevice, st));
	    if (ev) cudaEventRecord(ev[4 * si + 1], st);
	    if (elem == 4) {
		rc = rx_batch_any(ce, g, lc, ce->d_slab_in[k], 4, ns, stride, NULL, nsamples_all,
			ce->d_slab_frames[k], max_frames, ce->d_slab_states[k], st);
	    } else {
		rc = fused ? rx_batch_any(ce, g, lc, ce->d_slab_in[k], 2, ns, stride, NULL, nsamples_all,
			ce->d_slab_frames[k], max_frames, ce->d_slab_states[k], st) : -ENOTSUP;
		if (rc == -ENOTSUP) {		/* no int16 build for this mode's launch shape: widen first */
		    fused = false;
		    if (ce->slab_f32_floats < slab * stride) {
			for (int i = 0; i < 2; i++) {
			    cudaFree(ce->d_slab[i]); ce->d_slab[i] = NULL;
			}
			ce->slab_f32_floats = 0;
			for (int i = 0; i < 2; i++)
			    HOST_TRY(cudaMalloc(&ce->d_slab[i], slab * stride * sizeof(float)));
			ce->slab_f32_floats = slab * stride;
		    }
		    rc = fsk_b200_cuda_s16_to_f32((const int16_t *)ce->d_slab_in[k], ce->d_slab[k], ns, stride, st);
		    if (!rc)
			rc = rx_batch_any(ce, g, lc, ce->d_slab[k], 4, ns, stride, NULL, nsamples_all,
				ce->d_slab_frames[k], max_frames, ce->d_slab_states[k], st);
		}
	    }
	    if (rc)
		goto fail;
	    if (ev) cudaEventRecord(ev[4 * si + 2], st);
	    HOST_TRY(cudaMemcpyAsync(host_frames + s0 * (size_t)max_frames, ce->d_slab_frames[k],
			ns * (size_t)max_frames * sizeof(fsk_b200_frame), cudaMemcpyDeviceToHost, st));
	    HOST_TRY(cudaMemcpyAsync(host_states + s0, ce->d_slab_states[k], ns * sizeof(fsk_b200_stream_state),
			cudaMemcpyDeviceToHost, st));
	    if (ev) cudaEventRecord(ev[4 * si + 3], st);
	}
	HOST_TRY(cudaStreamSynchronize(ce->st[0]));
	HOST_TRY(cudaStreamSynchronize(ce->st[1]));
	if (ev) {
	    float h2d = 0, kern = 0, d2h = 0, wall = 0, gap = 0, t;
	    for (size_t i = 0; i < nslabs; i++) {
		cudaEventElapsedTime(&t, ev[4 * i], ev[4 * i + 1]); h2d += t;
		cudaEventElapsedTime(&t, ev[4 * i + 1], ev[4 * i + 2]); kern += t;
		cudaEventElapsedTime(&t, ev[4 * i + 2], ev[4 * i + 3]); d2h += t;
		if (i + 1 < nslabs) {	/* end of this slab's H2D to the end of the next one's, minus its duration */
		    float nx;
		    cudaEventElapsedTime(&t, ev[4 * i + 1], ev[4 * (i + 1) + 1]);
		    cudaEventElapsedTime(&nx, ev[4 * (i + 1)], ev[4 * (i + 1) + 1]);
		    (void)nx;
		    gap += t;
		}
	    }
	    cudaEventElapsedTime(&wall, ev[0], ev[4 * (nslabs - 1) + 3]);
	    fprintf(stderr, "fsk_b200 trace: %zu slabs of %zu streams (%s%s): wall %.2f ms; per slab: H2D+state %.3f ms, "
		    "kernel(s) %.3f ms, D2H %.3f ms; H2D-end to H2D-end %.3f ms; wire %.2f GB/s\n", nslabs, slab,
		    elem == 2 ? "int16" : "float32", elem == 2 ? (fused ? ", widened in the rx kernel" : ", separate widening pass") : "",
		    wall, h2d / nslabs, kern / nslabs, d2h / nslabs, nslabs > 1 ? gap / (nslabs - 1) : 0.f,
		    (double)nstreams * stride * elem / (wall * 1e6));
	    for (size_t i = 0; i < nslabs * 4; i++)
		cudaEventDestroy(ev[i]);
	    free(ev);
	}
    }
    return 0;
fail:
    /* nothing of this call may still be writing into the caller's buffers when it returns */
    if (ce->st[0]) cudaStreamSynchronize(ce->st[0]);
    if (ce->st[1]) cudaStreamSynchronize(ce->st[1]);
    (void)cudaGetLastError();
    return rc;
#undef HOST_TRY
}

extern "C" int fsk_b200_cuda_rx_batch_host(void *p, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const float *host_samples, size_t nstreams, size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames, fsk_b200_stream_state *host_states)
{
    return rx_batch_host_common((CudaEngine *)p, g, lc, host_samples, 4, nstreams, stride, nsamples_all,
	    host_frames, max_frames, host_states);
}

extern "C" int fsk_b200_cuda_rx_batch_host_s16(void *p, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const int16_t *host_samples, size_t nstreams, size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames, fsk_b200_stream_state *host_states)
{
    return rx_batch_host_common((CudaEngine *)p, g, lc, host_samples, 2, nstreams, stride, nsamples_all,
	    host_frames, max_frames, host_states);
}

extern "C" int fsk_b200_cuda_s16_to_f32(const int16_t *src, float *dst, size_t nstreams, size_t stride,
	void *stream)
{
    const size_t n = nstreams * stride;
    if (n == 0)
	return 0;
    if ((n & 7) == 0 && ((uintptr_t)src & 15) == 0) {
	const size_t n8 = n / 8;
	FSK_LAUNCH(k_s16_to_f32, (unsigned)((n8 + 255) / 256), 256, 0, (cudaStream_t)stream,
		reinterpret_cast<const int4 *>(src), reinterpret_cast<float4 *>(dst), n8);
    } else {
	FSK_LAUNCH(k_s16_to_f32_scalar, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, src, dst, n);
    }
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
	fsk_b200_set_error("s16_to_f32 launch: %s", cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

extern "C" int fsk_b200_cuda_stream_push(float *samples, size_t nstreams, size_t stride, uint32_t *fill,
	fsk_b200_stream_state *states, const float *chunk, size_t chunk_stride, const uint32_t *chunk_len,
	uint32_t chunk_len_all, uint32_t *dropped, void *stream)
{
    if (nstreams == 0)
	return 0;
    const unsigned threads = 128;
    const size_t blocks = (nstreams * 32 + threads - 1) / threads;
    FSK_LAUNCH(k_stream_push, (unsigned)blocks, threads, 0, (cudaStream_t)stream, samples, (unsigned)nstreams,
	    stride, fill, states, chunk, chunk_stride, chunk_len, chunk_len_all, dropped);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
	fsk_b200_set_error("stream_push launch: %s", cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

extern "C" int fsk_b200_cuda_decode(int kind, unsigned shift, unsigned n_data_bits, int msb_first,
	int do_rx_sync, unsigned long long sync_byte, const fsk_b200_frame *frames,
	const fsk_b200_stream_state *states, size_t nstreams, uint32_t max_frames,
	fsk_b200_decoder_state *dstates, uint8_t *out, uint32_t out_stride, uint32_t *out_count,
	void *stream)
{
    if (nstreams == 0)
	return 0;
    const unsigned blocks = (unsigned)((nstreams + 127) / 128);
    cudaStream_t st = (cudaStream_t)stream;
#define DECODE_CASE(K) case K: FSK_LAUNCH(k_decode<K>, blocks, 128, 0, st, shift, n_data_bits, msb_first, \
	    do_rx_sync, sync_byte, frames, states, (unsigned)nstreams, max_frames, dstates, out, \
	    out_stride, out_count); break
    switch (kind) {
	DECODE_CASE(FSK_B200_DECODE_ASCII);
	DECODE_CASE(FSK_B200_DECODE_BINARY);
	DECODE_CASE(FSK_B200_DECODE_BAUDOT);
	DECODE_CASE(FSK_B200_DECODE_CALLERID);
	DECODE_CASE(FSK_B200_DECODE_UIC_GROUND);
	DECODE_CASE(FSK_B200_DECODE_UIC_TRAIN);
	default:
	    fsk_b200_set_error("decode: unknown decoder %d", kind);
	    return -EINVAL;
    }
#undef DECODE_CASE
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
	fsk_b200_set_error("decode launch: %s", cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

/* the drop-in fsk_find_frame: one stream, host samples */
extern "C" int fsk_b200_cuda_find_frame_one(void *p, const fsk_b200_geom *g, const float *host_samples,
	unsigned nfloats, unsigned try_first, unsigned try_max, unsigned try_step, float limit,
	fsk_b200_frame *out)
{
    CudaEngine *ce = (CudaEngine *)p;
    const size_t cap = ((size_t)nfloats + 7) & ~(size_t)3;
    if (ce->d_one_cap < cap) {
	cudaFree(ce->d_one);
	ce->d_one = NULL;
	CUDA_TRY(cudaMalloc(&ce->d_one, cap * sizeof(float)));
	ce->d_one_cap = cap;
    }
    if (!ce->d_args) {
	CUDA_TRY(cudaMalloc(&ce->d_args, 8 * sizeof(uint32_t)));
	CUDA_TRY(cudaMalloc(&ce->d_frame, sizeof(fsk_b200_frame)));
    }
    uint32_t args[8] = { 0, nfloats, try_first, try_max, try_step, 0, 0, 0 };
    memcpy(&args[5], &limit, sizeof(float));
    CUDA_TRY(cudaMemcpy(ce->d_one, host_samples, (size_t)nfloats * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(ce->d_args, args, sizeof(args), cudaMemcpyHostToDevice));
    int rc = fsk_b200_cuda_find_frame_batch(ce, g, ce->d_one, 1, cap, ce->d_args + 0, ce->d_args + 1,
	    ce->d_args + 2, ce->d_args + 3, ce->d_args + 4, (const float *)(ce->d_args + 5), NULL,
	    ce->d_frame, NULL, NULL);
    if (rc)
	return rc;
    CUDA_TRY(cudaMemcpy(out, ce->d_frame, sizeof(*out), cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int fsk_b200_cuda_band_mags(void *p, int fftsize, const float *host_samples,
	unsigned nsamples, unsigned nbands, float *host_mags)
{
    CudaEngine *ce = (CudaEngine *)p;
    if (nsamples == 0) {
	for (unsigned i = 0; i < nbands; i++)
	    host_mags[i] = 0.f;
	return 0;
    }
    if (ce->d_one_cap < nsamples) {
	cudaFree(ce->d_one);
	ce->d_one = NULL;
	CUDA_TRY(cudaMalloc(&ce->d_one, (size_t)nsamples * sizeof(float)));
	ce->d_one_cap = nsamples;
    }
    if (ce->d_mags_cap < nbands) {
	cudaFree(ce->d_mags);
	ce->d_mags = NULL;
	CUDA_TRY(cudaMalloc(&ce->d_mags, (size_t)nbands * sizeof(float)));
	ce->d_mags_cap = nbands;
    }
    CUDA_TRY(cudaMemcpy(ce->d_one, host_samples, (size_t)nsamples * sizeof(float), cudaMemcpyHostToDevice));
    FSK_LAUNCH(k_band_mags, (nbands + 127) / 128, 128, 0, (cudaStream_t)0, ce->d_one, nsamples, fftsize, nbands,
	    ce->d_mags);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpy(host_mags, ce->d_mags, (size_t)nbands * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int fsk_b200_cuda_detect_carrier_batch(int fftsize, const float *samples, size_t nstreams,
	size_t stride, const uint32_t *offset, uint32_t nsamples, float min_mag_threshold,
	int32_t *out_band, void *stream)
{
    if (nstreams == 0)
	return 0;
    const unsigned nbands = (unsigned)fftsize / 2u + 1u;
    const unsigned threads = 128;
    const size_t blocks = (nstreams * 32 + threads - 1) / threads;
    FSK_LAUNCH(k_detect_carrier, (unsigned)blocks, threads, 0, (cudaStream_t)stream, samples, (unsigned)nstreams,
	    stride, offset, nsamples, fftsize, nbands, min_mag_threshold, out_band);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
	fsk_b200_set_error("detect_carrier_batch launch: %s", cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}

extern "C" void *fsk_b200_cuda_upload(const void *host, size_t bytes)
{
    void *d = NULL;
    if (cudaMalloc(&d, bytes ? bytes : 16) != cudaSuccess) {
	fsk_b200_set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(cudaGetLastError()));
	return NULL;
    }
    if (bytes && cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
	fsk_b200_set_error("cudaMemcpy: %s", cudaGetErrorString(cudaGetLastError()));
	cudaFree(d);
	return NULL;
    }
    return d;
}

extern "C" void fsk_b200_cuda_free(void *d)
{
    cudaFree(d);
}

template <typename T>
static void tx_launch(const fsk_b200_tx_plan *p, const void *lut, const fsk_b200_tx_io *io, cudaStream_t st)
{
    const unsigned blocks = (unsigned)((io->nstreams + TX_WARPS - 1) / TX_WARPS);
    /* the sine table goes to shared memory when it is small (16 KB at the default --lut=4096) */
    const unsigned lut_bytes = p->lut_len * (unsigned)sizeof(T);
    const unsigned in_smem = p->lut_len && lut_bytes <= 32768u;
    const size_t smem = (in_smem ? ((lut_bytes + 15u) & ~15u) : 0u) + 96 * sizeof(unsigned)
	    + TX_WARPS * (TX_RING * sizeof(float4) + TX_WRING * sizeof(unsigned));
    /* 16-byte stores when every row starts 16-byte aligned */
    const bool wide = ((uintptr_t)io->out & 15u) == 0 && (io->out_stride * sizeof(T)) % 16u == 0;
    const T *l = (const T *)lut;
    if (wide && p->lut_len)
	FSK_LAUNCH((k_tx_synth<T, 16 / sizeof(T), true>), blocks, TX_WARPS * 32, smem, st, *p, *io, l, in_smem);
    else if (wide)
	FSK_LAUNCH((k_tx_synth<T, 16 / sizeof(T), false>), blocks, TX_WARPS * 32, smem, st, *p, *io, l, in_smem);
    else if (p->lut_len)
	FSK_LAUNCH((k_tx_synth<T, 1, true>), blocks, TX_WARPS * 32, smem, st, *p, *io, l, in_smem);
    else
	FSK_LAUNCH((k_tx_synth<T, 1, false>), blocks, TX_WARPS * 32, smem, st, *p, *io, l, in_smem);
}

extern "C" int fsk_b200_cuda_tx_synth(const fsk_b200_tx_plan *p, const void *lut, const fsk_b200_tx_io *io,
	void *stream)
{
    if (io->nstreams == 0)
	return 0;
    if (p->float_samples)
	tx_launch<float>(p, lut, io, (cudaStream_t)stream);
    else
	tx_launch<int16_t>(p, lut, io, (cudaStream_t)stream);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
	fsk_b200_set_error("tx launch: %s", cudaGetErrorString(e));
	return -EIO;
    }
    return 0;
}
