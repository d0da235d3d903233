/*
 * fsk_b200_internal.h -- private interface between the C host layer
 * (fsk_b200_host.c) and the CUDA translation unit (fsk_b200_kernels.cu).
 * Not installed; include/fsk_b200.h is the public ABI.
 */
#ifndef FSK_B200_INTERNAL_H
#define FSK_B200_INTERNAL_H

#include "fsk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Geometry of one frame candidate as the kernels consume it (passed by value
 * as a kernel parameter, so changing it costs nothing). */
typedef struct fsk_b200_geom {
    unsigned int n_bits;
    unsigned int bit_nsamples;
    unsigned int span;			/* bit_begin[n_bits-1] + bit_nsamples */
    unsigned int lanes_per_window;	/* filled in at launch */
    float	mag_scalar;		/* 2.0f / bit_nsamples, src/fsk.c:132 */
    float	eps_unscaled;		/* FLT_EPSILON / mag_scalar: the :279 threshold before scaling */
    float	inv_n_bits;		/* 1.0f / n_bits */
    unsigned int tw_entries;		/* twiddle table entries the kernels stage in shared memory: bit_nsamples, or
					 * bit_nsamples + 2 * try_max for the sliding fine search (absolute phase index) */
    float	rot[4];			/* exp(-2 pi i b N / fftsize) for b = b_mark, b_space as (re, im), N = bit_nsamples:
					 * the phase step from one bit period to the next (shared-segment search) */
    unsigned int bit_begin[FSK_B200_MAX_BITS];
    unsigned char expect[2][FSK_B200_MAX_BITS];	/* [0]=data [1]=sync; 0,1 or 2 ('d') */
} fsk_b200_geom;

/* rx-loop constants for the rx kernel (by value as well) */
struct fsk_b200_loopc;
typedef struct fsk_b200_loopc {
    unsigned int frame_nsamples, expect_nsamples, nsamples_overscan;
    unsigned int try_max_nocarrier, try_max_carrier;
    float	confidence_threshold, confidence_search_limit;
    unsigned int slide;			/* 1: the per-candidate rx kernel runs its fine searches by sliding (geom.tw_entries covers it) */
} fsk_b200_loopc;

/* ---- shared-segment search plan (the "multi" rx kernel) --------------------------------------
 * When the bit windows of a frame candidate tile (bit_begin[w] == w * bit_nsamples, i.e.
 * expect_nsamples divisible by the number of expected bits: Bell202 1200, Bell103 300, RTTY 45.45 at
 * 8 and 48 kHz ...), all candidates of one fsk_find_frame call (src/fsk.c:477-502) read the same
 * samples cut at different places.  A BATCH of up to three candidates lays one grid of bit periods
 * over them, anchored at one candidate, and cuts every period at the (at most two) offsets where
 * the other candidates' windows begin: each sample is then correlated ONCE, into the sum of its
 * segment, and a window of any candidate of the batch is the sum of the tail segments of one period
 * and the head segments of the next (rotated by the tones' phase advance over one period, geom.rot).
 * A coarse search (try_step = try_max/3) is one batch; a fine search (try_max/8) is up to four. */
#define FSK_MULTI_MAXB 4
typedef struct fsk_b200_mbatch {
    uint16_t	anchor;		/* try offset the period grid is anchored at */
    uint16_t	rho1, rho2;	/* a period is cut into [0,rho1) [rho1,rho2) [rho2,N); segments may be empty */
    uint16_t	t[3];		/* candidate try offsets, in the order fsk_find_frame visits them */
    uint8_t	ncand;		/* 1..3 */
    uint8_t	csplit;		/* wrap-around slot: its segments >= csplit belong to the period BEFORE the anchor (3 = none) */
    uint8_t	cseg[3];	/* first segment of candidate i's windows (0 = it starts where a period starts) */
    int8_t	shift[3];	/* period that window w of candidate i starts in, minus w: -1, 0 or +1 */
    uint8_t	order[3];	/* index of candidate i in the whole search's visiting order */
    uint8_t	pad;
} fsk_b200_mbatch;
typedef struct fsk_b200_mkind {
    uint32_t	nbatch;
    fsk_b200_mbatch b[FSK_MULTI_MAXB];
} fsk_b200_mkind;
/* search kinds of the rx loop: [carrier + 2 * fine]; the fine search of the iteration that ACQUIRES
 * the carrier still uses the no-carrier window (src/minimodem.c:1236-1263 are evaluated before :1357) */
typedef struct fsk_b200_mplan {
    fsk_b200_mkind kind[4];
    uint32_t	always;		/* 1: every coarse search goes through the shared segments (no single-candidate fast path) */
} fsk_b200_mplan;
/* 0 and the plan if every search kind of this mode can run on `slots` period slots, else -1 */
int fsk_b200_mplan_build(const fsk_b200_geom *g, const struct fsk_b200_loopc *lc, unsigned int slots,
	fsk_b200_mplan *out);


/* ---- chunk-prefix table search (the "prefix" rx kernel, k_rx MODE 3) ------------------------------
 * Once per rx-loop iteration the 32 lanes of a stream's warp demodulate the whole search span
 * (try_max - 1 + span samples) against both tones -- every sample is multiplied once, whatever the number
 * of candidates the coarse and the fine search then visit.  Lane g walks its RUN of S consecutive 16-byte
 * pieces of the ring (S odd: the lanes' accesses then spread over all shared-memory banks) in chunks of 8
 * samples (the last chunk of a run holds 4) and leaves, per chunk, the sum of the run's earlier chunks,
 * plus one total per run.  A bit window of ANY candidate is then the difference of two boundary values
 * (the chunk's prefix + the at most seven samples of the boundary's own chunk) plus the totals of the runs
 * in between: a handful of loads instead of bit_nsamples multiply-adds.  The phase is absolute (counted
 * from the 16-byte piece that holds the search position), which changes a window's sums by a unit factor
 * only (src/fsk.c:107-114 takes the magnitude). */
typedef struct fsk_b200_pfx_kind {	/* one search of the rx loop: the candidate set of src/fsk.c:477-484 */
    uint32_t	k_up, k_dn;		/* try_first + k * step for -k_dn <= k <= k_up */
    uint32_t	ncands;			/* 1 + k_up + k_dn */
    uint32_t	step;
} fsk_b200_pfx_kind;
typedef struct fsk_b200_pfx {
    uint32_t	nbnd;		/* boundaries per candidate: n_bits + 1 when the windows tile, else 2 * n_bits (begin, end) */
    uint32_t	bs;		/* lanes per candidate slot (= nbnd); cpr = 32 / bs candidates are analysed side by side */
    uint32_t	cpr;
    uint32_t	pow2;		/* bs is a power of two: butterfly reductions */
    uint32_t	tiles;		/* 1: window w ends where window w + 1 begins */
    uint32_t	S;		/* 16-byte pieces per lane-run (odd) */
    float	inv_S;
    uint32_t	tstride;	/* table entries per lane-run: (S + 1) / 2 chunks, made odd */
    uint32_t	fp, s4;		/* the piece at index q is rotated by table entry (s4 * q) mod fp: fp = fftsize / gcd(4, fftsize), s4 = 4 / gcd */
    float	inv_fp;
    float	loc[4][4][2];	/* [p][k][h]: exp(-2 pi i b j / fftsize) for sample j = 2p + h of a chunk, k = (re, im) of b_mark, (re, im) of b_space */
    fsk_b200_pfx_kind kind[4];	/* [carrier + 2 * fine], as fsk_b200_mplan.kind */
    uint32_t	zero;		/* 0 (an operand the compiler cannot see through) */
} fsk_b200_pfx;

/* ---- transmitter ------------------------------------------------------------------------------
 * Everything the synthesis kernel needs, in the integers and floats fsk_transmit_stdin
 * (src/minimodem.c:114-250) and the tone generator compute them (passed by value). */
#define FSK_B200_ENCODE_WORDS 2		/* pre-encoded data words (fsk_b200_tx_batch) */
typedef struct fsk_b200_tx_plan {
    uint32_t	rate;			/* simpleaudio_get_rate(): the tone's wave length is (float)rate / freq */
    float	f_mark, f_space;
    uint32_t	bit, start, stop;	/* samples of a data bit, the start and the stop tone (0 = none), :96-97, :110-111, :132 */
    uint32_t	idle;			/* samples of the idle tone, idle_carrier_usec * rate / 1000000, :236 */
    uint32_t	n_data_bits;		/* 1..32 */
    uint32_t	tones_per_frame;	/* (start > 0) + n_data_bits + (stop > 0) */
    int		has_start, has_stop;	/* nstartbits > 0, nstopbits > 0 (:95, :109) */
    int		invert_start_stop, msb_first;
    uint32_t	nsync, sync_byte, leader, trailer;
    int		encoder;		/* FSK_B200_ENCODE_* */
    uint32_t	lut_len;		/* 0: sin() per sample */
    float	mag;			/* tone_mag (float output without a table) */
    float	mag_s;			/* (float)mag_s (int16 output without a table), src/simple-tone-generator.c:146-150 */
    int		float_samples;
} fsk_b200_tx_plan;

/* one launch: text rows (or pre-encoded words) in, sample rows out */
typedef struct fsk_b200_tx_io {
    const uint8_t *text;		/* encoder ASCII8 / BAUDOT: [nstreams][text_stride], text_len[s] bytes */
    size_t	text_stride;
    const uint32_t *text_len;
    const uint32_t *words;		/* encoder WORDS: [nstreams][nwords] */
    uint32_t	nwords;
    const uint32_t *lead_in;		/* WORDS: samples of silence before the signal (may be NULL) */
    fsk_b200_tx_state *states;		/* NULL: every stream fresh, and FINAL */
    void	*out;
    size_t	out_stride;
    uint32_t	*out_len;		/* samples written per stream (may be NULL when cap != 0) */
    uint32_t	cap;			/* 0: a row ends with its signal; else exactly cap samples, zero padded / truncated */
    uint32_t	flags;			/* FSK_B200_TX_* */
    size_t	nstreams;
} fsk_b200_tx_io;

void fsk_b200_set_error(const char *fmt, ...);

/* host-side pure derivations (fsk_b200_host.c) */
int fsk_b200_geom_from(unsigned int frame_nsamples, const char *expect_data,
	const char *expect_sync, fsk_b200_geom *g);

/* CUDA side (fsk_b200_kernels.cu) */
int  fsk_b200_cuda_device_ok(void);
void *fsk_b200_cuda_engine_new(void);
void fsk_b200_cuda_engine_destroy(void *ce);
/* (re)build the twiddle table for (fftsize, b_mark, b_space, bit_nsamples) */
int  fsk_b200_cuda_set_table(void *ce, int fftsize, unsigned int b_mark, unsigned int b_space,
	unsigned int bit_nsamples);
const char *fsk_b200_cuda_last_kernel(void *ce);
int  fsk_b200_cuda_tune(void *ce, int lanes_per_stream, int warps_per_block, int ring_floats);
int  fsk_b200_cuda_find_frame_batch(void *ce, const fsk_b200_geom *g, const float *samples,
	size_t nstreams, size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel, fsk_b200_frame *frames, float *bit_mags, void *stream);
int  fsk_b200_cuda_rx_batch(void *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const float *samples, size_t nstreams, size_t stride, const uint32_t *nsamples,
	uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream);
int  fsk_b200_cuda_rx_batch_s16(void *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const int16_t *samples, size_t nstreams, size_t stride, const uint32_t *nsamples,
	uint32_t nsamples_all, fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream);
int  fsk_b200_cuda_rx_batch_host(void *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const float *host_samples, size_t nstreams, size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames, fsk_b200_stream_state *host_states);
/* single-stream helpers behind the drop-in API: host buffers in, host results out */
int  fsk_b200_cuda_find_frame_one(void *ce, const fsk_b200_geom *g, const float *host_samples,
	unsigned int nfloats, unsigned int try_first, unsigned int try_max, unsigned int try_step,
	float limit, fsk_b200_frame *out);
int  fsk_b200_cuda_band_mags(void *ce, int fftsize, const float *host_samples,
	unsigned int nsamples, unsigned int nbands, float *host_mags);
int  fsk_b200_cuda_detect_carrier_batch(int fftsize, const float *samples, size_t nstreams, size_t stride,
	const uint32_t *offset, uint32_t nsamples, float min_mag_threshold, int32_t *out_band, void *stream);
int  fsk_b200_cuda_stream_push(float *samples, size_t nstreams, size_t stride, uint32_t *fill,
	fsk_b200_stream_state *states, const float *chunk, size_t chunk_stride, const uint32_t *chunk_len,
	uint32_t chunk_len_all, uint32_t *dropped, void *stream);
/* the synthesis kernel; lut: device table of plan->lut_len float or int16 entries */
int  fsk_b200_cuda_tx_synth(const fsk_b200_tx_plan *plan, const void *lut, const fsk_b200_tx_io *io,
	void *stream);
/* device copy of `bytes` host bytes (NULL on failure), and its release */
void *fsk_b200_cuda_upload(const void *host, size_t bytes);
void fsk_b200_cuda_free(void *dev);
int  fsk_b200_cuda_s16_to_f32(const int16_t *src, float *dst, size_t nstreams, size_t stride, void *stream);
int  fsk_b200_cuda_rx_batch_host_s16(void *ce, const fsk_b200_geom *g, const fsk_b200_loopc *lc,
	const int16_t *host_samples, size_t nstreams, size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames, fsk_b200_stream_state *host_states);
int  fsk_b200_cuda_decode(int kind, unsigned shift, unsigned n_data_bits, int msb_first, int do_rx_sync,
	unsigned long long sync_byte, const fsk_b200_frame *frames, const fsk_b200_stream_state *states,
	size_t nstreams, uint32_t max_frames, fsk_b200_decoder_state *dstates, uint8_t *out,
	uint32_t out_stride, uint32_t *out_count, void *stream);
unsigned long long fsk_b200_cuda_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
