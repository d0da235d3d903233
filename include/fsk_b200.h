/*
 * fsk_b200.h -- C ABI of the H100-native (sm_90a) FSK demodulation engine.
 *
 * Part 1 is a drop-in for the reference's src/fsk.h (kamalmostafa/minimodem
 * v0.24): same type name, same public scalar fields, same five functions with
 * the same signatures and error behaviour, so that the reference's rx loop
 * (src/minimodem.c:1045, :1265, :1373, :1188, :1219, :1478) links against this
 * library unchanged.  Part 2 is the batched extension the reference does not
 * have: many independent audio streams per call, samples resident in HBM.
 *
 * Plain C: pointers and sizes only, no CUDA or torch types.  `void *stream`
 * arguments are CUDA stream handles (cudaStream_t) passed opaquely; NULL is
 * the default stream.  All reference citations are path:line in the reference
 * tree.
 */
#ifndef FSK_B200_H
#define FSK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ======================================================================== */
/* Part 1 -- drop-in for src/fsk.h                                          */
/* ======================================================================== */

typedef struct fsk_plan fsk_plan;

/* Replaces `struct fsk_plan`, src/fsk.h:30-46.  The scalar fields keep the
 * reference's names, types and order because the rx loop reads them directly
 * (fftsize src/minimodem.c:1184; band_width :1203,:1217,:1340; nbands :1210;
 * b_mark :1340).  The three FFTW members (fftplan, fftin, fftout; src/fsk.h:
 * 42-44) become opaque engine pointers of the same size. */
struct fsk_plan {
    float	sample_rate;
    float	f_mark;
    float	f_space;
    float	filter_bw;	/* declared but never written by the reference either */

    int		fftsize;
    unsigned int nbands;
    float	band_width;
    unsigned int b_mark;
    unsigned int b_space;
    void	*engine;	/* was fftwf_plan fftplan: device-side engine state */
    float	*scratch_in;	/* was float *fftin:  pinned host staging buffer */
    void	*scratch_out;	/* was fftwf_complex *fftout: pinned result buffer */
};

/* src/fsk.h:49-55, src/fsk.c:33-95.  NULL + errno=EINVAL (and the reference's
 * message on stderr) when a tone band falls outside [0, nbands); NULL when the
 * engine cannot be created (no CUDA device: the library has no CPU fallback). */
fsk_plan *fsk_plan_new(float sample_rate, float f_mark, float f_space, float filter_bw);

/* src/fsk.h:57-58, src/fsk.c:97-104 */
void fsk_plan_destroy(fsk_plan *fskp);

/* src/fsk.h:61-71, src/fsk.c:449-538.  `samples` is host memory, borrowed for
 * the call; the callee reads samples[0 .. try_max_nsamples-1 + span) where span
 * is the frame's bit windows (the caller guarantees frame_nsamples valid floats
 * and, like the reference, an allocation that covers the rest).  Out-params are
 * always written.  Returns the best confidence (0.0 = nothing found; may be
 * +inf). */
float fsk_find_frame(fsk_plan *fskp, float *samples, unsigned int frame_nsamples,
	unsigned int try_first_sample,
	unsigned int try_max_nsamples,
	unsigned int try_step_nsamples,
	float try_confidence_search_limit,
	const char *expect_bits_string,
	unsigned long long *bits_outp,
	float *ampl_outp,
	unsigned int *frame_start_outp);

/* src/fsk.h:73-75, src/fsk.c:543-581.  Returns the strongest band >= 1 whose
 * magnitude is >= min_mag_threshold, or -1. */
int fsk_detect_carrier(fsk_plan *fskp, float *samples, unsigned int nsamples,
	float min_mag_threshold);

/* src/fsk.h:77-78, src/fsk.c:584-598 */
void fsk_set_tones_by_bandshift(fsk_plan *fskp, unsigned int b_mark, int b_shift);

/* ======================================================================== */
/* Part 2 -- batched extension (not in the reference)                       */
/* ======================================================================== */

#define FSK_B200_MAX_BITS 64	/* assert at src/fsk.c:463 */

/* What the reference's main() derives from `{baudmode}` + options before it
 * enters the rx loop (src/minimodem.c:819-965).  Fill by hand or with
 * fsk_b200_rx_config_for_mode(). */
typedef struct fsk_b200_rx_config {
    float	sample_rate;		/* :534 */
    float	data_rate;		/* bfsk_data_rate */
    float	f_mark, f_space;	/* :900-934, after --inverted :953 */
    int		inverted;		/* override input only: swap the tones, :953-957 */
    float	band_width;		/* after the clamp at :960 */
    unsigned int n_data_bits;
    int		nstartbits;
    float	nstopbits;
    int		invert_start_stop;
    int		msb_first;
    int		do_rx_sync;
    unsigned long long sync_byte;	/* (unsigned long long)-1 = none, :501 */
    float	confidence_threshold;	/* :513, -c */
    float	confidence_search_limit; /* :523, -l; raised to the threshold, :964 */
    char	expect_data_string[FSK_B200_MAX_BITS + 4]; /* "" = build it, :1116-1119 */
} fsk_b200_rx_config;

/* Restates the baudmode presets, src/minimodem.c:819-965: "rtty", "tdd", "same",
 * "callerid", "uic-train", "uic-ground", "V.21", or a number of baud.  Fields of
 * `overrides` that are non-zero (mark, space, band_width, n_data_bits) or >= 0
 * (nstartbits, nstopbits) take the place of the command-line options -M -S -b
 * -8/-7/-5 --startbits --stopbits; pass NULL for none.  Returns 0, or -1 for an
 * unusable mode (data rate 0, > 64 bits per frame). */
int fsk_b200_rx_config_for_mode(const char *baudmode, float sample_rate,
	const fsk_b200_rx_config *overrides, fsk_b200_rx_config *out);

/* Everything the rx loop derives once (src/minimodem.c:1037-1131) plus the bit
 * window geometry fsk_frame_analyze derives per call (src/fsk.c:183,204,465).
 * Plain data: this is the block that is broadcast to the other GPUs. */
typedef struct fsk_b200_rx_params {
    /* plan, src/fsk.c:45-57 */
    float	sample_rate, f_mark, f_space, band_width;
    int		fftsize;
    unsigned int nbands, b_mark, b_space;
    /* loop constants */
    float	nsamples_per_bit;	/* :1037 */
    unsigned int frame_n_bits;		/* :943 (truncating) */
    unsigned int frame_nsamples;	/* :1113 */
    unsigned int expect_n_bits;		/* :1118 */
    unsigned int expect_nsamples;	/* :1131 (truncating) */
    unsigned int nsamples_overscan;	/* :1105-1108 */
    unsigned int try_max_nocarrier, try_max_carrier;	/* :1236-1241 */
    float	confidence_threshold, confidence_search_limit;
    /* framing, for the host-side bit chop :1415-1428 */
    unsigned int n_data_bits;
    int		nstartbits;
    float	nstopbits;
    int		msb_first, do_rx_sync;
    unsigned long long sync_byte;
    /* bit windows of one frame candidate */
    float	samples_per_bit;	/* (float)expect_nsamples / expect_n_bits, src/fsk.c:465 */
    unsigned int bit_nsamples;		/* src/fsk.c:183 */
    unsigned int bit_begin[FSK_B200_MAX_BITS];	/* src/fsk.c:204,249 */
    unsigned int span_nsamples;		/* bit_begin[n-1] + bit_nsamples */
    char	expect_data[FSK_B200_MAX_BITS + 4];
    char	expect_sync[FSK_B200_MAX_BITS + 4];
} fsk_b200_rx_params;

/* Fails (-1, errno=EINVAL) like fsk_plan_new when a tone band is out of range. */
int fsk_b200_rx_params_derive(const fsk_b200_rx_config *cfg, fsk_b200_rx_params *out);

/* One decoded frame, 20 bytes.  `frame_start` is the within-window start the
 * reference calls frame_start_sample (src/minimodem.c:1257, after refinement);
 * bit 31 is set on the frame that acquired carrier (:1332-1355), which is also
 * where the downstream databits decoder is reset (:1351). */
typedef struct fsk_b200_frame {
    uint32_t	bits_lo, bits_hi;	/* raw fsk_find_frame bits, LSB first */
    float	confidence;		/* coarse-search confidence (:1265) */
    float	amplitude;
    uint32_t	frame_start;
} fsk_b200_frame;
#define FSK_B200_FRAME_ACQUIRED 0x80000000u
/* A record whose frame_start is FSK_B200_FRAME_REPORT is not a frame but the
 * statistics of the carrier session that just ended -- what the reference hands
 * to report_no_carrier() when it drops carrier (src/minimodem.c:1298-1307):
 * bits = carrier_nsamples, confidence = confidence_total, amplitude =
 * amplitude_total; nframes_decoded is the number of frame records since the
 * last ACQUIRED one.  A session still open when the stream ends is reported in
 * fsk_b200_stream_state instead (the reference prints it at exit, :1469-1474). */
#define FSK_B200_FRAME_REPORT 0xFFFFFFFFu

/* Per-stream loop state, readable after a run and accepted back to continue a
 * stream with more audio (streaming use). */
typedef struct fsk_b200_stream_state {
    uint64_t	pos;		/* absolute sample index of the next search window */
    uint32_t	nframes;	/* records written so far (frames + session reports) */
    uint32_t	carrier;	/* :1081 */
    uint32_t	noconfidence;	/* :1087 */
    float	track_amplitude;	/* :1132 */
    float	peak_confidence;	/* :1133 */
    uint32_t	done;		/* loop ended: fewer than expect_nsamples remain (:1229) */
    /* statistics of the open carrier session (:1082-1085) */
    uint64_t	carrier_nsamples;
    float	confidence_total;
    float	amplitude_total;
    uint32_t	nframes_decoded;
    /* statistics, accumulated over launches (not part of the reference's state): frame candidates
     * analysed (fsk_frame_analyze calls, src/fsk.c:487) and searches run (fsk_find_frame calls,
     * src/minimodem.c:1265/:1373) by the fast rx kernel; 0 on the generic path */
    uint32_t	stat_candidates;
    uint32_t	stat_searches;
    uint32_t	reserved;	/* engine-private search hint (part of the resumable state; keep it with the rest) */
} fsk_b200_stream_state;

typedef struct fsk_b200_engine fsk_b200_engine;

/* Creates an engine on the current CUDA device.  NULL + errno (EINVAL bad
 * params, ENODEV no usable CUDA device). */
fsk_b200_engine *fsk_b200_engine_new(const fsk_b200_rx_params *params);
void fsk_b200_engine_destroy(fsk_b200_engine *e);
const fsk_b200_rx_params *fsk_b200_engine_params(const fsk_b200_engine *e);

/* Tuning knobs (0 = engine default): lanes per stream (1..32, power of two),
 * warps per block, ring floats per stream (power of two). */
int fsk_b200_engine_tune(fsk_b200_engine *e, int lanes_per_stream, int warps_per_block,
	int ring_floats);

/* Batched fsk_find_frame (src/fsk.c:449-538): one search per stream, all
 * pointers DEVICE memory.  Stream s reads samples[s*stride + offset[s] ...];
 * floats at or beyond s*stride + nvalid[s] read as 0.  expect_sel[s] selects
 * expect_data (0) or expect_sync (1); try_* and limit follow the reference's
 * arguments.  Outputs: confidence[s], frames[s] (bits, confidence, amplitude,
 * frame_start).  Asynchronous on `stream`.  Returns 0 or a negative errno. */
int fsk_b200_find_frame_batch(fsk_b200_engine *e, const float *samples,
	size_t nstreams, size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel,
	fsk_b200_frame *frames, void *stream);

/* The same search, additionally exporting what fsk_bit_analyze (src/fsk.c:117-174) saw in every bit
 * window of the WINNING candidate: bit_mags[(s*n_bits + b)*2 + 0] = the larger of the two tone
 * magnitudes (the bit's signal, :163/:167), [.. + 1] = the smaller (its noise), both scaled by
 * 2/bit_nsamples as at :132; n_bits = the length of the expect string.  Meaningful for streams whose
 * returned confidence is > 0.  This is the hook the per-bit parity gate uses (tests); it costs one more
 * analysis of the winner per stream.  bit_mags: device memory, 8-byte aligned. */
int fsk_b200_find_frame_batch_bits(fsk_b200_engine *e, const float *samples,
	size_t nstreams, size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel,
	fsk_b200_frame *frames, float *bit_mags, void *stream);

/* Batched rx loop (src/minimodem.c:1137-1463) over whole streams resident in
 * HBM: stream s is samples[s*stride .. s*stride + nsamples[s]) (nsamples NULL =
 * all `nsamples_all` long; -EINVAL if that exceeds `stride`, per-stream lengths are
 * clamped to it).  Frame records go to frames[s*max_frames ...].  `states` (device,
 * one per stream) must be zeroed for a fresh stream; it is updated in place.
 * Limits: a row holds at most 2^32 - 4 samples (lengths and positions inside a row are
 * 32-bit; longer recordings are fed in pieces, see fsk_b200_stream_push), a call at most
 * 2^31 - 1 streams.
 * Output overflow: a stream that has written max_frames records stops there with done = 0
 * and nframes == max_frames; its position and loop state are saved, so it CAN be continued,
 * but only after the caller has consumed the records and set states[s].nframes back to 0
 * (fsk_b200_max_frames() sizes the buffer so that this never happens for a row of nsamples).
 * Asynchronous on `stream`.  Returns 0 or a negative errno. */
int fsk_b200_rx_batch(fsk_b200_engine *e, const float *samples, size_t nstreams,
	size_t stride, const uint32_t *nsamples, uint32_t nsamples_all,
	fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream);

/* Same, from HOST buffers: copies (pinned or pageable) host streams to the
 * device in slabs, overlapping copy and demodulation on two CUDA streams, and
 * copies the records back.  This is the call a host application makes.
 * Synchronous.  Returns 0 or a negative errno. */
int fsk_b200_rx_batch_host(fsk_b200_engine *e, const float *host_samples, size_t nstreams,
	size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames,
	fsk_b200_stream_state *host_states);

/* Live streams.  fsk_b200_rx_batch works on whatever each row holds; a receiver that is fed in
 * chunks keeps, per stream, the samples the loop has not consumed yet and appends the new ones:
 *
 *   fsk_b200_engine_set_holdback(e, fsk_b200_stream_window(p));   // once
 *   for every chunk:
 *       fsk_b200_stream_push(d_rows, n, stride, d_fill, d_states, d_chunk, chunk_stride, d_chunk_len, 0, NULL, st);
 *       fsk_b200_rx_batch(e, d_rows, n, stride, d_fill, 0, d_frames, max_frames, d_states, st);
 *       ... consume states[s].nframes records of each stream ...
 *   at the end of a stream: fsk_b200_engine_set_holdback(e, 0) and one more rx_batch (the reference's
 *   end-of-input rule: it analyses what is left as long as expect_nsamples remain, src/minimodem.c:1229)
 *
 * With the holdback at fsk_b200_stream_window() a search starts only when every sample it can touch
 * has arrived, so the records do not depend on how the stream was cut into chunks.
 *
 * fsk_b200_stream_push: per stream s, the unconsumed tail [states[s].pos, fill[s]) of row s moves to
 * the front, chunk_len[s] (or chunk_len_all when chunk_len is NULL) floats of chunk row s are
 * appended (what does not fit in `stride` is dropped and counted in dropped[s], if given),
 * fill[s] becomes the new length, and the state is set to pos = 0, nframes = 0, done = 0 with the
 * carrier/squelch/session fields untouched.  All pointers are device memory. */
uint32_t fsk_b200_stream_window(const fsk_b200_rx_params *p);
int fsk_b200_engine_set_holdback(fsk_b200_engine *e, uint32_t nsamples);
int fsk_b200_stream_push(float *samples, size_t nstreams, size_t stride, uint32_t *fill,
	fsk_b200_stream_state *states, const float *chunk, size_t chunk_stride, const uint32_t *chunk_len,
	uint32_t chunk_len_all, uint32_t *dropped, void *stream);

/* N3, batched -- fsk_detect_carrier (src/fsk.c:543-581, the --auto-carrier probe of
 * src/minimodem.c:1179-1220) for many streams in one launch: stream s is analysed over the
 * nsamples (1..fftsize) floats at samples[s*stride + offset[s]] (offset may be NULL = 0), zero
 * padded to fftsize; out_band[s] = the band (1..fftsize/2) with the largest magnitude among those
 * >= min_mag_threshold, the lowest such band on a tie, or -1.  The caller applies
 * fsk_set_tones_by_bandshift's rule per stream.  Device pointers. */
int fsk_b200_detect_carrier_batch(int fftsize, const float *samples, size_t nstreams, size_t stride,
	const uint32_t *offset, uint32_t nsamples, float min_mag_threshold, int32_t *out_band, void *stream);

/* --auto-carrier (-a, src/minimodem.c:1179-1220) inside the batched rx loop: every stream finds its own
 * tone pair, and finds it again after each carrier loss.  While a stream has no band it scans windows of
 * min(nsamples_per_bit, fftsize) samples with fsk_detect_carrier's rule; a band b is accepted when its
 * space band b + b_shift lies in [1, nbands), and the same iteration searches a frame on (b, b + b_shift).
 * More than 20 iterations without confidence drop the band (:1295-1297).  The scan covers what the
 * reference's sample ring would hold, so the scan grid is the reference CLI's on the same audio; DESIGN.md
 * section 5, item 10, says where the records can still differ from the CLI's.
 *
 * fsk_b200_auto_state: 16 bytes per stream, all zeros for a fresh stream, kept with the
 * fsk_b200_stream_state to continue a stream.
 * fsk_b200_rx_config_autodetect_shift: the autodetect_shift the reference derives from the data rate
 * (:900-934).
 * fsk_b200_engine_set_auto_carrier: enables the calls below; threshold 0.001 is the CLI's -a, inverted its
 * --inverted.  The band shift is b_shift = (int)(-(float)(autodetect_shift + band_width/2) / band_width),
 * negated when inverted.  -EINVAL (and the calls below disabled) for a threshold that is not positive
 * and finite, for b_shift == 0 (the reference asserts there, src/fsk.c:587), and for a scan window
 * min(nsamples_per_bit, fftsize) under one sample, i.e. a data rate above the sample rate (the
 * reference's scan never advances there).
 * fsk_b200_rx_batch_auto / _s16: fsk_b200_rx_batch / _s16 with the scan; auto_states (device, one per
 * stream) as above; rec_band (device, optional, [nstreams][max_frames]) receives the mark band of every
 * record, the band of the session that ended for a REPORT record.  -ENOTSUP, with nothing launched, where
 * the per-candidate rx kernel cannot take the mode (e.g. 0.5 baud).
 * fsk_b200_auto_stream_window: the holdback for live streams with auto-carrier, max(stream window,
 * samplebuf_size): with it the records do not depend on how a stream is cut into chunks. */
typedef struct fsk_b200_auto_state {
    uint32_t	carrier_band;	/* accepted mark band; 0 = none (bands start at 1) */
    uint32_t	v;		/* virtual ring count: the samples from pos on the reference's ring would hold */
    uint32_t	reserved[2];
} fsk_b200_auto_state;
int fsk_b200_rx_config_autodetect_shift(const fsk_b200_rx_config *cfg);
int fsk_b200_engine_set_auto_carrier(fsk_b200_engine *e, float threshold, int autodetect_shift, int inverted);
int fsk_b200_rx_batch_auto(fsk_b200_engine *e, const float *samples, size_t nstreams,
	size_t stride, const uint32_t *nsamples, uint32_t nsamples_all,
	fsk_b200_frame *frames, uint32_t max_frames, fsk_b200_stream_state *states,
	fsk_b200_auto_state *auto_states, uint32_t *rec_band, void *stream);
int fsk_b200_rx_batch_auto_s16(fsk_b200_engine *e, const int16_t *samples, size_t nstreams,
	size_t stride, const uint32_t *nsamples, uint32_t nsamples_all,
	fsk_b200_frame *frames, uint32_t max_frames, fsk_b200_stream_state *states,
	fsk_b200_auto_state *auto_states, uint32_t *rec_band, void *stream);
uint32_t fsk_b200_auto_stream_window(const fsk_b200_rx_params *p);

/* N2 -- 16-bit PCM ingest (the reference transmitter's default sample format, read back by
 * its rx as float = short / 32768: src/simpleaudio-sndfile.c:43-57, src/minimodem.c:786-788).
 * fsk_b200_s16_to_f32: device conversion (exact: a power-of-two scale), asynchronous on `stream`.
 * fsk_b200_rx_batch_host_s16: like fsk_b200_rx_batch_host, but the host streams are int16 --
 * half the bytes cross PCIe, the widening happens on the device. */
int fsk_b200_s16_to_f32(const int16_t *src, float *dst, size_t nstreams, size_t stride, void *stream);

/* fsk_b200_rx_batch over int16 PCM rows resident in HBM: the samples stay 2 bytes wide in device
 * memory and are widened (short / 32768, exact) inside the rx kernel's shared-memory ring fill, so
 * a sample costs 2 bytes of HBM traffic instead of the 2 + 4 + 4 of a separate widening pass.  Same
 * records, bit for bit, as fsk_b200_rx_batch on the widened floats.  samples: device memory, 16-byte
 * aligned; stride: a multiple of 8 samples.  -ENOTSUP when the mode's launch shape has no int16
 * build (unusual framings; widen with fsk_b200_s16_to_f32 then).  fsk_b200_rx_batch_host_s16 uses
 * this path whenever it can. */
int fsk_b200_rx_batch_s16(fsk_b200_engine *e, const int16_t *samples, size_t nstreams,
	size_t stride, const uint32_t *nsamples, uint32_t nsamples_all,
	fsk_b200_frame *frames, uint32_t max_frames,
	fsk_b200_stream_state *states, void *stream);

/* N2, the file side: where the samples of a RIFF/WAVE image are (the container the reference's
 * tests and its default `--file` output use; the reference itself goes through libsndfile,
 * src/simpleaudio-sndfile.c:88-160).  Mono PCM16 (format 1) and IEEE float32 (format 3) only, which
 * is what its transmitter writes (src/minimodem.c:533, --float-samples).  Host memory.  Returns 0 and
 * fills data_offset (bytes from the start of the image), nsamples, sample_rate and is_float, or
 * -EINVAL for anything else (truncated data chunks are clipped to the image). */
int fsk_b200_wav_locate(const void *image, size_t nbytes, size_t *data_offset, size_t *nsamples,
	uint32_t *sample_rate, int *is_float);
int fsk_b200_rx_batch_host_s16(fsk_b200_engine *e, const int16_t *host_samples, size_t nstreams,
	size_t stride, uint32_t nsamples_all,
	fsk_b200_frame *host_frames, uint32_t max_frames,
	fsk_b200_stream_state *host_states);

/* N1 -- on-device databits decode for the stateless ASCII decoder
 * (databits_decode_ascii8, src/databits_ascii.c:35-44, applied as the rx loop does at
 * src/minimodem.c:1415-1446: prev-stop chop, bit_window, optional bit_reverse, sync-byte
 * suppression).  For every stream, the records [0, states[s].nframes) of
 * frames[s*max_frames ...] become bytes in out[s*out_stride ...]; out_count[s] receives the
 * number of bytes (at most out_stride).  All pointers are device memory. */
int fsk_b200_decode_ascii_batch(const fsk_b200_rx_params *p, const fsk_b200_frame *frames,
	const fsk_b200_stream_state *states, size_t nstreams, uint32_t max_frames,
	uint8_t *out, uint32_t out_stride, uint32_t *out_count, void *stream);

/* N1, all decoders -- the same for any databits decoder of the reference, with the decoder
 * state the reference keeps in file-static variables (src/baudot.c:197,
 * src/databits_callerid.c:45-47) held per stream. */
#define FSK_B200_DECODE_ASCII		0	/* databits_decode_ascii8, src/databits_ascii.c:35-44 */
#define FSK_B200_DECODE_BINARY		1	/* databits_decode_binary, src/databits_binary.c:29-41 */
#define FSK_B200_DECODE_BAUDOT		2	/* databits_decode_baudot, src/databits_baudot.c:30-40 */
#define FSK_B200_DECODE_CALLERID	3	/* databits_decode_callerid, src/databits_callerid.c:163-209 */
#define FSK_B200_DECODE_UIC_GROUND	4	/* databits_decode_uic_ground, src/databits_uic.c:54-63 */
#define FSK_B200_DECODE_UIC_TRAIN	5	/* databits_decode_uic_train, src/databits_uic.c:65-74 */

typedef struct fsk_b200_decoder_state {
    uint32_t	baudot_charset;		/* src/baudot.c:197: 0 unknown, 1 LTRS, 2 FIGS */
    uint32_t	cid_msgtype;		/* src/databits_callerid.c:45 */
    uint32_t	cid_ndata;		/* :46 */
    uint32_t	reserved;
    uint8_t	cid_buf[256];		/* :47; never cleared between messages, as there */
} fsk_b200_decoder_state;		/* 272 bytes; all zeros = the reference at program start */

/* Which decoder the reference's main() would pick (src/minimodem.c:552, :675, :820, :828, :856,
 * :866-868, :891-892): baudmode as given to fsk_b200_rx_config_for_mode, n_data_bits == 5 stands
 * for the -5/--baudot option, binary_output for the --binary-output / --binary-raw switches. */
int fsk_b200_decoder_for_mode(const char *baudmode, unsigned int n_data_bits, int binary_output);

/* Most bytes one frame record can become under `kind` (Caller-ID prints a whole message on
 * its last byte), and most bytes `nframes` records of one stream can become -- the out_stride
 * that never truncates (Caller-ID: a message of L bytes takes L+2 records, so the bound is an
 * amortised 141 bytes per record plus one message carried in from an earlier batch). */
uint32_t fsk_b200_decode_max_bytes_per_frame(int kind, unsigned int n_data_bits);
uint64_t fsk_b200_decode_max_bytes(int kind, unsigned int n_data_bits, uint32_t nframes);

/* For every stream, the records [0, states[s].nframes) of frames[s*max_frames ...] go through
 * the rx loop's chop (src/minimodem.c:1415-1439), the decoder reset on the record that
 * acquired the carrier (:1351) and decoder `kind`; bytes land in out[s*out_stride ...],
 * out_count[s] = bytes produced, at most out_stride (the excess is dropped).  dstates: one
 * fsk_b200_decoder_state per stream, read and written back, so that a stream decoded in
 * several batches continues where it stopped; NULL = start every stream from zeros.
 * All pointers are device memory. */
int fsk_b200_decode_batch(const fsk_b200_rx_params *p, int kind, const fsk_b200_frame *frames,
	const fsk_b200_stream_state *states, size_t nstreams, uint32_t max_frames,
	fsk_b200_decoder_state *dstates,
	uint8_t *out, uint32_t out_stride, uint32_t *out_count, void *stream);

/* Upper bound on frame records a stream of nsamples can produce. */
uint32_t fsk_b200_max_frames(const fsk_b200_rx_params *p, uint32_t nsamples);

/* src/minimodem.c:1415-1428: frame bits -> the data word handed to the
 * databits decoder (prev-stop chop, bit_window, optional bit_reverse). */
unsigned long long fsk_b200_frame_databits(const fsk_b200_rx_params *p, const fsk_b200_frame *f);

/* Device-side synthesis of test streams in the reference transmitter's signal
 * model (src/minimodem.c:81-250, src/simple-tone-generator.c:107-175; float
 * samples through a sine table of table_len entries computed by the caller on
 * the host).  Stream s carries words[s*nwords .. +nwords) after lead_in[s]
 * samples of silence; writes exactly nsamples_out floats per stream (zero
 * padded / truncated).  All pointers are device memory.  -EINVAL for
 * n_data_bits outside 1..32 or nsamples_out > stride. */
typedef struct fsk_b200_tx_config {
    float	sample_rate, data_rate, f_mark, f_space;
    unsigned int n_data_bits;
    float	nstartbits, nstopbits;
    int		invert_start_stop, msb_first;
    unsigned int do_tx_sync_bytes, sync_byte;
    int		leader_bits, trailer_bits;
} fsk_b200_tx_config;

/* The float sine table of the reference tone generator
 * (src/simple-tone-generator.c:53-54): out[i] = mag * sinf((float)M_PI*2*i/len). */
void fsk_b200_sin_table(float *out, unsigned int len, float mag);

int fsk_b200_tx_batch(const fsk_b200_tx_config *cfg, const float *sin_table, uint32_t table_len,
	const uint32_t *words, uint32_t nwords, const uint32_t *lead_in,
	float *samples_out, size_t nstreams, size_t stride, uint32_t nsamples_out, void *stream);

/* ---- the batched transmitter: text in, the reference's `--tx` audio out ----------------------
 *
 *   fsk_b200_tx_config_from_rx(&rx_cfg, &tx_cfg);                 // or fill tx_cfg by hand
 *   te = fsk_b200_tx_engine_new(&tx_cfg, &signal, fsk_b200_encoder_for_mode(mode, n_data_bits));
 *   for every tick:
 *       fsk_b200_tx_text_batch(te, d_text, n, text_stride, d_len, FSK_B200_TX_IDLE_IF_EMPTY,
 *                              d_states, d_audio, out_stride, d_out_len, st);
 *   at the end: one more call with FSK_B200_TX_FINAL (and zero lengths) for the trailers
 *
 * Per stream a call does what the reference's fsk_transmit_stdin (src/minimodem.c:114-250) does
 * for those bytes, with every piece of state the reference keeps in static variables held in
 * the stream's fsk_b200_tx_state, so that a text cut into any pieces gives the same audio. */

/* The encoders of src/databits.h:48-65 */
#define FSK_B200_ENCODE_ASCII8	0	/* databits_encode_ascii8, src/databits_ascii.c:28-33 */
#define FSK_B200_ENCODE_BAUDOT	1	/* baudot_encode, src/baudot.c:258-310 */

/* --volume, --lut and --float-samples (src/minimodem.c:537-538, :686-693, :749) */
typedef struct fsk_b200_tx_signal {
    float	amplitude;		/* tone_mag; 1.0 = full scale */
    uint32_t	sin_table_len;		/* 0: sin() per sample (see DESIGN.md 5 on its rounding) */
    int		float_samples;		/* 0: int16 PCM, 1: float32 */
} fsk_b200_tx_signal;

/* 16 bytes per stream, device memory; all zeros = a fresh reference process */
typedef struct fsk_b200_tx_state {
    float	cphase;			/* sa_tone_cphase, src/simple-tone-generator.c:98 */
    uint32_t	baudot_charset;		/* src/baudot.c:197: 0 unknown, 1 LTRS, 2 FIGS */
    uint32_t	transmitting;		/* tx_transmitting, src/minimodem.c:164-232: 0 idle, 1 carrier, 2 sending */
    uint32_t	reserved;
} fsk_b200_tx_state;

#define FSK_B200_TX_IDLE_IF_EMPTY 1u	/* a stream with no bytes sends one idle tone (the reference's
					 * select() timeout, :230-237) and drops to transmitting = 1 */
#define FSK_B200_TX_FINAL	  2u	/* end of input: transmitting streams send the trailer (:60-74, :246) */

typedef struct fsk_b200_tx_engine fsk_b200_tx_engine;

/* Which encoder the reference's main() would pick (src/minimodem.c:553, :676, :821, :829): Baudot
 * for "rtty", "tdd" and n_data_bits == 5 (the -5 option), ascii8 otherwise. */
int fsk_b200_encoder_for_mode(const char *baudmode, unsigned int n_data_bits);

/* The TX fields main() derives for a receive configuration: leader 2 bits (0 without start
 * bits, :949-951), trailer 2 bits, 16 sync bytes for "same" and --sync-byte (:716-720, :844-845). */
int fsk_b200_tx_config_from_rx(const fsk_b200_rx_config *rx, fsk_b200_tx_config *out);

/* Creates a transmitter on the current CUDA device; it owns the device sine tables, built on the
 * host exactly as simpleaudio_tone_init builds them (src/simple-tone-generator.c:38-72).  NULL +
 * errno: EINVAL for n_data_bits outside 1..32 (the reference's `bits >> i` is undefined beyond),
 * a bit of 0 samples or an unknown encoder; ENODEV without a usable CUDA device. */
fsk_b200_tx_engine *fsk_b200_tx_engine_new(const fsk_b200_tx_config *cfg, const fsk_b200_tx_signal *sig,
	int encoder);
void fsk_b200_tx_engine_destroy(fsk_b200_tx_engine *te);

/* Most samples a row of `nbytes` text bytes can become under `flags` (leader, preamble, Baudot's
 * at most 2 words per byte, the idle tone, the trailer); exact for ascii8 text of nbytes bytes
 * from a fresh state.  0 when it exceeds 2^32 - 1. */
uint64_t fsk_b200_tx_max_samples(const fsk_b200_tx_engine *te, uint32_t nbytes, unsigned int flags);

/* One tick of every stream.  text: uint8 [nstreams][text_stride], text_len[s] bytes of row s
 * (clamped to text_stride); states: one fsk_b200_tx_state per stream, read and written back;
 * out: int16 or float32 (as the signal says) rows [nstreams][out_stride], out_len[s] = samples
 * written to row s (the rest of the row is not touched).  All pointers are device memory;
 * asynchronous on `stream`.  -EINVAL (and no launch) for a NULL pointer or an out_stride below
 * fsk_b200_tx_max_samples(te, text_stride, flags). */
int fsk_b200_tx_text_batch(fsk_b200_tx_engine *te, const uint8_t *text, size_t nstreams, size_t text_stride,
	const uint32_t *text_len, unsigned int flags, fsk_b200_tx_state *states, void *out, size_t out_stride,
	uint32_t *out_len, void *stream);

/* Diagnostics: which kernel instance the engine's latest fsk_b200_rx_batch or fsk_b200_find_frame_batch
 * launched ("k_rx<G=8,W=3,L=2,mode=2(shared-segment),fill=0,src=f32> threads=64 ring=640 smem=23232
 * blocks=8192", "k_find_frame<G=8,W=2,L=1,mode=0(per-candidate)> ..."; "" before the first launch).  `fill`
 * is 1 for the prefix-table kernel's TMA bulk fill (float rows, FSK_B200_PFX_FILL not 0) and 0 otherwise. */
const char *fsk_b200_engine_last_kernel(const fsk_b200_engine *e);

/* Library / build information: "fsk_b200 <version> sm_90a". */
const char *fsk_b200_version(void);
/* Number of kernel launches issued by this library in this process. */
unsigned long long fsk_b200_launch_count(void);
/* Last error message of the calling thread ("" if none). */
const char *fsk_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* FSK_B200_H */
