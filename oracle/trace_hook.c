/*
 * trace_hook.c -- TEST INFRASTRUCTURE.  Interposes on the reference's
 * fsk_find_frame (declared src/fsk.h:61-71) and on its fftwf_execute call
 * (src/fsk.c:157) WITHOUT modifying reference sources: oracle/Makefile
 * compiles the unmodified src/fsk.c with
 *     -Dfsk_find_frame=fsk_find_frame__real -Dfftwf_execute=fftwf_execute__traced
 * so that the rx loop in the unmodified src/minimodem.c (:1265, :1373) calls
 * the wrapper below.  Every call is appended to the binary file named by
 * $ORACLE_TRACE_FILE: inputs, outputs, the raw complex FFT bins (b_mark,
 * b_space) of every bit window analysed, and (if $ORACLE_TRACE_SAMPLES=1) the
 * sample window itself.  tests/golden/make_golden.py turns these traces into
 * the committed golden vectors the reference's own tests lack.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>

#include "fsk.h"	/* the reference's header, via -I/root/reference/src */

float fsk_find_frame__real(fsk_plan *fskp, float *samples, unsigned int frame_nsamples,
	unsigned int try_first_sample, unsigned int try_max_nsamples,
	unsigned int try_step_nsamples, float try_confidence_search_limit,
	const char *expect_bits_string, unsigned long long *bits_outp,
	float *ampl_outp, unsigned int *frame_start_outp);

static FILE *trace_f;
static int trace_samples;
static fsk_plan *cur_plan;
#define MAX_FFT_PER_CALL 4096
static float fft_bins[MAX_FFT_PER_CALL][4];
static uint32_t n_fft;

#undef fftwf_execute
void fftwf_execute__traced(const fftwf_plan plan)
{
    fftwf_execute(plan);
    if (cur_plan && n_fft < MAX_FFT_PER_CALL) {
	fft_bins[n_fft][0] = cur_plan->fftout[cur_plan->b_mark][0];
	fft_bins[n_fft][1] = cur_plan->fftout[cur_plan->b_mark][1];
	fft_bins[n_fft][2] = cur_plan->fftout[cur_plan->b_space][0];
	fft_bins[n_fft][3] = cur_plan->fftout[cur_plan->b_space][1];
	n_fft++;
    }
}

struct trace_rec {
    uint32_t magic;		/* 0x46534b54 "FSKT" */
    uint32_t frame_nsamples, try_first, try_max, try_step;
    float limit;
    char expect[68];
    float confidence;
    uint32_t bits_lo, bits_hi;
    float ampl;
    uint32_t frame_start;
    uint32_t fftsize, b_mark, b_space;
    uint32_t n_fft;
    uint32_t n_window;		/* floats of window that follow the bins */
};

float fsk_find_frame(fsk_plan *fskp, float *samples, unsigned int frame_nsamples,
	unsigned int try_first_sample, unsigned int try_max_nsamples,
	unsigned int try_step_nsamples, float try_confidence_search_limit,
	const char *expect_bits_string, unsigned long long *bits_outp,
	float *ampl_outp, unsigned int *frame_start_outp)
{
    if (!trace_f) {
	const char *path = getenv("ORACLE_TRACE_FILE");
	if (path)
	    trace_f = fopen(path, "wb");
	const char *ws = getenv("ORACLE_TRACE_SAMPLES");
	trace_samples = ws && ws[0] == '1';
    }
    cur_plan = fskp;
    n_fft = 0;
    float c = fsk_find_frame__real(fskp, samples, frame_nsamples,
	    try_first_sample, try_max_nsamples, try_step_nsamples,
	    try_confidence_search_limit, expect_bits_string,
	    bits_outp, ampl_outp, frame_start_outp);
    cur_plan = NULL;
    if (trace_f) {
	struct trace_rec r;
	memset(&r, 0, sizeof(r));
	r.magic = 0x46534b54u;
	r.frame_nsamples = frame_nsamples;
	r.try_first = try_first_sample;
	r.try_max = try_max_nsamples;
	r.try_step = try_step_nsamples;
	r.limit = try_confidence_search_limit;
	strncpy(r.expect, expect_bits_string, sizeof(r.expect) - 1);
	r.confidence = c;
	r.bits_lo = (uint32_t)(*bits_outp & 0xffffffffu);
	r.bits_hi = (uint32_t)(*bits_outp >> 32);
	r.ampl = *ampl_outp;
	r.frame_start = *frame_start_outp;
	r.fftsize = fskp->fftsize;
	r.b_mark = fskp->b_mark;
	r.b_space = fskp->b_space;
	r.n_fft = n_fft;
	/* the callee may touch [0, try_max-1 + span); the rx loop's buffer is
	 * at least 2*(nbits+1)*ceil(spb) floats (src/minimodem.c:1063-1064) so
	 * try_max + frame_nsamples floats are always addressable. */
	r.n_window = trace_samples ? try_max_nsamples + frame_nsamples : 0;
	fwrite(&r, sizeof(r), 1, trace_f);
	fwrite(fft_bins, sizeof(fft_bins[0]), n_fft, trace_f);
	if (r.n_window)
	    fwrite(samples, sizeof(float), r.n_window, trace_f);
	fflush(trace_f);
    }
    return c;
}
