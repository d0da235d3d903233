/*
 * auto_oracle.c -- TEST INFRASTRUCTURE: the reference's rx loop with --auto-carrier
 * (src/minimodem.c:1176-1220, :1295-1297) and its carrier detector (src/fsk.c:543-581).
 *
 * fsk_oracle.c restates the rx loop for fixed tones (orc_rx_run).  This file includes it for its plan,
 * frame search (orc_find_frame) and loop set-up (orc_rx_derive), and restates the loop itself once more
 * with the carrier scan added: the ring, the search calls, the refinement and the session bookkeeping
 * below are a copy of orc_rx_run's, kept separate so that orc_rx_run and its golden results stay
 * exactly as they are.  A fix to one loop has to be made in the other as well; the CLI comparison in
 * tests/test_auto_carrier_cpu.py covers this copy.  Two modes, as there:
 *   ORC_RX_LITERAL  the reference's sample ring: the scan covers its fill, samples_nvalid;
 *   ORC_RX_FLAT     everything that remains is searchable, and the scan covers a virtual ring
 *                   count v that follows the reference's fill (DESIGN.md section 5): at the loop top
 *                   v = advance >= v ? 0 : v - advance, then, while v < S/2, v grows by
 *                   min(S/2, samples left after pos + v).
 * Every record carries the mark band it was decoded on, and on request every scan is logged (where, which
 * window decided, the band, none / accepted / rejected, and why the loop scanned).  Built by
 * tests/autoorc.py; nothing in the product links it.
 */
#include "fsk_oracle.c"

/* one carrier scan (:1181-1220) */
enum { ORC_SCAN_NONE = 0, ORC_SCAN_ACCEPTED = 1, ORC_SCAN_REJECTED = 2 };	/* outcome */
enum { ORC_SCAN_START = 0, ORC_SCAN_AGAIN = 1, ORC_SCAN_AFTER_DROP = 2, ORC_SCAN_AFTER_STRIKE = 3 }; /* cause */
typedef struct {
    unsigned long long pos;	/* the loop's position */
    unsigned long long nvalid;	/* the samples from pos on that the loop holds */
    int window;			/* the window that found a band; for none, the number of windows scanned */
    int band;			/* the band found, or -1 */
    int outcome;
    int cause;			/* the first scan, one after a scan without a band, after a carrier drop, or
				 * after a strike past the 20th without a carrier */
    unsigned nframes, nreports;	/* records before the scan */
} orc_auto_scan;

typedef struct {
    unsigned *frame_band;	/* [nframes] of the orc_rx_result */
    unsigned *report_band;	/* [nreports] */
    size_t cap_f, cap_r;
    /* the smallest relative margin of any scan window's decision: between its two largest band
     * magnitudes, and between its largest and the threshold (a screen for near-ties) */
    float min_margin;
} orc_auto_bands;

/* the optional scan log of orc_rx_run_auto_log (kept out of orc_auto_bands, whose layout its callers share) */
typedef struct {
    orc_auto_scan *scans;	/* [nscans] */
    size_t nscans, cap;
} orc_auto_scan_log;

static int auto_log(orc_auto_scan_log *l, const orc_auto_scan *e)
{
    if (l->nscans >= l->cap) {
	size_t c = l->cap ? l->cap * 2 : 256;
	orc_auto_scan *p = realloc(l->scans, c * sizeof(*p));
	if (!p)
	    return -1;
	l->scans = p;
	l->cap = c;
    }
    l->scans[l->nscans++] = *e;
    return 0;
}

void orc_auto_scan_log_free(orc_auto_scan_log *l)
{
    free(l->scans);
    memset(l, 0, sizeof(*l));
}

static int auto_push(unsigned **arr, size_t *cap, size_t n, unsigned v)
{
    if (n >= *cap) {
	size_t c = *cap ? *cap * 2 : 256;
	unsigned *p = realloc(*arr, c * sizeof(unsigned));
	if (!p)
	    return -1;
	*arr = p;
	*cap = c;
    }
    (*arr)[n] = v;
    return 0;
}

void orc_auto_bands_free(orc_auto_bands *b)
{
    free(b->frame_band);
    free(b->report_band);
    memset(b, 0, sizeof(*b));
}

/* fsk_detect_carrier (src/fsk.c:543-581): band magnitudes of the first n samples zero-padded to
 * fftsize, bands 1 .. nbands-1, the first strictly largest at or above the threshold; -1 if none.
 * The transform is a DFT in double with the argument reduced exactly in integers (cs: cos and sin
 * of 2 pi r / fftsize for r = 0 .. fftsize-1). */
static int auto_detect(const orc_plan *p, const double *cs, const float *x, unsigned n, float thr,
	float *min_margin)
{
    const unsigned F = (unsigned)p->fftsize;
    const float magscalar = 1.0f / ((float)n / 2.0f);		/* :553 */
    float max_mag = 0.0f, top1 = 0.0f, top2 = 0.0f;
    int best = -1;
    for (unsigned k = 1; k < p->nbands; k++) {			/* :556, :568 */
	double re = 0, im = 0;
	unsigned r = 0;
	for (unsigned i = 0; i < n; i++) {
	    re += (double)x[i] * cs[2 * r];
	    im -= (double)x[i] * cs[2 * r + 1];
	    r += k;
	    if (r >= F)
		r -= F;
	}
	float mag = hypotf((float)re, (float)im) * magscalar;	/* band_mag, :108-113 */
	if (mag > top1) {
	    top2 = top1;
	    top1 = mag;
	} else if (mag > top2) {
	    top2 = mag;
	}
	if (mag < thr)						/* :570 */
	    continue;
	if (max_mag < mag) {					/* :572 */
	    max_mag = mag;
	    best = (int)k;
	}
    }
    const float m = top1 < thr ? (thr - top1) / thr
	    : fminf((top1 - top2) / top1, (top1 - thr) / thr);
    if (m < *min_margin)
	*min_margin = m;
    return best;
}

/* The b_shift of src/minimodem.c:1200-1203 for a plan of this band width. */
int orc_auto_b_shift(float band_width, int autodetect_shift, int inverted)
{
    int b_shift = -(float)(autodetect_shift + band_width / 2.0f) / band_width;
    if (inverted)
	b_shift *= -1;
    return b_shift;
}

/* orc_rx_run (fsk_oracle.c) with carrier_autodetect_threshold = threshold > 0, without --Xrxnoise or
 * call records.  find_frame (NULL: orc_find_frame) is called with ctx = the loop's orc_plan, whose
 * b_mark / b_space are the tones of the moment (the near-tie screen of tests/autoorc.py reads them).
 * res and bands must be zero-initialised before their first use, as there; so must log, which (when not
 * NULL) receives every scan. */
int orc_rx_run_auto_log(const orc_rx_config *cfg, const float *samples, size_t nsamples, int mode,
	float threshold, int autodetect_shift, int inverted, orc_find_frame_fn find_frame,
	orc_rx_result *res, orc_auto_bands *bands, orc_auto_scan_log *log)
{
    if (!find_frame)
	find_frame = default_find_frame;
    orc_rx_derived d;
    orc_plan plan;
    res->nframes = res->nreports = res->ncalls = 0;
    res->n_find_frame_calls = 0;
    bands->min_margin = INFINITY;
    if (log)
	log->nscans = 0;
    orc_rx_derive(cfg, &d);
    if (d.expect_n_bits == 0 || d.expect_n_bits > 64 || !(threshold > 0.0f))
	return -1;
    if (orc_plan_init(&plan, cfg->sample_rate, cfg->f_mark, cfg->f_space, cfg->band_width) != 0)
	return -1;
    const int b_shift = orc_auto_b_shift(plan.band_width, autodetect_shift, inverted);
    float nsamples_per_scan = d.nsamples_per_bit;			/* :1183-1185 */
    if (nsamples_per_scan > plan.fftsize)
	nsamples_per_scan = plan.fftsize;
    const unsigned F = (unsigned)plan.fftsize;

    const size_t S = d.samplebuf_size;
    const size_t touch_max = (size_t)(d.nsamples_per_bit + d.nsamples_overscan) + 2
	    + d.expect_nsamples + (size_t)d.nsamples_per_bit + 2;
    const size_t want_floats = mode == ORC_RX_LITERAL ? S + touch_max : 2 * touch_max + 8;
    float *scratch = calloc(want_floats, sizeof(float));
    double *cs = malloc(sizeof(double) * 2 * F);
    if (!scratch || !cs) {
	free(scratch);
	free(cs);
	return -1;
    }
    for (unsigned r = 0; r < F; r++) {
	cs[2 * r] = cos(2.0 * M_PI * (double)r / (double)F);
	cs[2 * r + 1] = sin(2.0 * M_PI * (double)r / (double)F);
    }
    float *ring = mode == ORC_RX_LITERAL ? scratch : NULL;
    float *tail = mode == ORC_RX_LITERAL ? NULL : scratch;
    size_t samples_nvalid = 0;		/* literal: the ring's fill */
    size_t v = 0;			/* flat: the virtual ring count */
    size_t rd = 0;			/* literal: next unread sample */
    unsigned long long pos = 0;
    size_t nf = 0, nr = 0;

    int carrier_band = -1;				/* :1180 */
    int scan_cause = ORC_SCAN_START;
    int carrier = 0;
    float confidence_total = 0, amplitude_total = 0;
    unsigned nframes_decoded = 0;
    size_t carrier_nsamples = 0;
    unsigned noconfidence = 0;
    unsigned advance = 0;
    float track_amplitude = 0.0f, peak_confidence = 0.0f;
    int rc = 0;

    for (;;) {
	const float *buf;
	size_t nvalid, scan_n;
	if (mode == ORC_RX_LITERAL) {
	    if (advance == S) {				/* :1146-1149 */
		samples_nvalid = 0;
		pos += advance;
		advance = 0;
	    }
	    if (advance) {				/* :1150-1156 */
		if (advance > samples_nvalid)
		    break;
		memmove(ring, ring + advance, (S - advance) * sizeof(float));
		samples_nvalid -= advance;
		pos += advance;
	    }
	    if (samples_nvalid < S / 2) {		/* :1158-1174 */
		size_t r = nsamples - rd;
		if (r > S / 2) r = S / 2;
		memcpy(ring + samples_nvalid, samples + rd, r * sizeof(float));
		rd += r;
		samples_nvalid += r;
	    }
	    nvalid = scan_n = samples_nvalid;
	    buf = ring;
	} else {
	    size_t remaining = nsamples - (size_t)pos;
	    if (advance) {
		if (advance > remaining)
		    break;
		pos += advance;
		remaining -= advance;
	    }
	    v = advance >= v ? 0 : v - advance;
	    if (v < S / 2) {
		size_t add = remaining - v;
		v += add < S / 2 ? add : S / 2;
	    }
	    nvalid = remaining;
	    scan_n = v;
	    buf = samples + pos;
	}
	if (nvalid == 0)				/* :1176 */
	    break;

	if (carrier_band < 0) {				/* :1181-1220 */
	    unsigned i;
	    for (i = 0; i + nsamples_per_scan <= scan_n; i += nsamples_per_scan) {
		carrier_band = auto_detect(&plan, cs, buf + i, (unsigned)nsamples_per_scan, threshold,
			&bands->min_margin);
		if (carrier_band >= 0)
		    break;
	    }
	    advance = i + nsamples_per_scan;
	    if (advance > scan_n)
		advance = scan_n;
	    int b_space = carrier_band + b_shift;
	    if (log) {
		orc_auto_scan e = { pos, nvalid, (int)(i / (unsigned)nsamples_per_scan), carrier_band,
		    carrier_band < 0 ? ORC_SCAN_NONE
			    : b_space < 1 || b_space >= (int)plan.nbands ? ORC_SCAN_REJECTED : ORC_SCAN_ACCEPTED,
		    scan_cause, (unsigned)res->nframes, (unsigned)res->nreports };
		if (auto_log(log, &e))
		    rc = -1;
	    }
	    scan_cause = ORC_SCAN_AGAIN;
	    if (carrier_band < 0)
		continue;
	    if (b_space < 1 || b_space >= (int)plan.nbands) {
		carrier_band = -1;
		continue;
	    }
	    if (plan.b_mark != (unsigned)carrier_band || plan.b_space != (unsigned)b_space) {
		plan.b_mark = (unsigned)carrier_band;	/* fsk_set_tones_by_bandshift, src/fsk.c:585-598 */
		plan.b_space = (unsigned)b_space;
		orc_plan_free(&plan);			/* the tone table follows the bands */
	    }
	}

	if (nvalid < d.expect_nsamples)			/* :1229 */
	    break;

	unsigned try_max;
	if (carrier)
	    try_max = d.nsamples_per_bit * 0.75f + 0.5f;
	else
	    try_max = d.nsamples_per_bit;
	try_max += d.nsamples_overscan;
	unsigned try_step = try_max / 3;
	if (try_step == 0)
	    try_step = 1;

	if (mode != ORC_RX_LITERAL) {
	    /* samples past the end read as zero (batched-API semantic) */
	    size_t need = (size_t)try_max + d.expect_nsamples + (size_t)d.nsamples_per_bit + 2;
	    if (need > 2 * touch_max) need = 2 * touch_max;
	    if (nvalid < need) {
		memset(tail, 0, (2 * touch_max + 8) * sizeof(float));
		memcpy(tail, samples + pos, nvalid * sizeof(float));
		buf = tail;
	    }
	}

	float confidence, amplitude = 0.0f;
	unsigned long long bits = 0;
	unsigned frame_start_sample = 0;
	float limit = cfg->confidence_search_limit;
	unsigned try_first = carrier ? d.nsamples_overscan : 0;
	const char *expect = carrier ? d.expect_data : d.expect_sync;

	confidence = find_frame(&plan, buf, d.expect_nsamples, try_first, try_max,
		try_step, limit, expect, &bits, &amplitude, &frame_start_sample);
	res->n_find_frame_calls++;

	int do_refine_frame = 0;
	if (confidence < peak_confidence * 0.75f) {
	    do_refine_frame = 1;
	    peak_confidence = 0;
	}
	if (amplitude < track_amplitude * 0.25f)
	    confidence = 0;

	if (confidence <= cfg->confidence_threshold) {
	    if (++noconfidence > 20) {
		carrier_band = -1;				/* :1297 */
		scan_cause = carrier ? ORC_SCAN_AFTER_DROP : ORC_SCAN_AFTER_STRIKE;
		if (carrier) {
		    orc_rx_report rp = { nframes_decoded, carrier_nsamples,
			confidence_total, amplitude_total, (unsigned)res->nframes };
		    PUSH(res, reports, nreports, cap_reports, rp);
		    if (auto_push(&bands->report_band, &bands->cap_r, nr++, plan.b_mark))
			rc = -1;
		    carrier = 0;
		    carrier_nsamples = 0;
		    confidence_total = 0;
		    amplitude_total = 0;
		    nframes_decoded = 0;
		    track_amplitude = 0.0f;
		}
	    }
	    advance = try_max;
	    continue;
	}

	carrier_nsamples += d.frame_nsamples;
	unsigned acquired = 0;
	if (carrier) {
	    carrier_nsamples += frame_start_sample;
	    carrier_nsamples -= d.nsamples_overscan;
	} else {
	    carrier = 1;
	    acquired = 1;
	    do_refine_frame = 1;
	}

	if (do_refine_frame && confidence < INFINITY && try_step > 1) {
	    try_step = try_max / 8;
	    if (try_step == 0)
		try_step = 1;
	    float confidence2, amplitude2 = 0.0f;
	    unsigned long long bits2 = 0;
	    unsigned fss2 = 0;
	    confidence2 = find_frame(&plan, buf, d.expect_nsamples, try_first, try_max, try_step,
		    INFINITY, d.expect_data, &bits2, &amplitude2, &fss2);
	    res->n_find_frame_calls++;
	    if (confidence2 > confidence) {
		bits = bits2;
		amplitude = amplitude2;
		frame_start_sample = fss2;
	    }
	}

	track_amplitude = (track_amplitude + amplitude) / 2;
	if (peak_confidence < confidence)
	    peak_confidence = confidence;
	confidence_total += confidence;
	amplitude_total += amplitude;
	nframes_decoded++;
	noconfidence = 0;

	advance = frame_start_sample + d.frame_nsamples - d.nsamples_overscan;

	orc_rx_frame fr = { bits, confidence, amplitude, frame_start_sample, acquired, pos };
	PUSH(res, frames, nframes, cap_frames, fr);
	if (auto_push(&bands->frame_band, &bands->cap_f, nf++, plan.b_mark))
	    rc = -1;
    }

    if (carrier) {
	orc_rx_report rp = { nframes_decoded, carrier_nsamples,
	    confidence_total, amplitude_total, (unsigned)res->nframes };
	PUSH(res, reports, nreports, cap_reports, rp);
	if (auto_push(&bands->report_band, &bands->cap_r, nr++, plan.b_mark))
	    rc = -1;
    }
    orc_plan_free(&plan);
    free(scratch);
    free(cs);
    return rc;
}

/* orc_rx_run_auto_log without the scan log */
int orc_rx_run_auto(const orc_rx_config *cfg, const float *samples, size_t nsamples, int mode,
	float threshold, int autodetect_shift, int inverted, orc_find_frame_fn find_frame,
	orc_rx_result *res, orc_auto_bands *bands)
{
    return orc_rx_run_auto_log(cfg, samples, nsamples, mode, threshold, autodetect_shift, inverted, find_frame,
	    res, bands, NULL);
}
