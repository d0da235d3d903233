/*
 * fsk_b200_host.c -- host layer of the FSK engine, plain C.
 *
 *  - the drop-in for the reference's src/fsk.h (fsk_plan_new, fsk_find_frame,
 *    fsk_detect_carrier, fsk_set_tones_by_bandshift, fsk_plan_destroy),
 *  - the scalar derivations the reference's main() performs before its rx loop
 *    (mode presets, frame geometry), restated so that the device kernels see
 *    exactly the integers the reference would compute,
 *  - the batched engine entry points, which validate arguments and hand over
 *    to the CUDA translation unit (fsk_b200_kernels.cu).
 *
 * There is no CPU implementation of the signal path in this library: every
 * analysis call ends in a CUDA kernel, and creation fails with ENODEV when no
 * CUDA device is usable.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <ctype.h>
#include <assert.h>

#include "fsk_b200_internal.h"

static __thread char last_error[256];

void fsk_b200_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(last_error, sizeof(last_error), fmt, ap);
    va_end(ap);
}

const char *fsk_b200_last_error(void) { return last_error; }
#ifdef FSK_EMU	/* tests/emu: the kernels' source on the host SIMT emulator; never the product */
const char *fsk_b200_version(void) { return "fsk_b200 0.1 HOST-EMULATION (tests only)"; }
#else
const char *fsk_b200_version(void) { return "fsk_b200 0.1 sm_90a"; }
#endif
unsigned long long fsk_b200_launch_count(void) { return fsk_b200_cuda_launch_count(); }

/* ------------------------------------------------------------------------ */
/* tone bands: the arithmetic of src/fsk.c:50-57, float32 throughout         */
/* ------------------------------------------------------------------------ */

static int derive_bands(float sample_rate, float f_mark, float f_space, float bw,
	int *fftsize, unsigned int *nbands, unsigned int *b_mark, unsigned int *b_space)
{
    float half = bw / 2.0f;
    *fftsize = (sample_rate + half) / bw;
    *nbands = *fftsize / 2 + 1;
    *b_mark = (f_mark + half) / bw;
    *b_space = (f_space + half) / bw;
    return (*b_mark >= *nbands || *b_space >= *nbands) ? -1 : 0;
}

/* ------------------------------------------------------------------------ */
/* mode presets (src/minimodem.c:819-965)                                   */
/* ------------------------------------------------------------------------ */

int fsk_b200_rx_config_for_mode(const char *baudmode, float sample_rate,
	const fsk_b200_rx_config *ov, fsk_b200_rx_config *out)
{
    fsk_b200_rx_config c;
    memset(&c, 0, sizeof(c));
    c.sample_rate = sample_rate;
    c.nstartbits = -1;
    c.nstopbits = -1;
    c.sync_byte = (unsigned long long)-1;
    c.confidence_threshold = 1.5f;		/* :513 */
    c.confidence_search_limit = 2.3f;		/* :523 */
    if (ov) {					/* what the option switch would have set */
	c.f_mark = ov->f_mark;
	c.f_space = ov->f_space;
	c.band_width = ov->band_width;
	c.n_data_bits = ov->n_data_bits;
	c.nstartbits = ov->nstartbits;
	c.nstopbits = ov->nstopbits;
	c.invert_start_stop = ov->invert_start_stop;
	c.msb_first = ov->msb_first;
	if (ov->do_rx_sync) {
	    c.do_rx_sync = 1;
	    c.sync_byte = ov->sync_byte;
	}
	if (ov->confidence_threshold > 0.0f)
	    c.confidence_threshold = ov->confidence_threshold;
	if (ov->confidence_search_limit > 0.0f)
	    c.confidence_search_limit = ov->confidence_search_limit;
    }

    if (strncasecmp(baudmode, "rtty", 5) == 0) {		/* :819 */
	c.data_rate = 45.45;
	if (c.n_data_bits == 0) c.n_data_bits = 5;
	if (c.nstopbits < 0) c.nstopbits = 1.5;
    } else if (strncasecmp(baudmode, "tdd", 4) == 0) {		/* :827 */
	c.data_rate = 45.45;
	if (c.n_data_bits == 0) c.n_data_bits = 5;
	if (c.nstopbits < 0) c.nstopbits = 2.0;
	c.f_mark = 1400;
	c.f_space = 1800;
    } else if (strncasecmp(baudmode, "same", 5) == 0) {		/* :837 */
	c.data_rate = 520.0 + 5 / 6.0;
	c.n_data_bits = 8;
	c.nstartbits = 0;
	c.nstopbits = 0;
	c.do_rx_sync = 1;
	c.sync_byte = 0xAB;
	c.f_mark = 2083.0 + 1 / 3.0;
	c.f_space = 1562.5;
	c.band_width = c.data_rate;
    } else if (strncasecmp(baudmode, "caller", 6) == 0) {	/* :849 */
	c.data_rate = 1200;
	c.n_data_bits = 8;
    } else if (strncasecmp(baudmode, "uic", 3) == 0) {		/* :859 */
	c.data_rate = 600;
	c.n_data_bits = 39;
	c.f_mark = 1300;
	c.f_space = 1700;
	c.nstartbits = 8;
	c.nstopbits = 0;
	strcpy(c.expect_data_string, "11110010ddddddddddddddddddddddddddddddddddddddd");
    } else if (strncasecmp(baudmode, "V.21", 4) == 0) {		/* :877 */
	c.data_rate = 300;
	c.f_mark = 980;
	c.f_space = 1180;
	c.n_data_bits = 8;
    } else {							/* :882 */
	c.data_rate = atof(baudmode);
	if (c.n_data_bits == 0) c.n_data_bits = 8;
    }
    if (c.data_rate == 0.0f) {
	fsk_b200_set_error("unusable baudmode '%s'", baudmode);
	errno = EINVAL;
	return -1;
    }

    int shift;
    if (c.data_rate >= 400) {					/* :900 Bell202-like */
	shift = -(c.data_rate * 5 / 6);
	if (c.f_mark == 0) c.f_mark = c.data_rate / 2 + 600;
	if (c.f_space == 0) c.f_space = c.f_mark - shift;
	if (c.band_width == 0) c.band_width = 200;
    } else if (c.data_rate >= 100) {				/* :911 Bell103-like */
	shift = 200;
	if (c.f_mark == 0) c.f_mark = 1270;
	if (c.f_space == 0) c.f_space = c.f_mark - shift;
	if (c.band_width == 0) c.band_width = 50;
    } else {							/* :922 RTTY-like */
	shift = 170;
	if (c.f_mark == 0) c.f_mark = 1585;
	if (c.f_space == 0) c.f_space = c.f_mark - shift;
	if (c.band_width == 0) c.band_width = 10;
    }
    if (c.nstartbits < 0) c.nstartbits = 1;			/* :937-940 */
    if (c.nstopbits < 0) c.nstopbits = 1.0;

    unsigned int frame_n_bits = c.n_data_bits + c.nstartbits + c.nstopbits;	/* :943 */
    if (frame_n_bits > 64) {
	fsk_b200_set_error("total number of bits per frame must be <= 64");
	errno = EINVAL;
	return -1;
    }
    if (ov && ov->inverted) {				/* --inverted, :953-957 */
	float t = c.f_mark;
	c.f_mark = c.f_space;
	c.f_space = t;
    }
    if (c.band_width > c.data_rate)				/* :960 */
	c.band_width = c.data_rate;
    if (c.confidence_search_limit < c.confidence_threshold)	/* :964 */
	c.confidence_search_limit = c.confidence_threshold;
    *out = c;
    return 0;
}

/* ------------------------------------------------------------------------ */
/* frame geometry and loop constants                                        */
/* ------------------------------------------------------------------------ */

/* the expect string, src/minimodem.c:442-487 */
static int build_expect(char *s, int nstartbits, int n_data_bits, float nstopbits,
	int invert_start_stop, int use_bits, unsigned long long bits)
{
    const char startv = invert_start_stop ? '1' : '0';
    const char stopv = invert_start_stop ? '0' : '1';
    int n = 0;
    if (nstopbits != 0.0f)
	s[n++] = stopv;
    for (int i = 0; i < nstartbits; i++)
	s[n++] = startv;
    for (int i = 0; i < n_data_bits; i++)
	s[n++] = use_bits ? (char)('0' + ((bits >> i) & 1)) : 'd';
    if (nstopbits != 0.0f)
	s[n++] = stopv;
    s[n] = 0;
    return n;
}

int fsk_b200_geom_from(unsigned int frame_nsamples, const char *expect_data,
	const char *expect_sync, fsk_b200_geom *g)
{
    memset(g, 0, sizeof(*g));
    size_t n = strlen(expect_data);
    if (n == 0 || n > FSK_B200_MAX_BITS || (expect_sync && strlen(expect_sync) != n))
	return -1;
    g->n_bits = (unsigned int)n;
    float spb = (float)frame_nsamples / (int)n;		/* src/fsk.c:465 */
    g->bit_nsamples = (float)(spb + 0.5f);		/* src/fsk.c:183 */
    if (g->bit_nsamples == 0)
	return -1;
    for (unsigned int b = 0; b < g->n_bits; b++)
	g->bit_begin[b] = (float)(spb * (int)b + 0.5f);	/* src/fsk.c:204,249 */
    g->span = g->bit_begin[g->n_bits - 1] + g->bit_nsamples;
    g->mag_scalar = 2.0f / (float)g->bit_nsamples;	/* src/fsk.c:132 */
    g->eps_unscaled = 1.1920928955078125e-07f / g->mag_scalar;
    g->inv_n_bits = 1.0f / (float)(int)g->n_bits;
    g->lanes_per_window = 1;
    g->tw_entries = g->bit_nsamples;
    for (int k = 0; k < 2; k++) {
	const char *e = k ? (expect_sync ? expect_sync : expect_data) : expect_data;
	for (unsigned int b = 0; b < g->n_bits; b++) {
	    if (e[b] == 'd') g->expect[k][b] = 2;
	    else if (e[b] == '0' || e[b] == '1') g->expect[k][b] = (unsigned char)(e[b] - '0');
	    else return -1;				/* assert at src/fsk.c:202 */
	}
    }
    return 0;
}

int fsk_b200_rx_params_derive(const fsk_b200_rx_config *cfg, fsk_b200_rx_params *p)
{
    memset(p, 0, sizeof(*p));
    p->sample_rate = cfg->sample_rate;
    p->f_mark = cfg->f_mark;
    p->f_space = cfg->f_space;
    p->band_width = cfg->band_width;
    if (!(cfg->band_width > 0) || !(cfg->sample_rate > 0) || !(cfg->data_rate > 0)) {
	fsk_b200_set_error("rx config: rates and band width must be positive");
	errno = EINVAL;
	return -1;
    }
    if (derive_bands(cfg->sample_rate, cfg->f_mark, cfg->f_space, cfg->band_width,
		&p->fftsize, &p->nbands, &p->b_mark, &p->b_space) != 0) {
	fprintf(stderr, "b_mark=%u or b_space=%u is invalid (nbands=%u)\n",
		p->b_mark, p->b_space, p->nbands);		/* src/fsk.c:59-60 */
	errno = EINVAL;
	return -1;
    }
    unsigned int sample_rate = (unsigned int)cfg->sample_rate;
    p->nsamples_per_bit = sample_rate / cfg->data_rate;		/* :1037 */
    p->frame_n_bits = cfg->n_data_bits + cfg->nstartbits + cfg->nstopbits;	/* :943 */

    const float overscan = 0.5f;				/* :1091 */
    p->nsamples_overscan = p->nsamples_per_bit * overscan + 0.5f;	/* :1105 */
    if (p->nsamples_overscan == 0)
	p->nsamples_overscan = 1;
    float frame_n_bits = p->frame_n_bits;
    p->frame_nsamples = p->nsamples_per_bit * frame_n_bits + 0.5f;	/* :1113 */

    if (cfg->expect_data_string[0]) {				/* :1116 (uic supplies one) */
	/* at most FSK_B200_MAX_BITS characters (the reference asserts that in src/fsk.c:463) */
	size_t n = strnlen(cfg->expect_data_string, FSK_B200_MAX_BITS);
	memcpy(p->expect_data, cfg->expect_data_string, n);
	p->expect_data[n] = 0;
	p->expect_n_bits = (unsigned int)n;
    } else {
	p->expect_n_bits = build_expect(p->expect_data, cfg->nstartbits, cfg->n_data_bits,
		cfg->nstopbits, cfg->invert_start_stop, 0, 0);
    }
    if (cfg->do_rx_sync && (long long)cfg->sync_byte >= 0)	/* :1123 */
	build_expect(p->expect_sync, cfg->nstartbits, cfg->n_data_bits, cfg->nstopbits,
		cfg->invert_start_stop, 1, cfg->sync_byte);
    else
	strcpy(p->expect_sync, p->expect_data);
    if (p->expect_n_bits == 0 || p->expect_n_bits > FSK_B200_MAX_BITS
	    || strlen(p->expect_sync) != p->expect_n_bits) {
	fsk_b200_set_error("expect string must be 1..64 bits");
	errno = EINVAL;
	return -1;
    }
    p->expect_nsamples = p->nsamples_per_bit * p->expect_n_bits;	/* :1131 */

    p->try_max_carrier = p->nsamples_per_bit * 0.75f + 0.5f;	/* :1238 */
    p->try_max_carrier += p->nsamples_overscan;			/* :1241 */
    p->try_max_nocarrier = p->nsamples_per_bit;			/* :1240 */
    p->try_max_nocarrier += p->nsamples_overscan;

    p->confidence_threshold = cfg->confidence_threshold;
    p->confidence_search_limit = cfg->confidence_search_limit;
    p->n_data_bits = cfg->n_data_bits;
    p->nstartbits = cfg->nstartbits;
    p->nstopbits = cfg->nstopbits;
    p->msb_first = cfg->msb_first;
    p->do_rx_sync = cfg->do_rx_sync;
    p->sync_byte = cfg->sync_byte;

    fsk_b200_geom g;
    if (fsk_b200_geom_from(p->expect_nsamples, p->expect_data, p->expect_sync, &g) != 0) {
	fsk_b200_set_error("bad expect string or empty bit window");
	errno = EINVAL;
	return -1;
    }
    p->samples_per_bit = (float)p->expect_nsamples / (int)p->expect_n_bits;
    p->bit_nsamples = g.bit_nsamples;
    memcpy(p->bit_begin, g.bit_begin, sizeof(p->bit_begin));
    p->span_nsamples = g.span;
    return 0;
}

/* ------------------------------------------------------------------------ */
/* shared-segment search plan (fsk_b200_internal.h)                          */
/* ------------------------------------------------------------------------ */

struct cand { int t; unsigned order; };

/* the visiting order of src/fsk.c:477-484 */
static unsigned enumerate_candidates(unsigned first, unsigned tmax, unsigned step, struct cand *c, unsigned cap)
{
    unsigned n = 0, order = 0;
    if (step == 0)
	step = 1;
    for (int j = 0;; j++) {
	const int up = (j & 1) ? 1 : -1;
	const int t = (int)first + up * ((j + 1) / 2) * (int)step;
	if (t >= (int)tmax)
	    break;
	if (t < 0) {
	    if (j > 4 * (int)tmax + 8)
		break;			/* cannot happen: the upward side ends the scan */
	    continue;
	}
	if (n == cap)
	    return cap + 1;
	c[n].t = t;
	c[n].order = order++;
	n++;
    }
    return n;
}

/* one batch over candidates c[0..n) (n <= 3) anchored at `anchor`; -1 if they do not fit the scheme */
static int plan_batch(const struct cand *c, unsigned n, int anchor, unsigned N, unsigned n_bits,
	unsigned slots, fsk_b200_mbatch *b)
{
    memset(b, 0, sizeof(*b));
    int r[3], d[3];
    unsigned rho[3] = { 0, 0, 0 }, nrho = 1;
    for (unsigned i = 0; i < n; i++) {
	const int off = c[i].t - anchor;
	d[i] = off >= 0 ? off / (int)N : -((-off + (int)N - 1) / (int)N);
	r[i] = off - d[i] * (int)N;
	if (d[i] == 1 && r[i] != 0)
	    return -1;
	if (d[i] == -1 && r[i] == 0)
	    return -1;
	if (d[i] < -1 || d[i] > 1)
	    return -1;
	unsigned k;
	for (k = 0; k < nrho; k++)
	    if (rho[k] == (unsigned)r[i])
		break;
	if (k == nrho) {
	    if (nrho == 3)
		return -1;
	    rho[nrho++] = (unsigned)r[i];
	}
    }
    /* sort the residues; rho[0] = 0 is the smallest by construction */
    if (nrho == 3 && rho[1] > rho[2]) { unsigned x = rho[1]; rho[1] = rho[2]; rho[2] = x; }
    b->anchor = (uint16_t)anchor;
    b->rho1 = (uint16_t)(nrho > 1 ? rho[1] : N);
    b->rho2 = (uint16_t)(nrho > 2 ? rho[2] : N);
    b->ncand = (uint8_t)n;
    unsigned max_fwd = 0, min_back = 3, need_last_full = 0, any_back = 0;
    for (unsigned i = 0; i < n; i++) {
	unsigned k;
	for (k = 0; k < nrho; k++)
	    if (rho[k] == (unsigned)r[i])
		break;
	b->t[i] = (uint16_t)c[i].t;
	b->cseg[i] = (uint8_t)k;
	b->shift[i] = (int8_t)d[i];
	b->order[i] = (uint8_t)c[i].order;
	if (d[i] == 0 && k > max_fwd)
	    max_fwd = k;		/* reads segments < k of period n_bits */
	if (d[i] == 1)
	    need_last_full = 1;		/* reads all of period n_bits */
	if (d[i] == -1) {
	    any_back = 1;
	    if (k < min_back)
		min_back = k;		/* reads segments >= k of period -1 */
	}
    }
    /* periods 0..n_bits need a slot each; period -1 lives in the last slot (wrap-around) */
    if (slots < n_bits + 1u)
	return -1;
    b->csplit = 3;
    if (any_back) {
	if (slots - 1u > n_bits)
	    b->csplit = 0;			/* a slot of its own */
	else if (!need_last_full && max_fwd <= min_back)
	    b->csplit = (uint8_t)min_back;	/* shared with period n_bits: disjoint segments */
	else
	    return -1;
    }
    return 0;
}

int fsk_b200_mplan_build(const fsk_b200_geom *g, const fsk_b200_loopc *lc, unsigned int slots,
	fsk_b200_mplan *out)
{
    memset(out, 0, sizeof(*out));
    const unsigned N = g->bit_nsamples;
    if (N < 2 || N > 0xfff0u || g->n_bits > 32)
	return -1;
    for (unsigned w = 0; w < g->n_bits; w++)
	if (g->bit_begin[w] != w * N)
	    return -1;				/* the bit windows do not tile */
    for (int kind = 0; kind < 4; kind++) {
	const int carrier = kind & 1, fine = kind >> 1;
	const unsigned tmax = carrier ? lc->try_max_carrier : lc->try_max_nocarrier;	/* src/minimodem.c:1236-1241 */
	const unsigned first = carrier ? lc->nsamples_overscan : 0u;			/* :1263 */
	unsigned step = tmax / 3u;							/* :1248-1251 */
	if (step == 0)
	    step = 1;
	if (tmax > 0xfff0u)
	    return -1;
	if (fine) {
	    if (step <= 1u) {			/* :1357: no fine search in this mode */
		out->kind[kind].nbatch = 0;
		continue;
	    }
	    step = tmax / 8u;								/* :1360-1362 */
	    if (step == 0)
		step = 1;
	}
	struct cand c[3 * FSK_MULTI_MAXB];
	const unsigned n = enumerate_candidates(first, tmax, step, c, 3 * FSK_MULTI_MAXB);
	if (n == 0 || n > 3 * FSK_MULTI_MAXB)
	    return -1;
	fsk_b200_mkind *k = &out->kind[kind];
	if (!fine) {
	    /* one batch, anchored at the candidate visited first: in the steady state that one wins
	     * (src/fsk.c:499) and it is the cheapest to evaluate (its windows are whole periods) */
	    if (n > 3 || plan_batch(c, n, c[0].t, N, g->n_bits, slots, &k->b[0]) != 0)
		return -1;
	    k->nbatch = 1;
	} else {
	    /* sorted by offset, three neighbours per batch, anchored at the smallest */
	    for (unsigned i = 1; i < n; i++)
		for (unsigned j = i; j > 0 && c[j].t < c[j - 1].t; j--) {
		    struct cand x = c[j]; c[j] = c[j - 1]; c[j - 1] = x;
		}
	    unsigned nb = 0;
	    for (unsigned i = 0; i < n; i += 3, nb++) {
		const unsigned m = n - i < 3 ? n - i : 3;
		/* inside a batch the kernel keeps the visiting order */
		struct cand bc[3];
		for (unsigned q = 0; q < m; q++)
		    bc[q] = c[i + q];
		for (unsigned q = 1; q < m; q++)
		    for (unsigned j = q; j > 0 && bc[j].order < bc[j - 1].order; j--) {
			struct cand x = bc[j]; bc[j] = bc[j - 1]; bc[j - 1] = x;
		    }
		if (nb == FSK_MULTI_MAXB || plan_batch(bc, m, c[i].t, N, g->n_bits, slots, &k->b[nb]) != 0)
		    return -1;
	    }
	    k->nbatch = nb;
	}
    }
    return 0;
}

uint32_t fsk_b200_max_frames(const fsk_b200_rx_params *p, uint32_t nsamples)
{
    /* every recorded frame advances by at least frame_nsamples - overscan (:1407);
     * every session report is preceded by 21 no-confidence advances of try_max (:1295,:1318) */
    unsigned int min_adv = p->frame_nsamples > p->nsamples_overscan
	? p->frame_nsamples - p->nsamples_overscan : 1;
    unsigned int drop_adv = 21u * (p->try_max_carrier ? p->try_max_carrier : 1u);
    return nsamples / min_adv + nsamples / drop_adv + 4;
}

unsigned long long fsk_b200_frame_databits(const fsk_b200_rx_params *p, const fsk_b200_frame *f)
{
    unsigned long long bits = ((unsigned long long)f->bits_hi << 32) | f->bits_lo;
    if (p->nstopbits != 0.0f)			/* :1415 drop the previous frame's stop bit */
	bits >>= 1;
    bits >>= p->nstartbits;			/* bit_window, src/databits.h:35-46 */
    if (p->n_data_bits < 64)
	bits &= (1ULL << p->n_data_bits) - 1;
    if (p->msb_first) {				/* bit_reverse keeps 32 bits, src/databits.h:21-33 */
	unsigned int r = 0;
	for (unsigned int i = 0; i < p->n_data_bits; i++)
	    r = (r << 1) | (unsigned int)((bits >> i) & 1);
	bits = r;
    }
    return bits;
}

/* ------------------------------------------------------------------------ */
/* batched engine                                                           */
/* ------------------------------------------------------------------------ */

struct fsk_b200_engine {
    fsk_b200_rx_params params;
    fsk_b200_geom geom;
    fsk_b200_loopc loopc;
    void *ce;			/* CUDA-side state */
};

fsk_b200_engine *fsk_b200_engine_new(const fsk_b200_rx_params *params)
{
    if (!params || params->expect_n_bits == 0 || params->expect_n_bits > FSK_B200_MAX_BITS) {
	fsk_b200_set_error("engine_new: bad params");
	errno = EINVAL;
	return NULL;
    }
    if (!fsk_b200_cuda_device_ok()) {
	fsk_b200_set_error("engine_new: no usable CUDA device (this library has no CPU path)");
	errno = ENODEV;
	return NULL;
    }
    fsk_b200_engine *e = calloc(1, sizeof(*e));
    if (!e)
	return NULL;
    e->params = *params;
    if (fsk_b200_geom_from(params->expect_nsamples, params->expect_data, params->expect_sync,
		&e->geom) != 0) {
	free(e);
	fsk_b200_set_error("engine_new: bad frame geometry");
	errno = EINVAL;
	return NULL;
    }
    {	/* phase advance of the two tones over one bit period, argument reduced exactly in integers */
	const unsigned long long F = (unsigned long long)(params->fftsize > 0 ? params->fftsize : 1);
	const double am = 2.0 * M_PI * (double)(((unsigned long long)params->b_mark * e->geom.bit_nsamples) % F) / (double)F;
	const double as = 2.0 * M_PI * (double)(((unsigned long long)params->b_space * e->geom.bit_nsamples) % F) / (double)F;
	e->geom.rot[0] = (float)cos(am);
	e->geom.rot[1] = (float)-sin(am);
	e->geom.rot[2] = (float)cos(as);
	e->geom.rot[3] = (float)-sin(as);
    }
    e->loopc.frame_nsamples = params->frame_nsamples;
    e->loopc.expect_nsamples = params->expect_nsamples;
    e->loopc.nsamples_overscan = params->nsamples_overscan;
    e->loopc.try_max_nocarrier = params->try_max_nocarrier;
    e->loopc.try_max_carrier = params->try_max_carrier;
    e->loopc.confidence_threshold = params->confidence_threshold;
    e->loopc.confidence_search_limit = params->confidence_search_limit;
    {	/* the sliding fine search indexes the table by (candidate offset + sample): up to try_max + N + a step */
	const unsigned tmax = params->try_max_nocarrier > params->try_max_carrier
	    ? params->try_max_nocarrier : params->try_max_carrier;
	const unsigned want = e->geom.bit_nsamples + 2u * tmax;
	if ((size_t)want * 16u <= 12u * 1024u && !getenv("FSK_B200_NO_SLIDE")) {
	    e->geom.tw_entries = want;
	    e->loopc.slide = 1;
	}
    }
    e->ce = fsk_b200_cuda_engine_new();
    if (!e->ce || fsk_b200_cuda_set_table(e->ce, params->fftsize, params->b_mark,
		params->b_space, e->geom.tw_entries) != 0) {
	if (e->ce)
	    fsk_b200_cuda_engine_destroy(e->ce);
	free(e);
	errno = ENODEV;
	return NULL;
    }
    return e;
}

const char *fsk_b200_engine_last_kernel(const fsk_b200_engine *e)
{
    return e ? fsk_b200_cuda_last_kernel(e->ce) : "";
}

void fsk_b200_engine_destroy(fsk_b200_engine *e)
{
    if (!e)
	return;
    fsk_b200_cuda_engine_destroy(e->ce);
    free(e);
}

const fsk_b200_rx_params *fsk_b200_engine_params(const fsk_b200_engine *e) { return &e->params; }

int fsk_b200_engine_tune(fsk_b200_engine *e, int lanes_per_stream, int warps_per_block,
	int ring_floats)
{
    return fsk_b200_cuda_tune(e->ce, lanes_per_stream, warps_per_block, ring_floats);
}

static int check_layout(const float *samples, size_t stride)
{
    if (!samples || ((uintptr_t)samples & 15) || (stride & 3)) {
	fsk_b200_set_error("samples must be 16-byte aligned and stride a multiple of 4 floats");
	return -EINVAL;
    }
    return 0;
}

int fsk_b200_find_frame_batch(fsk_b200_engine *e, const float *samples, size_t nstreams,
	size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel, fsk_b200_frame *frames, void *stream)
{
    if (nstreams == 0)
	return 0;
    int rc = check_layout(samples, stride);
    if (rc)
	return rc;
    if (!nvalid || !try_first || !try_max || !try_step || !limit || !frames) {
	fsk_b200_set_error("find_frame_batch: NULL argument");
	return -EINVAL;
    }
    return fsk_b200_cuda_find_frame_batch(e->ce, &e->geom, samples, nstreams, stride, offset,
	    nvalid, try_first, try_max, try_step, limit, expect_sel, frames, NULL, stream);
}

int fsk_b200_find_frame_batch_bits(fsk_b200_engine *e, const float *samples, size_t nstreams,
	size_t stride, const uint32_t *offset, const uint32_t *nvalid,
	const uint32_t *try_first, const uint32_t *try_max, const uint32_t *try_step,
	const float *limit, const uint8_t *expect_sel, fsk_b200_frame *frames, float *bit_mags, void *stream)
{
    if (nstreams == 0)
	return 0;
    int rc = check_layout(samples, stride);
    if (rc)
	return rc;
    if (!nvalid || !try_first || !try_max || !try_step || !limit || !frames || !bit_mags
	    || ((uintptr_t)bit_mags & 7)) {
	fsk_b200_set_error("find_frame_batch_bits: NULL or misaligned argument");
	return -EINVAL;
    }
    return fsk_b200_cuda_find_frame_batch(e->ce, &e->geom, samples, nstreams, stride, offset,
	    nvalid, try_first, try_max, try_step, limit, expect_sel, frames, bit_mags, stream);
}

int fsk_b200_rx_batch(fsk_b200_engine *e, const float *samples, size_t nstreams, size_t stride,
	const uint32_t *nsamples, uint32_t nsamples_all, fsk_b200_frame *frames,
	uint32_t max_frames, fsk_b200_stream_state *states, void *stream)
{
    if (nstreams == 0)
	return 0;
    int rc = check_layout(samples, stride);
    if (rc)
	return rc;
    if (!frames || !states || max_frames == 0) {
	fsk_b200_set_error("rx_batch: NULL argument");
	return -EINVAL;
    }
    if (!nsamples && (size_t)nsamples_all > stride) {
	fsk_b200_set_error("rx_batch: nsamples_all (%u) exceeds the row stride (%zu)", nsamples_all, stride);
	return -EINVAL;
    }
    if (nstreams > 0x7fffffffu) {
	fsk_b200_set_error("rx_batch: at most 2^31-1 streams per call");
	return -EINVAL;
    }
    return fsk_b200_cuda_rx_batch(e->ce, &e->geom, &e->loopc, samples, nstreams, stride,
	    nsamples, nsamples_all, frames, max_frames, states, stream);
}

int fsk_b200_rx_batch_s16(fsk_b200_engine *e, const int16_t *samples, size_t nstreams, size_t stride,
	const uint32_t *nsamples, uint32_t nsamples_all, fsk_b200_frame *frames,
	uint32_t max_frames, fsk_b200_stream_state *states, void *stream)
{
    if (nstreams == 0)
	return 0;
    if (!samples || ((uintptr_t)samples & 15) || (stride & 7)) {
	fsk_b200_set_error("rx_batch_s16: samples must be 16-byte aligned and stride a multiple of 8 samples");
	return -EINVAL;
    }
    if (!frames || !states || max_frames == 0) {
	fsk_b200_set_error("rx_batch_s16: NULL argument");
	return -EINVAL;
    }
    if ((!nsamples && (size_t)nsamples_all > stride) || nstreams > 0x7fffffffu) {
	fsk_b200_set_error("rx_batch_s16: nsamples_all (%u) exceeds the row stride (%zu), or too many streams",
		nsamples_all, stride);
	return -EINVAL;
    }
    int rc = fsk_b200_cuda_rx_batch_s16(e->ce, &e->geom, &e->loopc, samples, nstreams, stride,
	    nsamples, nsamples_all, frames, max_frames, states, stream);
    if (rc == -ENOTSUP)
	fsk_b200_set_error("rx_batch_s16: this mode's launch shape has no int16 build; widen with fsk_b200_s16_to_f32 "
		"and call fsk_b200_rx_batch (fsk_b200_rx_batch_host_s16 does that by itself)");
    return rc;
}

/* ---- live streams ------------------------------------------------------------ */

uint32_t fsk_b200_stream_window(const fsk_b200_rx_params *p)
{
    /* the farthest sample a loop iteration that starts at `pos` can depend on: its last candidate
     * plus the span of the frame's bit windows (src/fsk.c:481, :204) -- or, for frames with more stop
     * bits than the search string covers (frame_n_bits > expect_n_bits, e.g. 3 stop bits), the largest
     * advance frame_start + frame_nsamples - overscan (src/minimodem.c:1407): an iteration held back
     * by this many samples can neither read past the chunk nor hit the end-of-input exit of :1151
     * after it has already recorded its frame */
    if (!p)
	return 0u;
    const unsigned adv = p->frame_nsamples > p->nsamples_overscan ? p->frame_nsamples - p->nsamples_overscan : 0u;
    const unsigned tmax = p->try_max_nocarrier > p->try_max_carrier ? p->try_max_nocarrier : p->try_max_carrier;
    return tmax - 1u + (p->span_nsamples > adv ? p->span_nsamples : adv);
}

int fsk_b200_engine_set_holdback(fsk_b200_engine *e, uint32_t nsamples)
{
    if (!e) {
	fsk_b200_set_error("set_holdback: NULL engine");
	return -EINVAL;
    }
    /* the loop's own stop rule (src/minimodem.c:1229) is the floor */
    e->loopc.expect_nsamples = nsamples > e->params.expect_nsamples ? nsamples : e->params.expect_nsamples;
    return 0;
}

int fsk_b200_stream_push(float *samples, size_t nstreams, size_t stride, uint32_t *fill,
	fsk_b200_stream_state *states, const float *chunk, size_t chunk_stride, const uint32_t *chunk_len,
	uint32_t chunk_len_all, uint32_t *dropped, void *stream)
{
    if (nstreams == 0)
	return 0;
    int rc = check_layout(samples, stride);
    if (rc)
	return rc;
    if (!fill || !states || (!chunk && (chunk_len || chunk_len_all))) {
	fsk_b200_set_error("stream_push: NULL argument");
	return -EINVAL;
    }
    if (!fsk_b200_cuda_device_ok()) {
	fsk_b200_set_error("no usable CUDA device (there is no CPU fallback)");
	return -ENODEV;
    }
    return fsk_b200_cuda_stream_push(samples, nstreams, stride, fill, states, chunk, chunk_stride, chunk_len,
	    chunk_len_all, dropped, stream);
}

int fsk_b200_rx_batch_host(fsk_b200_engine *e, const float *host_samples, size_t nstreams,
	size_t stride, uint32_t nsamples_all, fsk_b200_frame *host_frames, uint32_t max_frames,
	fsk_b200_stream_state *host_states)
{
    if (nstreams == 0)
	return 0;
    if (!host_samples || !host_frames || !host_states || (stride & 3) || max_frames == 0) {
	fsk_b200_set_error("rx_batch_host: bad argument (stride must be a multiple of 4)");
	return -EINVAL;
    }
    if ((size_t)nsamples_all > stride || nstreams > 0x7fffffffu) {
	fsk_b200_set_error("rx_batch_host: nsamples_all (%u) exceeds the row stride (%zu), or too many streams",
		nsamples_all, stride);
	return -EINVAL;
    }
    return fsk_b200_cuda_rx_batch_host(e->ce, &e->geom, &e->loopc, host_samples, nstreams,
	    stride, nsamples_all, host_frames, max_frames, host_states);
}

int fsk_b200_s16_to_f32(const int16_t *src, float *dst, size_t nstreams, size_t stride, void *stream)
{
    if (!src || !dst || (stride & 3) || ((uintptr_t)dst & 15) || ((uintptr_t)src & 7)) {
	fsk_b200_set_error("s16_to_f32: stride must be a multiple of 4, src 8-byte and dst 16-byte aligned");
	return -EINVAL;
    }
    return fsk_b200_cuda_s16_to_f32(src, dst, nstreams, stride, stream);
}

static uint32_t rd_u32le(const unsigned char *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }
static uint32_t rd_u16le(const unsigned char *p) { return p[0] | p[1] << 8; }

int fsk_b200_wav_locate(const void *image, size_t nbytes, size_t *data_offset, size_t *nsamples,
	uint32_t *sample_rate, int *is_float)
{
    const unsigned char *b = image;
    if (!b || !data_offset || !nsamples || !sample_rate || !is_float || nbytes < 12
	    || memcmp(b, "RIFF", 4) != 0 || memcmp(b + 8, "WAVE", 4) != 0) {
	fsk_b200_set_error("wav_locate: not a RIFF/WAVE image");
	return -EINVAL;
    }
    size_t pos = 12;
    int have_fmt = 0;
    unsigned fmt = 0, channels = 0, bits = 0;
    while (pos + 8 <= nbytes) {
	const uint32_t len = rd_u32le(b + pos + 4);
	const unsigned char *body = b + pos + 8;
	if (memcmp(b + pos, "fmt ", 4) == 0 && len >= 16 && pos + 8 + 16 <= nbytes) {
	    fmt = rd_u16le(body);
	    channels = rd_u16le(body + 2);
	    *sample_rate = rd_u32le(body + 4);
	    bits = rd_u16le(body + 14);
	    have_fmt = 1;
	} else if (memcmp(b + pos, "data", 4) == 0) {
	    if (!have_fmt || channels != 1 || !((fmt == 1 && bits == 16) || (fmt == 3 && bits == 32))) {
		fsk_b200_set_error("wav_locate: only mono PCM16 and float32 are supported (format %u, %u channels, %u bits)",
			fmt, channels, bits);
		return -EINVAL;
	    }
	    size_t n = len;
	    if (n > nbytes - (pos + 8))
		n = nbytes - (pos + 8);		/* a writer that died before patching the header */
	    *data_offset = pos + 8;
	    *is_float = fmt == 3;
	    *nsamples = n / (bits / 8);
	    return 0;
	}
	pos += 8 + (size_t)len + (len & 1);
    }
    fsk_b200_set_error("wav_locate: no data chunk");
    return -EINVAL;
}

int fsk_b200_rx_batch_host_s16(fsk_b200_engine *e, const int16_t *host_samples, size_t nstreams,
	size_t stride, uint32_t nsamples_all, fsk_b200_frame *host_frames, uint32_t max_frames,
	fsk_b200_stream_state *host_states)
{
    if (nstreams == 0)
	return 0;
    if (!host_samples || !host_frames || !host_states || (stride & 3) || max_frames == 0) {
	fsk_b200_set_error("rx_batch_host_s16: bad argument (stride must be a multiple of 4)");
	return -EINVAL;
    }
    return fsk_b200_cuda_rx_batch_host_s16(e->ce, &e->geom, &e->loopc, host_samples, nstreams,
	    stride, nsamples_all, host_frames, max_frames, host_states);
}

int fsk_b200_decoder_for_mode(const char *baudmode, unsigned int n_data_bits, int binary_output)
{
    int kind = FSK_B200_DECODE_ASCII;				/* src/minimodem.c:552 */
    if (!baudmode)
	return -EINVAL;
    if (n_data_bits == 5)					/* -5/--baudot, :673-676 */
	kind = FSK_B200_DECODE_BAUDOT;
    if (strncasecmp(baudmode, "rtty", 5) == 0 || strncasecmp(baudmode, "tdd", 4) == 0)
	kind = FSK_B200_DECODE_BAUDOT;				/* :820, :828 */
    else if (strncasecmp(baudmode, "caller", 6) == 0)
	kind = FSK_B200_DECODE_CALLERID;			/* :856 */
    else if (strncasecmp(baudmode, "uic", 3) == 0)		/* :865-868: "uic-t..." is train-to-ground */
	kind = strlen(baudmode) > 4 && tolower((unsigned char)baudmode[4]) == 't'
		? FSK_B200_DECODE_UIC_TRAIN : FSK_B200_DECODE_UIC_GROUND;
    if (binary_output)
	kind = FSK_B200_DECODE_BINARY;				/* :891-892 */
    return kind;
}

uint32_t fsk_b200_decode_max_bytes_per_frame(int kind, unsigned int n_data_bits)
{
    switch (kind) {
	case FSK_B200_DECODE_ASCII:
	case FSK_B200_DECODE_BAUDOT:
	    return 1;
	case FSK_B200_DECODE_BINARY:
	    return n_data_bits + 1;
	case FSK_B200_DECODE_CALLERID:
	    /* "CALLER-ID\n" + at most 127 two-byte fields of 10 label bytes, or one 255-byte field */
	    return 10 + 127 * 10 + 256;
	case FSK_B200_DECODE_UIC_GROUND:
	case FSK_B200_DECODE_UIC_TRAIN:
	    /* "Train ID: XXXXXX - Message: XX (" + the longest meaning (25) + ")\n" */
	    return 32 + 25 + 2;
	default:
	    return 0;
    }
}

uint64_t fsk_b200_decode_max_bytes(int kind, unsigned int n_data_bits, uint32_t nframes)
{
    if (kind == FSK_B200_DECODE_CALLERID)
	/* SDMF with a wrapped length is the densest: "CALLER-ID\n" + two labels + a date + up to
	 * 246 buffer bytes + '\n' = 282 bytes for 2 records */
	return (uint64_t)141 * nframes + fsk_b200_decode_max_bytes_per_frame(kind, n_data_bits);
    return (uint64_t)fsk_b200_decode_max_bytes_per_frame(kind, n_data_bits) * nframes;
}

int fsk_b200_decode_batch(const fsk_b200_rx_params *p, int kind, const fsk_b200_frame *frames,
	const fsk_b200_stream_state *states, size_t nstreams, uint32_t max_frames,
	fsk_b200_decoder_state *dstates,
	uint8_t *out, uint32_t out_stride, uint32_t *out_count, void *stream)
{
    if (!p || !frames || !states || !out || !out_count || out_stride == 0 || max_frames == 0) {
	fsk_b200_set_error("decode_batch: NULL argument");
	return -EINVAL;
    }
    if (kind < FSK_B200_DECODE_ASCII || kind > FSK_B200_DECODE_UIC_TRAIN) {
	fsk_b200_set_error("decode_batch: unknown decoder %d", kind);
	return -EINVAL;
    }
    /* src/minimodem.c:1415 (drop the previous stop bit) + bit_window's offset */
    unsigned shift = (p->nstopbits != 0.0f ? 1u : 0u) + (unsigned)p->nstartbits;
    return fsk_b200_cuda_decode(kind, shift, p->n_data_bits, p->msb_first, p->do_rx_sync, p->sync_byte,
	    frames, states, nstreams, max_frames, dstates, out, out_stride, out_count, stream);
}

int fsk_b200_decode_ascii_batch(const fsk_b200_rx_params *p, const fsk_b200_frame *frames,
	const fsk_b200_stream_state *states, size_t nstreams, uint32_t max_frames,
	uint8_t *out, uint32_t out_stride, uint32_t *out_count, void *stream)
{
    return fsk_b200_decode_batch(p, FSK_B200_DECODE_ASCII, frames, states, nstreams, max_frames, NULL,
	    out, out_stride, out_count, stream);
}

void fsk_b200_sin_table(float *out, unsigned int len, float mag)
{
    for (unsigned int i = 0; i < len; i++)
	out[i] = mag * sinf((float)M_PI * 2 * i / len);
}

/* ------------------------------------------------------------------------ */
/* transmitter                                                              */
/* ------------------------------------------------------------------------ */

/* the integers fsk_transmit_stdin derives (src/minimodem.c:131-132, :96-97, :110-111, :155, :236) */
static int tx_plan_from(const fsk_b200_tx_config *c, int encoder, fsk_b200_tx_plan *p)
{
    memset(p, 0, sizeof(*p));
    if (c->n_data_bits < 1 || c->n_data_bits > 32) {
	fsk_b200_set_error("tx: n_data_bits must be 1..32 (got %u)", c->n_data_bits);
	return -EINVAL;
    }
    if (encoder != FSK_B200_ENCODE_ASCII8 && encoder != FSK_B200_ENCODE_BAUDOT && encoder != FSK_B200_ENCODE_WORDS) {
	fsk_b200_set_error("tx: unknown encoder %d", encoder);
	return -EINVAL;
    }
    if (!(c->sample_rate >= 1.0f && c->sample_rate < 16777216.0f) || !(c->data_rate > 0.0f)
	    || !(c->f_mark > 0.0f) || !(c->f_space > 0.0f) || c->leader_bits < 0 || c->trailer_bits < 0) {
	fsk_b200_set_error("tx: bad sample rate, data rate, tone or leader/trailer length");
	return -EINVAL;
    }
    const size_t sample_rate = (size_t)c->sample_rate;
    const size_t bit = sample_rate / c->data_rate + 0.5f;
    if (bit == 0 || bit > 0xffffffffu) {
	fsk_b200_set_error("tx: a bit of %zu samples", bit);
	return -EINVAL;
    }
    p->rate = (uint32_t)sample_rate;
    p->f_mark = c->f_mark;
    p->f_space = c->f_space;
    p->bit = (uint32_t)bit;
    p->has_start = c->nstartbits > 0;
    p->has_stop = c->nstopbits > 0;
    p->start = p->has_start ? (uint32_t)(size_t)(bit * c->nstartbits) : 0;
    p->stop = p->has_stop ? (uint32_t)(size_t)(bit * c->nstopbits) : 0;
    p->idle = (uint32_t)((1000000u / 25) * sample_rate / 1000000);
    p->n_data_bits = c->n_data_bits;
    p->tones_per_frame = (uint32_t)p->has_start + c->n_data_bits + (uint32_t)p->has_stop;
    p->invert_start_stop = c->invert_start_stop;
    p->msb_first = c->msb_first;
    p->nsync = c->do_tx_sync_bytes;
    p->sync_byte = c->sync_byte;
    p->leader = (uint32_t)c->leader_bits;
    p->trailer = (uint32_t)c->trailer_bits;
    p->encoder = encoder;
    return 0;
}

int fsk_b200_tx_batch(const fsk_b200_tx_config *cfg, const float *sin_table, uint32_t table_len,
	const uint32_t *words, uint32_t nwords, const uint32_t *lead_in, float *samples_out,
	size_t nstreams, size_t stride, uint32_t nsamples_out, void *stream)
{
    if (!cfg || !sin_table || table_len == 0 || !words || !samples_out) {
	fsk_b200_set_error("tx_batch: NULL argument");
	return -EINVAL;
    }
    if (nsamples_out > stride) {
	fsk_b200_set_error("tx_batch: nsamples_out %u exceeds the stride %zu", nsamples_out, stride);
	return -EINVAL;
    }
    fsk_b200_tx_plan p;
    int rc = tx_plan_from(cfg, FSK_B200_ENCODE_WORDS, &p);
    if (rc)
	return rc;
    p.lut_len = table_len;
    p.float_samples = 1;
    if (nsamples_out == 0)
	return 0;
    fsk_b200_tx_io io;
    memset(&io, 0, sizeof(io));
    io.words = words;
    io.nwords = nwords;
    io.lead_in = lead_in;
    io.out = samples_out;
    io.out_stride = stride;
    io.cap = nsamples_out;
    io.nstreams = nstreams;
    return fsk_b200_cuda_tx_synth(&p, sin_table, &io, stream);
}

struct fsk_b200_tx_engine {
    fsk_b200_tx_plan plan;
    void *d_lut;		/* the sine table of the output format, device memory */
};

int fsk_b200_encoder_for_mode(const char *baudmode, unsigned int n_data_bits)
{
    if (!baudmode)
	return -EINVAL;
    if (n_data_bits == 5 || strncasecmp(baudmode, "rtty", 5) == 0 || strncasecmp(baudmode, "tdd", 4) == 0)
	return FSK_B200_ENCODE_BAUDOT;				/* :676, :821, :829 */
    return FSK_B200_ENCODE_ASCII8;				/* :553 */
}

int fsk_b200_tx_config_from_rx(const fsk_b200_rx_config *rx, fsk_b200_tx_config *out)
{
    if (!rx || !out)
	return -EINVAL;
    memset(out, 0, sizeof(*out));
    out->sample_rate = rx->sample_rate;
    out->data_rate = rx->data_rate;
    out->f_mark = rx->f_mark;
    out->f_space = rx->f_space;
    out->n_data_bits = rx->n_data_bits;
    out->nstartbits = (float)rx->nstartbits;
    out->nstopbits = rx->nstopbits;
    out->invert_start_stop = rx->invert_start_stop;
    out->msb_first = rx->msb_first;
    out->do_tx_sync_bytes = rx->do_rx_sync ? 16u : 0u;			/* :716-720, :844-845 */
    out->sync_byte = rx->do_rx_sync ? (unsigned int)rx->sync_byte : 0u;
    out->leader_bits = rx->nstartbits == 0 ? 0 : 2;			/* :51, :949-951 */
    out->trailer_bits = 2;						/* :52 */
    return 0;
}

fsk_b200_tx_engine *fsk_b200_tx_engine_new(const fsk_b200_tx_config *cfg, const fsk_b200_tx_signal *sig,
	int encoder)
{
    if (!cfg || !sig || !(sig->amplitude > 0.0f) || (encoder != FSK_B200_ENCODE_ASCII8
		&& encoder != FSK_B200_ENCODE_BAUDOT)) {
	fsk_b200_set_error("tx_engine_new: bad argument");
	errno = EINVAL;
	return NULL;
    }
    fsk_b200_tx_engine *te = calloc(1, sizeof(*te));
    if (!te) {
	errno = ENOMEM;
	return NULL;
    }
    if (tx_plan_from(cfg, encoder, &te->plan)) {
	free(te);
	errno = EINVAL;
	return NULL;
    }
    if (!fsk_b200_cuda_device_ok()) {
	fsk_b200_set_error("tx_engine_new: no usable CUDA device");
	free(te);
	errno = ENODEV;
	return NULL;
    }
    /* simpleaudio_tone_init, src/simple-tone-generator.c:38-72, and the mag_s of :145-150 */
    const float mag = sig->amplitude;
    unsigned short mag_s = 32767.0f * mag + 0.5f;
    if (mag > 1.0f)
	mag_s = 32767;
    if (mag_s < 1)
	mag_s = 1;
    te->plan.lut_len = sig->sin_table_len;
    te->plan.mag = mag;
    te->plan.mag_s = (float)mag_s;
    te->plan.float_samples = sig->float_samples != 0;
    const unsigned len = sig->sin_table_len;
    if (len) {
	const size_t bytes = (size_t)len * (te->plan.float_samples ? sizeof(float) : sizeof(short));
	void *t = malloc(bytes);
	if (!t) {
	    free(te);
	    errno = ENOMEM;
	    return NULL;
	}
	if (te->plan.float_samples)
	    fsk_b200_sin_table((float *)t, len, mag);
	else
	    for (unsigned i = 0; i < len; i++)
		((short *)t)[i] = lroundf(mag_s * sinf((float)M_PI * 2 * i / len));
	te->d_lut = fsk_b200_cuda_upload(t, bytes);
	free(t);
	if (!te->d_lut) {
	    free(te);
	    errno = ENODEV;
	    return NULL;
	}
    }
    return te;
}

void fsk_b200_tx_engine_destroy(fsk_b200_tx_engine *te)
{
    if (!te)
	return;
    if (te->d_lut)
	fsk_b200_cuda_free(te->d_lut);
    free(te);
}

uint64_t fsk_b200_tx_max_samples(const fsk_b200_tx_engine *te, uint32_t nbytes, unsigned int flags)
{
    if (!te)
	return 0;
    const fsk_b200_tx_plan *p = &te->plan;
    const uint64_t frame = (uint64_t)p->start + (uint64_t)p->n_data_bits * p->bit + p->stop;
    const uint64_t words = (uint64_t)nbytes * (p->encoder == FSK_B200_ENCODE_BAUDOT ? 2u : 1u);
    uint64_t n = 0;
    if (nbytes)					/* leader, preamble and the frames (:202-228) */
	n = (uint64_t)p->leader * p->bit + (p->nsync + words) * frame;
    if ((flags & FSK_B200_TX_IDLE_IF_EMPTY) && n < p->idle)	/* or the idle tone of an empty row */
	n = p->idle;
    if (flags & FSK_B200_TX_FINAL)
	n += (uint64_t)p->trailer * p->bit;
    return n > 0xffffffffu ? 0 : n;
}

int fsk_b200_tx_text_batch(fsk_b200_tx_engine *te, const uint8_t *text, size_t nstreams, size_t text_stride,
	const uint32_t *text_len, unsigned int flags, fsk_b200_tx_state *states, void *out, size_t out_stride,
	uint32_t *out_len, void *stream)
{
    if (!te || !text || !text_len || !states || !out || !out_len) {
	fsk_b200_set_error("tx_text_batch: NULL argument");
	return -EINVAL;
    }
    if (flags & ~(FSK_B200_TX_IDLE_IF_EMPTY | FSK_B200_TX_FINAL)) {
	fsk_b200_set_error("tx_text_batch: unknown flags 0x%x", flags);
	return -EINVAL;
    }
    const uint64_t need = fsk_b200_tx_max_samples(te, text_stride > 0xffffffffu ? 0xffffffffu : (uint32_t)text_stride,
	    flags);
    if (text_stride > 0xffffffffu || (need == 0 && text_stride > 0) || out_stride < need) {
	fsk_b200_set_error("tx_text_batch: out_stride %zu is below the %llu samples a row of %zu bytes can need",
		out_stride, (unsigned long long)need, text_stride);
	return -EINVAL;
    }
    fsk_b200_tx_io io;
    memset(&io, 0, sizeof(io));
    io.text = text;
    io.text_stride = text_stride;
    io.text_len = text_len;
    io.states = states;
    io.out = out;
    io.out_stride = out_stride;
    io.out_len = out_len;
    io.flags = flags;
    io.nstreams = nstreams;
    return fsk_b200_cuda_tx_synth(&te->plan, te->d_lut, &io, stream);
}

/* ------------------------------------------------------------------------ */
/* drop-in for src/fsk.h                                                    */
/* ------------------------------------------------------------------------ */

fsk_plan *fsk_plan_new(float sample_rate, float f_mark, float f_space, float filter_bw)
{
    fsk_plan *fskp = malloc(sizeof(fsk_plan));
    if (!fskp)
	return NULL;
    memset(fskp, 0, sizeof(*fskp));
    fskp->sample_rate = sample_rate;
    fskp->f_mark = f_mark;
    fskp->f_space = f_space;
    fskp->band_width = filter_bw;		/* like the reference, filter_bw itself stays unset */
    if (derive_bands(sample_rate, f_mark, f_space, filter_bw, &fskp->fftsize, &fskp->nbands,
		&fskp->b_mark, &fskp->b_space) != 0) {
	fprintf(stderr, "b_mark=%u or b_space=%u is invalid (nbands=%u)\n",
		fskp->b_mark, fskp->b_space, fskp->nbands);
	free(fskp);
	errno = EINVAL;
	return NULL;
    }
    if (!fsk_b200_cuda_device_ok() || !(fskp->engine = fsk_b200_cuda_engine_new())) {
	fprintf(stderr, "fsk_plan_new: no usable CUDA device\n");
	free(fskp);
	errno = EINVAL;
	return NULL;
    }
    return fskp;
}

void fsk_plan_destroy(fsk_plan *fskp)
{
    if (!fskp)
	return;
    fsk_b200_cuda_engine_destroy(fskp->engine);
    free(fskp);
}

float fsk_find_frame(fsk_plan *fskp, float *samples, unsigned int frame_nsamples,
	unsigned int try_first_sample, unsigned int try_max_nsamples,
	unsigned int try_step_nsamples, float try_confidence_search_limit,
	const char *expect_bits_string, unsigned long long *bits_outp, float *ampl_outp,
	unsigned int *frame_start_outp)
{
    fsk_b200_geom g;
    assert(strlen(expect_bits_string) <= 64);		/* src/fsk.c:463 */
    int rc = fsk_b200_geom_from(frame_nsamples, expect_bits_string, NULL, &g);
    assert(rc == 0);					/* src/fsk.c:202 */
    (void)rc;
    /* the widest read of the reference: candidates t < try_max, each touching
     * [t, t + span) (src/fsk.c:477-502, :204-206) */
    unsigned int nfloats = try_max_nsamples ? try_max_nsamples - 1 + g.span : 0;
    fsk_b200_frame out;
    memset(&out, 0, sizeof(out));
    if (nfloats && fsk_b200_cuda_set_table(fskp->engine, fskp->fftsize, fskp->b_mark,
		fskp->b_space, g.bit_nsamples) == 0)
	rc = fsk_b200_cuda_find_frame_one(fskp->engine, &g, samples, nfloats, try_first_sample,
		try_max_nsamples, try_step_nsamples, try_confidence_search_limit, &out);
    else
	rc = nfloats ? -1 : 0;
    if (rc != 0) {
	fprintf(stderr, "fsk_find_frame: CUDA engine failure: %s\n", fsk_b200_last_error());
	abort();			/* the reference has no error return here either */
    }
    *bits_outp = ((unsigned long long)out.bits_hi << 32) | out.bits_lo;
    *ampl_outp = out.amplitude;
    *frame_start_outp = out.frame_start;
    return out.confidence;
}

int fsk_detect_carrier(fsk_plan *fskp, float *samples, unsigned int nsamples,
	float min_mag_threshold)
{
    assert(nsamples <= (unsigned int)fskp->fftsize);	/* src/fsk.c:547 */
    float *mags = malloc(sizeof(float) * fskp->nbands);
    if (!mags)
	return -1;
    if (fsk_b200_cuda_band_mags(fskp->engine, fskp->fftsize, samples, nsamples, fskp->nbands,
		mags) != 0) {
	fprintf(stderr, "fsk_detect_carrier: CUDA engine failure: %s\n", fsk_b200_last_error());
	abort();
    }
    /* the pick itself: first band, from 1 up, with the strictly largest magnitude
     * among those >= the threshold (src/fsk.c:554-580) */
    float max_mag = 0.0f;
    int best = -1;
    for (unsigned int i = 1; i < fskp->nbands; i++) {
	if (mags[i] < min_mag_threshold)
	    continue;
	if (max_mag < mags[i]) {
	    max_mag = mags[i];
	    best = (int)i;
	}
    }
    free(mags);
    return best;
}

int fsk_b200_detect_carrier_batch(int fftsize, const float *samples, size_t nstreams, size_t stride,
	const uint32_t *offset, uint32_t nsamples, float min_mag_threshold, int32_t *out_band, void *stream)
{
    if (!samples || !out_band || fftsize < 2) {
	fsk_b200_set_error("detect_carrier_batch: NULL argument");
	return -EINVAL;
    }
    if (nsamples == 0 || nsamples > (uint32_t)fftsize) {	/* the assert of src/fsk.c:547 */
	fsk_b200_set_error("detect_carrier_batch: nsamples %u outside 1..fftsize %d", nsamples, fftsize);
	return -EINVAL;
    }
    if (!fsk_b200_cuda_device_ok()) {
	fsk_b200_set_error("no usable CUDA device (there is no CPU fallback)");
	return -ENODEV;
    }
    return fsk_b200_cuda_detect_carrier_batch(fftsize, samples, nstreams, stride, offset, nsamples,
	    min_mag_threshold, out_band, stream);
}

void fsk_set_tones_by_bandshift(fsk_plan *fskp, unsigned int b_mark, int b_shift)
{
    assert(b_shift != 0);				/* src/fsk.c:587-592 */
    assert(b_mark < fskp->nbands);
    int b_space = (int)b_mark + b_shift;
    assert(b_space >= 0);
    assert(b_space < (int)fskp->nbands);
    fskp->b_mark = b_mark;
    fskp->b_space = b_space;
    fskp->f_mark = b_mark * fskp->band_width;
    fskp->f_space = b_space * fskp->band_width;
}
