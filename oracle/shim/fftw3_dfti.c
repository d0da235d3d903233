/*
 * fftw3_dfti.c -- TEST INFRASTRUCTURE: the fftw3.h stand-in backed by MKL's DFTI, the
 * single-precision SIMD FFT that ships inside PyTorch's libtorch_cpu.so in this image.
 *
 * Why a second stand-in: the reference's speed on a CPU is the speed of its FFT library.  The
 * portable shim (fftw3_shim.c) is a scalar mixed-radix transform, several times slower than
 * FFTW's SIMD codelets; timing the reference with it would flatter the GPU.  MKL's DFTI is the
 * closest thing to FFTW that exists here (it is NOT FFTW), so the CPU arms of
 * bench.py time the unmodified src/fsk.c on this one when it loads (oracle/_ref/libfsk_ref_dfti.so)
 * and say so in their `sample` string.  Parity never depends on it: the golden vectors were
 * minted with the portable shim, and tests/test_oracle_vs_ref.py holds the two against each other.
 *
 * No MKL header exists in the image; the five entry points and the constants below are the
 * public DFTI ABI (mkl_dfti.h), declared by hand.
 */
#include <stdlib.h>
#include <string.h>

#include "fftw3.h"

typedef struct DFTI_DESCRIPTOR *DFTI_DESCRIPTOR_HANDLE;
extern long DftiCreateDescriptor_s_1d(DFTI_DESCRIPTOR_HANDLE *, int domain, long n);
extern long DftiSetValue(DFTI_DESCRIPTOR_HANDLE, int param, ...);
extern long DftiCommitDescriptor(DFTI_DESCRIPTOR_HANDLE);
extern long DftiComputeForward(DFTI_DESCRIPTOR_HANDLE, void *in, ...);
extern long DftiFreeDescriptor(DFTI_DESCRIPTOR_HANDLE *);

enum {
    DFTI_CONJUGATE_EVEN_STORAGE = 10, DFTI_PLACEMENT = 11, DFTI_REAL = 33, DFTI_COMPLEX_COMPLEX = 39,
    DFTI_NOT_INPLACE = 44
};

struct oracle_fftwf_plan_s {
    DFTI_DESCRIPTOR_HANDLE h;
    float *in;
    fftwf_complex *out;
};

void *fftwf_malloc(size_t n)
{
    void *p = NULL;
    n = (n + 127) & ~(size_t)127;
    return posix_memalign(&p, 128, n ? n : 128) == 0 ? p : NULL;
}

void fftwf_free(void *p) { free(p); }

fftwf_plan fftwf_plan_many_dft_r2c(int rank, const int *n, int howmany,
	float *in, const int *inembed, int istride, int idist,
	fftwf_complex *out, const int *onembed, int ostride, int odist,
	unsigned flags)
{
    (void)inembed; (void)onembed; (void)idist; (void)odist; (void)flags;
    if (rank != 1 || howmany != 1 || istride != 1 || ostride != 1 || n[0] < 1)
	return NULL;
    struct oracle_fftwf_plan_s *pl = calloc(1, sizeof(*pl));
    if (!pl)
	return NULL;
    pl->in = in;
    pl->out = out;
    if (DftiCreateDescriptor_s_1d(&pl->h, DFTI_REAL, (long)n[0]) != 0
	    || DftiSetValue(pl->h, DFTI_PLACEMENT, DFTI_NOT_INPLACE) != 0
	    || DftiSetValue(pl->h, DFTI_CONJUGATE_EVEN_STORAGE, DFTI_COMPLEX_COMPLEX) != 0
	    || DftiCommitDescriptor(pl->h) != 0) {
	if (pl->h)
	    DftiFreeDescriptor(&pl->h);
	free(pl);
	return NULL;
    }
    return pl;
}

void fftwf_execute(const fftwf_plan pl) { DftiComputeForward(pl->h, pl->in, pl->out); }

void fftwf_destroy_plan(fftwf_plan pl)
{
    if (!pl)
	return;
    DftiFreeDescriptor(&pl->h);
    free(pl);
}
