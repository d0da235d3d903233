/*
 * tests/emu/cuda_runtime.h -- TEST INFRASTRUCTURE: a host stand-in for the CUDA language
 * extensions and the few runtime calls that minimodem_b200/csrc/fsk_b200_kernels.cu uses, so
 * that the product's kernel SOURCE can be compiled by g++ and run on CPU cores under a small
 * SIMT emulator (tests/emu/Makefile -> tests/emu/libfsk_b200_emu.so).
 *
 * Why: the build container has no GPU.  With this, the parity tests that normally need an H100
 * (tests/test_gpu_parity.py) can exercise the kernels' control flow, ring bookkeeping, lane
 * exchanges and record formats on the CPU before GPU minutes are spent.  It is NOT a product
 * path: nothing in minimodem_b200/ loads it, the library it builds is only ever selected by the
 * tests through FSK_B200_LIB, and it is orders of magnitude slower than the oracle.
 *
 * What it emulates
 *   - one thread block = one OS thread running blockDim.x fibers (ucontext), round-robin;
 *     blocks of a grid are spread over a few OS threads;
 *   - __syncthreads / __syncwarp / __shfl_xor_sync / __any_sync / __ballot_sync as rendezvous
 *     among exactly the lanes named by the mask (a lane that never arrives = reported deadlock);
 *   - dynamic shared memory as a per-block buffer; "shared addresses" are byte offsets into it;
 *   - cp.async: copies are queued per lane and land when that lane executes the matching
 *     wait_group (FSK_EMU_ASYNC=late, the default: a missing wait reads stale data) or at once
 *     (FSK_EMU_ASYNC=eager: a copy issued while its target is still being read corrupts it);
 *   - sqrt.approx / div.approx as IEEE sqrtf and division (the GPU's are <= 2 ulp away);
 *     FSK_EMU_ULP=n perturbs both by up to n ulp to show that no test hinges on their rounding.
 * What it does not: timing, bank conflicts, memory coalescing, the TMA/mbarrier variant.
 */
#ifndef FSK_EMU_CUDA_RUNTIME_H
#define FSK_EMU_CUDA_RUNTIME_H

#ifndef FSK_EMU
#define FSK_EMU 1
#endif

#include <ucontext.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <type_traits>
#include <vector>

/* ---- language ------------------------------------------------------------------------- */
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __grid_constant__

struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
struct int4 { int x, y, z, w; };
struct uint3 { unsigned x, y, z; };
static inline float2 make_float2(float x, float y) { float2 r = { x, y }; return r; }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = { x, y, z, w }; return r; }

template <class A, class B>
static inline typename std::common_type<A, B>::type min(A a, B b)
{
    typedef typename std::common_type<A, B>::type T;
    return (T)a < (T)b ? (T)a : (T)b;
}
template <class A, class B>
static inline typename std::common_type<A, B>::type max(A a, B b)
{
    typedef typename std::common_type<A, B>::type T;
    return (T)a < (T)b ? (T)b : (T)a;
}

/* ---- the emulator ----------------------------------------------------------------------- */
namespace emu {

struct Pending { unsigned dst; unsigned char data[16]; };

struct Lane {
    ucontext_t ctx;
    bool done;
    /* cp.async: copies of the open group, and the sizes of the committed groups still in flight */
    std::vector<Pending> queue;
    std::vector<unsigned> groups;
};

struct Slot { unsigned mask; unsigned count; unsigned long gen; };

struct Block {
    uint3 bidx, bdim, gdim;
    unsigned char *smem;
    size_t smem_bytes;
    std::vector<Lane> lanes;
    std::vector<uint64_t> xchg;		/* one exchange word per lane */
    std::vector<std::vector<Slot> > slots;	/* per warp: one rendezvous per distinct mask */
    Slot all;				/* __syncthreads */
    ucontext_t sched;
    unsigned cur;
    unsigned long progress;
    const void *body;			/* the launch lambda */
    void (*call)(const void *);
};

extern thread_local Block *blk;
extern int async_eager;

static inline uint3 tidx() { uint3 r = { blk->cur, 0, 0 }; return r; }

static inline void yield() { swapcontext(&blk->lanes[blk->cur].ctx, &blk->sched); }

[[noreturn]] void die(const char *what);

static inline void wait_on(Slot &s, unsigned need)
{
    Block *b = blk;
    const unsigned long g = s.gen;
    b->progress++;
    if (++s.count == need) {
	s.count = 0;
	s.gen++;
	return;
    }
    while (s.gen == g)
	yield();
}

static inline void rendezvous(unsigned mask)
{
    Block *b = blk;
    const unsigned warp = b->cur >> 5;
    const unsigned lanes_here = std::min(32u, b->bdim.x - warp * 32u);
    if (lanes_here < 32u)
	mask &= (1u << lanes_here) - 1u;
    if (!(mask >> (b->cur & 31) & 1u))
	die("a lane took part in a *_sync whose mask does not name it");
    std::vector<Slot> &v = b->slots[warp];
    size_t i = 0;
    for (; i < v.size(); i++)
	if (v[i].mask == mask)
	    break;
    if (i == v.size()) {
	/* waiting lanes hold references into v: it is reserved up front and must never grow past that */
	if (v.size() == v.capacity())
	    die("too many distinct *_sync masks in one warp");
	/* masks of one kernel never overlap partially (groups of a warp, or the whole warp) */
	for (size_t j = 0; j < v.size(); j++)
	    if ((v[j].mask & mask) && v[j].count)
		die("overlapping *_sync masks in flight");
	Slot s = { mask, 0, 0 };
	v.push_back(s);
    }
    wait_on(v[i], (unsigned)__builtin_popcount(mask));
}

template <class T>
static inline T shfl_xor(unsigned mask, T v, int o)
{
    static_assert(sizeof(T) <= 8, "shuffle width");
    Block *b = blk;
    uint64_t bits = 0;
    memcpy(&bits, &v, sizeof(T));
    b->xchg[b->cur] = bits;
    rendezvous(mask);
    const unsigned src = b->cur ^ (unsigned)o;
    T r = v;
    if (src < b->bdim.x) {
	bits = b->xchg[src];
	memcpy(&r, &bits, sizeof(T));
    }
    rendezvous(mask);
    return r;
}

/* __shfl_sync(mask, v, srcLane, width): the source is lane (srcLane mod width) of the caller's
 * width-wide segment of the warp */
template <class T>
static inline T shfl_idx(unsigned mask, T v, int src_lane, int width)
{
    static_assert(sizeof(T) <= 8, "shuffle width");
    Block *b = blk;
    uint64_t bits = 0;
    memcpy(&bits, &v, sizeof(T));
    b->xchg[b->cur] = bits;
    rendezvous(mask);
    const unsigned lane = b->cur & 31u, w = (unsigned)width;
    const unsigned src = (b->cur & ~31u) + (lane & ~(w - 1u)) + ((unsigned)src_lane & (w - 1u));
    T r = v;
    if (src < b->bdim.x) {
	if (!((mask >> (src & 31u)) & 1u))
	    die("__shfl_sync: source lane is not in the mask");
	bits = b->xchg[src];
	memcpy(&r, &bits, sizeof(T));
    }
    rendezvous(mask);
    return r;
}

static inline unsigned ballot(unsigned mask, int pred)
{
    Block *b = blk;
    b->xchg[b->cur] = pred ? 1u : 0u;
    rendezvous(mask);
    unsigned r = 0;
    const unsigned base = b->cur & ~31u;
    for (unsigned l = 0; l < 32u && base + l < b->bdim.x; l++)
	if ((mask >> l & 1u) && b->xchg[base + l])
	    r |= 1u << l;
    rendezvous(mask);
    return r;
}

/* __reduce_max_sync (redux.sync.max.u32): the largest value among the lanes of the mask */
static inline unsigned reduce_max(unsigned mask, unsigned v)
{
    Block *b = blk;
    b->xchg[b->cur] = v;
    rendezvous(mask);
    unsigned r = 0;
    const unsigned base = b->cur & ~31u;
    for (unsigned l = 0; l < 32u && base + l < b->bdim.x; l++)
	if ((mask >> l & 1u) && (unsigned)b->xchg[base + l] > r)
	    r = (unsigned)b->xchg[base + l];
    rendezvous(mask);
    return r;
}

/* cp.async */
static inline void land(const Pending &p)
{
    Block *b = blk;
    if ((size_t)p.dst + 16 > b->smem_bytes)
	die("cp.async destination outside the block's shared memory");
    memcpy(b->smem + p.dst, p.data, 16);
}

static inline void cp_async_16(unsigned dst, const void *src, unsigned valid)
{
    Pending p;
    p.dst = dst;
    if (dst & 15u)
	die("cp.async destination not 16-byte aligned");
    if (valid && ((uintptr_t)src & 15u))
	die("cp.async source not 16-byte aligned");
    memset(p.data, 0, 16);
    if (valid)
	memcpy(p.data, src, valid > 16 ? 16 : valid);
    if (async_eager)
	land(p);
    else
	blk->lanes[blk->cur].queue.push_back(p);
}

static inline void cp_async_commit_group()
{
    Lane &l = blk->lanes[blk->cur];
    unsigned open = (unsigned)l.queue.size();
    for (size_t i = 0; i < l.groups.size(); i++)
	open -= l.groups[i];
    l.groups.push_back(open);
}

static inline void cp_async_wait_group(unsigned keep)
{
    Lane &l = blk->lanes[blk->cur];
    while (l.groups.size() > keep) {
	const unsigned n = l.groups.front();
	for (unsigned i = 0; i < n; i++)
	    land(l.queue[i]);
	l.queue.erase(l.queue.begin(), l.queue.begin() + n);
	l.groups.erase(l.groups.begin());
    }
}

void run_grid(unsigned grid, unsigned block, size_t smem, const void *body, void (*call)(const void *));

template <class F>
static void call_body(const void *p) { (*static_cast<const F *>(p))(); }

template <class F>
static inline void launch(unsigned grid, unsigned block, size_t smem, const F &f)
{
    run_grid(grid, block, smem, &f, &call_body<F>);
}

}  /* namespace emu */

#define threadIdx (emu::tidx())
#define blockIdx (emu::blk->bidx)
#define blockDim (emu::blk->bdim)
#define gridDim (emu::blk->gdim)

#define FSK_LAUNCH(kernel, grid, block, smem, stream, ...) \
    emu::launch((unsigned)(grid), (unsigned)(block), (size_t)(smem), [=] { kernel(__VA_ARGS__); })
#define FSK_DYN_SMEM(name) float4 *name = reinterpret_cast<float4 *>(emu::blk->smem)

/* ---- intrinsics --------------------------------------------------------------------------- */
static inline void __syncthreads() { emu::wait_on(emu::blk->all, emu::blk->bdim.x); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::rendezvous(mask); }
template <class T>
static inline T __shfl_xor_sync(unsigned mask, T v, int o) { return emu::shfl_xor(mask, v, o); }
template <class T>
static inline T __shfl_sync(unsigned mask, T v, int src_lane, int width = 32) { return emu::shfl_idx(mask, v, src_lane, width); }
static inline int __any_sync(unsigned mask, int pred) { return emu::ballot(mask, pred) != 0u; }
static inline unsigned __ballot_sync(unsigned mask, int pred) { return emu::ballot(mask, pred); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) { return emu::reduce_max(mask, v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
template <class T>
static inline T __ldg(const T *p) { return *p; }
static inline void __trap() { emu::die("__trap()"); }
static inline void sincospif(float x, float *s, float *c)
{
    *s = (float)sin(M_PI * (double)x);
    *c = (float)cos(M_PI * (double)x);
}
static inline size_t __cvta_generic_to_shared(const void *p)
{
    return (size_t)((const unsigned char *)p - emu::blk->smem);
}
static inline void *__cvta_shared_to_generic(size_t a) { return emu::blk->smem + a; }

/* the inline-PTX wrappers of fsk_b200_device.cuh (guarded there by FSK_EMU) */
/* FSK_EMU_ULP=n: perturb the two approximate units by up to n ulp (pseudo-randomly, either way), to
 * see that no test hinges on their exact rounding -- the GPU's sqrt.approx / div.approx are within
 * 2 ulp of these */
namespace emu {
extern int approx_ulp;
static inline float jitter(float v)
{
    if (approx_ulp <= 0 || !std::isfinite(v) || v == 0.0f)
	return v;
    /* a fixed function of the value, like a hardware unit: the same operand gives the same result */
    int32_t bits;
    memcpy(&bits, &v, 4);
    uint32_t h = (uint32_t)bits * 2654435761u;
    h ^= h >> 15;
    h *= 2246822519u;
    h ^= h >> 13;
    const int k = (int)(h % (2u * (unsigned)approx_ulp + 1u)) - approx_ulp;
    bits += v > 0 ? k : -k;
    float r;
    memcpy(&r, &bits, 4);
    return std::isfinite(r) ? r : v;
}
}
static inline float fast_sqrt(float x) { return emu::jitter(sqrtf(x)); }
static inline float fast_div(float a, float b) { return emu::jitter(a / b); }
static inline void cp_async_commit() { emu::cp_async_commit_group(); }
template <int NKEEP>
static inline void cp_async_wait() { emu::cp_async_wait_group(NKEEP); }
static inline void ldgsts16(unsigned dst, const float *src) { emu::cp_async_16(dst, src, 16); }
static inline void ldgsts16_zfill(unsigned dst, const float *src, unsigned valid) { emu::cp_async_16(dst, src, valid); }
/* the TMA/mbarrier fill of the prefix-table kernel (FSK_B200_PFX_FILL=1) is not emulated */
static inline void mbar_init(unsigned, unsigned) { emu::die("mbarrier path is not emulated"); }
static inline void mbar_fence_init() {}
static inline void mbar_arrive_expect_tx(unsigned, unsigned) { emu::die("mbarrier path is not emulated"); }
static inline bool mbar_try_wait(unsigned, unsigned) { emu::die("mbarrier path is not emulated"); }
static inline void bulk_g2s(unsigned, const void *, unsigned, unsigned) { emu::die("bulk copy is not emulated"); }

/* ---- runtime API ---------------------------------------------------------------------------- */
typedef int cudaError_t;
typedef void *cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };
enum { cudaStreamNonBlocking = 1 };

static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated failure"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize(void) { return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int *v, int attr, int)
{
    /* the H100 figures the launch-shape logic is written for */
    *v = attr == cudaDevAttrMultiProcessorCount ? 132 : 232448;
    return cudaSuccess;
}
template <class T>
static inline cudaError_t cudaMalloc(T **p, size_t n)
{
    void *q = NULL;
    if (posix_memalign(&q, 256, n ? n : 256) != 0)
	return cudaErrorMemoryAllocation;
    memset(q, 0xA5, n);			/* device memory is not zero */
    *p = (T *)q;
    return cudaSuccess;
}
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = 0)
{
    memcpy(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = NULL; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
typedef void *cudaEvent_t;
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = NULL; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
template <class F>
static inline cudaError_t cudaFuncSetAttribute(F, int, int v) { return v <= 232448 ? cudaSuccess : cudaErrorInvalidValue; }

#endif
