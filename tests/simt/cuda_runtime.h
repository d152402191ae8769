/* tests/simt/cuda_runtime.h -- TEST INFRASTRUCTURE, not product code.
 *
 * A small SIMT interpreter: just enough of the CUDA language and runtime surface for the product's
 * kernel sources (ntsc-crt_b200/csrc/*.cu, *.cuh, compiled UNCHANGED by g++ through tests/simt/build.py) to
 * execute on a CPU, thread by thread, so that kernel logic can be debugged and checked against the oracle in a
 * container that has no GPU.  Every CUDA thread of a block is a fiber; __syncthreads / __syncwarp / shuffles /
 * ballots / mbarrier waits are scheduling points; bulk copies are deferred to the latest moment the hardware
 * could perform them (see crt_ptx.cuh beside this file).
 *
 * The product never includes, links or loads anything from this directory (tests/test_product_isolation.py);
 * libraries built from it are called libcrt_simt_<variant>.so, live under tests/simt/_build/ and are only opened
 * by tests/test_simt_*.py.  Nothing measured or shipped runs here.
 */
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <functional>

#define __CUDACC__ 1 /* crt_sys.cuh keys its __host__ / __device__ fall-backs on this */
#define __host__
#define __device__
#define __global__ static
#define __constant__ static const
#define __shared__ static /* one block runs at a time; "extern __shared__" is rewritten by build.py */
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

struct __attribute__((aligned(8))) uint2 { unsigned x, y; };
struct uint3 { unsigned x, y, z; };
struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
static inline uint2 make_uint2(unsigned x, unsigned y) { uint2 v = { x, y }; return v; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 v = { x, y, z, w }; return v; }

namespace simt {

struct Warp;
struct Thread { /* what a running fiber knows about itself */
    uint3 tid, bid;
    dim3 bdim, gdim;
    int lin, lane;
    Warp *warp;
};
extern Thread *g_cur;

void yield_blocked();                 /* give the processor away while waiting for something */
void note_progress();                 /* some thread got past a wait (deadlock detection) */
void block_barrier(int pred, int *any);
const uint64_t *warp_exchange(unsigned mask, uint64_t v); /* all lanes in mask deposit v; returns the 32 slots */
void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()> &body);
extern unsigned char *g_smem_anchor;   /* shared-memory "addresses" are byte offsets from here */
extern long g_launches, g_blocks;

} // namespace simt

#define threadIdx (::simt::g_cur->tid)
#define blockIdx (::simt::g_cur->bid)
#define blockDim (::simt::g_cur->bdim)
#define gridDim (::simt::g_cur->gdim)

/* ---- integer min / max the way CUDA overloads them ---- */
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned min(int a, unsigned b) { return min((unsigned) a, b); }
static inline unsigned min(unsigned a, int b) { return min(a, (unsigned) b); }
static inline unsigned max(int a, unsigned b) { return max((unsigned) a, b); }
static inline unsigned max(unsigned a, int b) { return max(a, (unsigned) b); }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }

/* ---- synchronisation and warp collectives ---- */
static inline void __syncthreads() { ::simt::block_barrier(0, NULL); }
static inline int __syncthreads_or(int pred) { int any = 0; ::simt::block_barrier(pred, &any); return any; }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { (void) ::simt::warp_exchange(mask, 0); }
template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32)
{
    static_assert(sizeof(T) <= 8, "shuffle of up to 8 bytes");
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint64_t *slots = ::simt::warp_exchange(mask, raw);
    const int lane = ::simt::g_cur->lane;
    const int from = (lane & ~(width - 1)) | (src & (width - 1));
    T out;
    memcpy(&out, &slots[from], sizeof(T));
    return out;
}
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32)
{
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint64_t *slots = ::simt::warp_exchange(mask, raw);
    const int lane = ::simt::g_cur->lane;
    int from = lane ^ lanemask;
    if ((from & ~(width - 1)) != (lane & ~(width - 1))) from = lane;
    T out;
    memcpy(&out, &slots[from], sizeof(T));
    return out;
}
template <typename T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32)
{
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint64_t *slots = ::simt::warp_exchange(mask, raw);
    const int lane = ::simt::g_cur->lane;
    int from = lane - (int) delta;
    if (from < (lane & ~(width - 1))) from = lane;
    T out;
    memcpy(&out, &slots[from], sizeof(T));
    return out;
}
static inline unsigned __ballot_sync(unsigned mask, int pred)
{
    const uint64_t *slots = ::simt::warp_exchange(mask, pred ? 1u : 0u);
    unsigned r = 0;
    for (int l = 0; l < 32; l++)
        if (((mask >> l) & 1u) && slots[l] == 1u) r |= 1u << l;
    return r;
}

/* ---- integer intrinsics ---- */
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __vimin_s32_relu(int a, int b) { const int m = a < b ? a : b; return m < 0 ? 0 : m; }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel)
{
    const uint64_t src = (uint64_t) a | ((uint64_t) b << 32);
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned s = (sel >> (4 * i)) & 0xf;
        unsigned byte = (unsigned) (src >> (8 * (s & 7))) & 0xffu;
        if (s & 8) byte = (byte & 0x80u) ? 0xffu : 0u; /* msb replication mode */
        r |= byte << (8 * i);
    }
    return r;
}
static inline unsigned __vmaxs4(unsigned a, unsigned b)
{
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const signed char x = (signed char) (a >> (8 * i)), y = (signed char) (b >> (8 * i));
        r |= ((unsigned) (unsigned char) (x > y ? x : y)) << (8 * i);
    }
    return r;
}
static inline unsigned __vmaxu4(unsigned a, unsigned b)
{
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned x = (a >> (8 * i)) & 0xffu, y = (b >> (8 * i)) & 0xffu;
        r |= (x > y ? x : y) << (8 * i);
    }
    return r;
}
static inline unsigned __vabsss4(unsigned a) /* per-byte |x| with signed saturation (-128 -> 127) */
{
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        int x = (signed char) (a >> (8 * i));
        x = x < 0 ? -x : x;
        if (x > 127) x = 127;
        r |= (unsigned) x << (8 * i);
    }
    return r;
}
template <typename T> static inline T __ldg(const T *p) { return *p; }
template <typename T> static inline T __ldcg(const T *p) { return *p; }
template <typename T> static inline void __stcg(T *p, T v) { *p = v; }
static inline int atomicMax(int *p, int v) { const int old = *p; if (v > old) *p = v; return old; }
static inline int atomicAdd(int *p, int v) { const int old = *p; *p = old + v; return old; }
static inline size_t __cvta_generic_to_shared(const void *p)
{
    return (size_t) ((const unsigned char *) p - ::simt::g_smem_anchor);
}

/* ---- runtime API: device memory is host memory, streams run at once ---- */
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
typedef struct simt_stream *cudaStream_t;
typedef struct simt_event *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2,
                      cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2 };
struct cudaPointerAttributes { int type; int device; void *devicePointer; void *hostPointer; };
struct cudaDeviceProp { char name[256]; int major, minor, multiProcessorCount; };

static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "simt: error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int)
{
    memset(p, 0, sizeof(*p));
    strcpy(p->name, "SIMT interpreter (CPU, tests only)");
    p->major = 9;
    p->minor = 0;
    p->multiProcessorCount = 4; /* small grids: everything runs serially anyway */
    return cudaSuccess;
}
namespace simt { void *dev_alloc(size_t bytes); void dev_free(void *p); }
template <typename T> static inline cudaError_t cudaMalloc(T **p, size_t bytes)
{
    *p = (T *) ::simt::dev_alloc(bytes);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void *p) { ::simt::dev_free(p); return cudaSuccess; }
template <typename T> static inline cudaError_t cudaHostAlloc(T **p, size_t bytes, unsigned)
{
    *p = (T *) ::simt::dev_alloc(bytes);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFreeHost(void *p) { ::simt::dev_free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = 0) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dpitch, const void *s, size_t spitch, size_t width, size_t height, cudaMemcpyKind, cudaStream_t = 0)
{
    for (size_t r = 0; r < height; r++) memmove((char *) d + r * dpitch, (const char *) s + r * spitch, width);
    return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = 0) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = 0; return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = 0; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = 0; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (cudaEvent_t) (uintptr_t) 1; return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.001f; return cudaSuccess; } /* (no clock here: a token value) */
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *p)
{
    memset(a, 0, sizeof(*a));
    /* SIMT_HOST_MAPPED=1: every host buffer counts as page-locked and mapped at its own address (what cudaHostAlloc
     * gives under unified addressing), so that the paths that read / write host images in place can run here */
    const char *e = getenv("SIMT_HOST_MAPPED");
    if (e && *e == '1') {
        a->type = cudaMemoryTypeHost;
        a->devicePointer = const_cast<void *>(p);
        a->hostPointer = const_cast<void *>(p);
        return cudaSuccess;
    }
    return cudaErrorInvalidValue;
}
template <typename F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
