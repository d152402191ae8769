// crt_ptx.cuh -- every line of inline PTX the kernels use, in one place: shared-memory addresses, mbarriers,
// 1-D bulk copies (TMA) in both directions, per-lane asynchronous 16-byte copies, shared loads at absolute
// addresses.  (tests/simt/ substitutes this one header to execute the unchanged kernels on a CPU for debugging;
// nothing in the product includes or links that.)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace crt {

// ---------------------------------------------------------------------------------------
// TMA (1-D bulk copy) + mbarrier primitives
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// global -> shared bulk copy; dst, src and bytes must all be multiples of 16
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, unsigned bytes, uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// 16-byte asynchronous copies global -> shared issued per lane (LDGSTS): the right tool when every lane
// fetches its own small span -- a per-lane bulk copy is a warp-serial instruction (one issue per lane)
__device__ __forceinline__ void cp_async_16(void *dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int PENDING> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(PENDING) : "memory"); }

// shared -> global bulk copy (the mirror of tma_load_1d) and its bookkeeping
__device__ __forceinline__ void tma_store_1d(void *dst, const void *src, unsigned bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int PENDING> __device__ __forceinline__ void tma_store_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(PENDING) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared-memory accesses at 32-bit shared-space ADDRESSES (+ constant byte offset) and global 16-byte accesses by
// explicit state space: the hot loops of k_lines2 keep absolute shared addresses in registers, so no generic-to-shared
// conversion or 64-bit pointer arithmetic is ever re-derived inside them, and images reached through pointers that were
// loaded from memory (generic as far as the compiler knows) are still written with st.global.
template <int OFF = 0> __device__ __forceinline__ uint4 lds_u4(unsigned addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4+%5];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr), "n"(OFF));
    return v;
}
template <int OFF = 0> __device__ __forceinline__ uint2 lds_u2(unsigned addr)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2+%3];" : "=r"(v.x), "=r"(v.y) : "r"(addr), "n"(OFF));
    return v;
}
template <int OFF = 0> __device__ __forceinline__ unsigned lds_u1(unsigned addr)
{
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
    return v;
}
template <int OFF = 0> __device__ __forceinline__ void sts_u1(unsigned addr, unsigned v)
{
    asm volatile("st.shared.u32 [%0+%1], %2;" ::"r"(addr), "n"(OFF), "r"(v) : "memory");
}
template <int OFF = 0> __device__ __forceinline__ void sts_u2(unsigned addr, uint2 v)
{
    asm volatile("st.shared.v2.u32 [%0+%1], {%2, %3};" ::"r"(addr), "n"(OFF), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void stg_u4(void *p, uint4 v)
{
    asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// 16-byte asynchronous copy global -> shared with the shared side given as an address
__device__ __forceinline__ void cp_async_16a(unsigned dst_addr, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_addr), "l"(src) : "memory");
}

// Two-way dot product of 16-bit by 8-bit values with 32-bit accumulate (IDP.2A): a holds two 16-bit values (signed when
// SIGNED_A, else unsigned), b four unsigned bytes of which the low (HI = false: bytes 0, 1) or the high pair (bytes 2, 3)
// takes part:  c + a.h0 * b.byte[0 | 2] + a.h1 * b.byte[1 | 3]  (mod 2^32).
template <bool HI, bool SIGNED_A> __device__ __forceinline__ int dp2a_u8(unsigned a, unsigned b, int c)
{
    int d;
    if (HI) {
        if (SIGNED_A) asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
        else asm("dp2a.hi.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    } else {
        if (SIGNED_A) asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
        else asm("dp2a.lo.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    }
    return d;
}

// Debug builds only (-DCRTX_PHASE_CLOCKS=1, `make custom`): thread `who` of every CTA stamps the SM's cycle counter at the
// phase boundaries of a kernel, and crtx_debug_clocks() (crtx.cu) hands the table to tools/phase_clocks.py.  Compiled out otherwise.
#if defined(CRTX_PHASE_CLOCKS) && CRTX_PHASE_CLOCKS
constexpr int kClkCtas = 512, kClkPhases = 16;
static __device__ unsigned long long g_phase_clk[4][kClkCtas][kClkPhases]; // [kernel][CTA][phase]
__device__ __forceinline__ void phase_mark(int kernel, int phase, int who = 0)
{
    if ((int) threadIdx.x == who) {
        const int cta = (int) (blockIdx.x + blockIdx.y * gridDim.x);
        if (cta < kClkCtas) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            // phase 0 = start, phase 14 = end: wall clock (ns) for the skew between CTAs, with the cycle counter beside it
            g_phase_clk[kernel][cta][phase] = (phase == 0 || phase == 14) ? t : (unsigned long long) clock64();
            if (phase == 0 || phase == 14) g_phase_clk[kernel][cta][phase == 0 ? 15 : 13] = (unsigned long long) clock64();
        }
    }
}
#else
__device__ __forceinline__ void phase_mark(int, int, int = 0) {}
#endif

// Row element at a shared-memory ADDRESS (+ constant byte offset), sign-extended.  The resampler keeps
// absolute shared addresses in registers; going through ld.shared directly keeps the address arithmetic
// out of the pixel loop (a generic pointer would be re-derived from the shared window base every time).
template <typename Elem, int OFF> __device__ __forceinline__ int lds_elem(unsigned addr)
{
    int v;
    if (sizeof(Elem) == 2) asm volatile("ld.shared.s16 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
    else asm volatile("ld.shared.s32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
    return v;
}

} // namespace crt
