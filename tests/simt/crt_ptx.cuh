// tests/simt/crt_ptx.cuh -- TEST INFRASTRUCTURE: the CPU stand-in for ntsc-crt_b200/csrc/crt_ptx.cuh (same
// functions, no PTX), used only by the SIMT interpreter build (tests/simt/build.py).
//
// Asynchronous copies are performed at the LATEST moment the hardware could perform them, which is the
// schedule most likely to expose a missing wait or a buffer reused too early:
//   * bulk loads (global -> shared, mbarrier-tracked) happen when somebody waits on their mbarrier;
//   * per-lane cp.async copies happen in cp_async_wait;
//   * bulk stores (shared -> global) read their shared source in tma_store_wait_read (or at thread exit).
// Alignment / size rules of the real instructions (16-byte granularity) are checked.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace simt {
void ptx_fail(const char *what);
void mbar_init(uint64_t *bar, unsigned count);
void mbar_expect_tx(uint64_t *bar, unsigned bytes);
void mbar_wait(uint64_t *bar, unsigned parity);
void bulk_load(void *dst, const void *src, unsigned bytes, uint64_t *bar);
void lane_copy16(void *dst, const void *src);
void lane_commit();
void lane_wait(int pending);
void bulk_store(void *dst, const void *src, unsigned bytes);
void bulk_store_commit();
void bulk_store_wait_read(int pending);
} // namespace simt

namespace crt {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) { ::simt::mbar_init(bar, count); }
__device__ __forceinline__ void mbar_fence_init() {}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) { ::simt::mbar_expect_tx(bar, bytes); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) { ::simt::mbar_wait(bar, parity); }
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, unsigned bytes, uint64_t *bar)
{
    ::simt::bulk_load(dst, src, bytes, bar);
}
__device__ __forceinline__ void cp_async_16(void *dst, const void *src) { ::simt::lane_copy16(dst, src); }
__device__ __forceinline__ void cp_async_commit() { ::simt::lane_commit(); }
template <int PENDING> __device__ __forceinline__ void cp_async_wait() { ::simt::lane_wait(PENDING); }

__device__ __forceinline__ void tma_store_1d(void *dst, const void *src, unsigned bytes) { ::simt::bulk_store(dst, src, bytes); }
__device__ __forceinline__ void tma_store_commit() { ::simt::bulk_store_commit(); }
template <int PENDING> __device__ __forceinline__ void tma_store_wait_read() { ::simt::bulk_store_wait_read(PENDING); }
__device__ __forceinline__ void fence_async_smem() {}

// explicit-state-space accesses of the real header: plain loads / stores here, with the instructions' alignment rules
template <typename T> __device__ __forceinline__ T *smem_at(unsigned addr, int off, const char *what)
{
    unsigned char *p = ::simt::g_smem_anchor + (int) (addr + (unsigned) off);
    if ((uintptr_t) p % sizeof(T)) ::simt::ptx_fail(what);
    return reinterpret_cast<T *>(p);
}
template <int OFF = 0> __device__ __forceinline__ uint4 lds_u4(unsigned addr) { return *smem_at<uint4>(addr, OFF, "ld.shared.v4: misaligned address"); }
template <int OFF = 0> __device__ __forceinline__ uint2 lds_u2(unsigned addr) { return *smem_at<uint2>(addr, OFF, "ld.shared.v2: misaligned address"); }
template <int OFF = 0> __device__ __forceinline__ unsigned lds_u1(unsigned addr) { return *smem_at<unsigned>(addr, OFF, "ld.shared.u32: misaligned address"); }
template <int OFF = 0> __device__ __forceinline__ void sts_u1(unsigned addr, unsigned v) { *smem_at<unsigned>(addr, OFF, "st.shared.u32: misaligned address") = v; }
template <int OFF = 0> __device__ __forceinline__ void sts_u2(unsigned addr, uint2 v) { *smem_at<uint2>(addr, OFF, "st.shared.v2: misaligned address") = v; }
__device__ __forceinline__ void stg_u4(void *p, uint4 v)
{
    if ((uintptr_t) p % 16) ::simt::ptx_fail("st.global.v4: misaligned address");
    *reinterpret_cast<uint4 *>(p) = v;
}
__device__ __forceinline__ void cp_async_16a(unsigned dst_addr, const void *src)
{
    ::simt::lane_copy16(::simt::g_smem_anchor + (int) dst_addr, src);
}

template <bool HI, bool SIGNED_A> __device__ __forceinline__ int dp2a_u8(unsigned a, unsigned b, int c)
{
    const unsigned b0 = (b >> (HI ? 16 : 0)) & 0xffu, b1 = (b >> (HI ? 24 : 8)) & 0xffu;
    const unsigned h0 = SIGNED_A ? (unsigned) (int) (short) (a & 0xffffu) : (a & 0xffffu);
    const unsigned h1 = SIGNED_A ? (unsigned) (int) (short) (a >> 16) : (a >> 16);
    return (int) ((unsigned) c + h0 * b0 + h1 * b1);
}

__device__ __forceinline__ void phase_mark(int, int, int = 0) {}

template <typename Elem, int OFF> __device__ __forceinline__ int lds_elem(unsigned addr)
{
    const unsigned char *p = ::simt::g_smem_anchor + (int) (addr + (unsigned) OFF); // offsets may be "negative"
    if ((uintptr_t) p % sizeof(Elem)) ::simt::ptx_fail("ld.shared: misaligned address");
    return (int) *reinterpret_cast<const Elem *>(p);
}

} // namespace crt
