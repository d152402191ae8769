// crt_kernels.cuh -- the sm_90a kernels of the composite modulate -> noise -> demodulate path.
//
// Kernel map (reference lines each one replaces):
//   k_mod_skeleton_rgb  sync / blanking / burst skeleton of all 262 lines  crt_ntsc.c:205-252, 325-329
//   k_mod_picture_rgb   RGB->YIQ, 3 band-limit IIRs, carrier mix -> analog crt_ntsc.c:254-324
//   k_mod_nes           PPU pixels -> square-wave IRE sums                 crt_nes.c:21-61, 81-201
//   k_sync              vsync search, hsync / burst-lock chain, line table crt_core.c:379-479;
//                       LCG noise, analog -> inp                           crt_core.c:346-367
//   k_lines             Y/I/Q equalisers, resample, YIQ->RGB, blend, store crt_core.c:511-664
//
// Everything is int32 fixed point with two's-complement wrap and arithmetic right shift, as the
// compiled reference behaves (SURVEY.md section 5); wrap-sensitive operations go through the
// w*() helpers so the compiler cannot exploit signed-overflow UB.
//
// Parallel shape: the recurrences along a scanline (eqf, iirf) round at every step and cannot be
// scanned, so one LANE carries one scanline (32 lines per warp); anything that is parallel along
// the line (pixel fetch, RGB->YIQ, row stores) runs lane-per-sample on tiles transposed through
// shared memory so that every global access is coalesced.  Scanline windows are staged into
// shared memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier), double buffered.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "crt_sys.cuh"
#include "crtx_batch.h"
#include "crt_records.h"
#include "crt_ptx.cuh"

namespace crt {


__constant__ int c_quarter15[18] = CRT_QUARTER15;

// ---------------------------------------------------------------------------------------
// arithmetic helpers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int wmul(int a, int b) { return (int) ((unsigned) a * (unsigned) b); }
__device__ __forceinline__ int wadd(int a, int b) { return (int) ((unsigned) a + (unsigned) b); }
__device__ __forceinline__ int wsub(int a, int b) { return (int) ((unsigned) a - (unsigned) b); }
__device__ __forceinline__ int posmod(int x, int n) { return ((x % n) + n) % n; }
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
// byte offset of image row `row` (>= 0) at `pitch` (> 0) bytes per row: 64-bit, one 32 x 32 -> 64 multiplication
__device__ __forceinline__ size_t row_offset(int row, int pitch) { return (size_t) (unsigned) row * (unsigned) pitch; }

__device__ __forceinline__ int quarter_d(int a)
{
    int k = (a >> 8) & 0xff, fr = a & 0xff;
    int lo = c_quarter15[k], hi = c_quarter15[k + 1];
    return lo + (((hi - lo) * fr) >> 8);
}

__device__ __forceinline__ void sincos14_d(int &s, int &c, int n) // crt_core.c:42-61
{
    n &= 16383;
    int h = n & 8191;
    if (h >= 4096) {
        c = -quarter_d(h - 4096);
        s = quarter_d(8192 - h);
    } else {
        c = quarter_d(4096 - h);
        s = quarter_d(h);
    }
    if (n >= 8192) {
        c = -c;
        s = -s;
    }
}

__device__ __forceinline__ int warp_scan_incl(int v, int lane)
{
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// byte positions of R, G, B in a pixel of each CRT_PIX_FORMAT (crt_core.h:62-67)
__device__ __forceinline__ void fmt_positions(int f, int &r, int &g, int &b)
{
    switch (f) {
        case CRT_PIX_FORMAT_RGB:  r = 0; g = 1; b = 2; break;
        case CRT_PIX_FORMAT_BGR:  r = 2; g = 1; b = 0; break;
        case CRT_PIX_FORMAT_ARGB: r = 1; g = 2; b = 3; break;
        case CRT_PIX_FORMAT_RGBA: r = 0; g = 1; b = 2; break;
        case CRT_PIX_FORMAT_ABGR: r = 3; g = 2; b = 1; break;
        default:                  r = 2; g = 1; b = 0; break; // BGRA
    }
}

// =======================================================================================
// encoder, RGB systems
// =======================================================================================
#if CRT_B200_BANDLIMITED

// Burst and carrier tables of the encoder, entry x of colour row `row`: sin() >> 10 of
//   NTSC / VHS (crt_ntsc.c:174-188): burst hue + 90x + 33, I hue + 90x, Q hue + 90x - 90 (one row);
//   template   (crt_template.c:166-183): with n = (row + dot_crawl_offset) * 180 + hue + 90x:
//              burst n - 90 + HUE_OFFSET, I n, Q n + Q_OFFSET (rows 0 and 1);
//   PV-1000    (crt_pv1k.c:166-181): with n = (row + dot_crawl_offset) * 144 + hue + 72x (x < 5):
//              burst n - 72, I n, Q n + 90 (rows 0..4).
__device__ __forceinline__ void enc_tables(const SrcCfg &s, int row, int x, int &burst, int &modI, int &modQ)
{
    burst = modI = modQ = 0;
    if (!s.as_color) return;
    int sn, cs;
    if (kIsPv1k) {
        const int step = 360 / 5;
        const int n = (row + s.dot_crawl_offset) * (360 * 2 / kVper) + s.hue + x * step;
        sincos14_d(sn, cs, (n - step) * 8192 / 180);
        burst = sn >> 10;
        sincos14_d(sn, cs, n * 8192 / 180);
        modI = sn >> 10;
        sincos14_d(sn, cs, (n + 90) * 8192 / 180);
        modQ = sn >> 10;
    } else if (kIsTemp) {
        const int step = 360 / 4;
        const int n = (row + s.dot_crawl_offset) * (360 / kVper) + s.hue + x * step;
        sincos14_d(sn, cs, (n - step + (-60)) * 8192 / 180); // HUE_OFFSET, crt_template.h:142
        burst = sn >> 10;
        sincos14_d(sn, cs, n * 8192 / 180);
        modI = sn >> 10;
        sincos14_d(sn, cs, (n + (-90)) * 8192 / 180); // Q_OFFSET, crt_template.h:139
        modQ = sn >> 10;
    } else {
        const int n = s.hue + x * 90;
        sincos14_d(sn, cs, (n + 33) * 8192 / 180);
        burst = sn >> 10;
        sincos14_d(sn, cs, n * 8192 / 180);
        modI = sn >> 10;
        sincos14_d(sn, cs, (n - 90) * 8192 / 180);
        modQ = sn >> 10;
    }
}

// first / last line of the equalising and vertical-sync groups (crt_ntsc.c:214,222; crt_template.h:149-156; the
// PV-1000 has one equalising group and syncs at the bottom of the field, crt_pv1k.c:208,214)
constexpr int kEquAHi = kIsPv1k ? -1 : kIsTemp ? 2 : 3, kEquBLo = 7, kEquBHi = 9;
constexpr int kVsyncLo = kIsPv1k ? 258 : kIsTemp ? 3 : 4, kVsyncHi = kIsPv1k ? 260 : 6;

// Lines above CRT_TOP are written whole, active lines only up to AV_BEG (the rest of an active line belongs to the
// picture pass or keeps its old content).  One warp per line (lines w0, w0 + wstride, ...); every line is a handful of
// constant runs (crt_ntsc.c:205-252), written as warp-wide byte fills -- no per-byte classification.
__device__ __forceinline__ void mod_skeleton_lines(const SrcCfg &s, signed char *analog, const int (*burst)[kCc], int w0,
                                                   int wstride, int lane)
{
    static_assert(kHres % 2 == 0 && kAvBeg % 2 == 0, "pairs");
    const int field = s.field & 1, frame = s.frame & 1;
    const int flip = kRowCarrier ? 0 : (field == frame); // the template system and the PV-1000 have no phase inversion
    const int aberration = s.aberration;
    constexpr int H = kHres;
    for (int n = w0; n < kVres; n += wstride) {
        signed char *line = analog + n * H;
        auto fill = [&](int from, int to, int level) {
            for (int t = from + lane; t < to; t += 32) line[t] = (signed char) level;
        };
        if (n <= kEquAHi || (n >= kEquBLo && n <= kEquBHi)) { // equalising pulses
            fill(0, 4 * H / 100, kSync);
            fill(4 * H / 100, 50 * H / 100, kBlank);
            fill(50 * H / 100, 54 * H / 100, kSync);
            fill(54 * H / 100, H, kBlank);
        } else if (n >= kVsyncLo && n <= kVsyncHi) { // vertical sync
            const int first = (field == 1 ? 4 : 46) * H / 100;
            fill(0, first, kSync);
            fill(first, 50 * H / 100, kBlank);
            fill(50 * H / 100, 96 * H / 100, kSync);
            fill(96 * H / 100, H, kBlank);
        } else { // video line: porch, sync tip, breezeway, burst, back porch (+ blank picture above TOP)
            fill(0, kSyncBeg, kBlank);
            fill(kSyncBeg, kBwBeg, (n < kVres - aberration) ? kSync : kBlank); // crt_ntscvhs.c:234-238
            fill(kBwBeg, kCbBeg, kBlank);
            for (int t = kCbBeg + lane; t < kCbBeg + kBurstLen; t += 32) // crt_ntsc.c:236-246, crt_template.c:236-240
                line[t] = (signed char) ((kBlank + burst[n % kVper][(t + flip * 2) % kCc] * kBurst) >> 5);
            fill(kCbBeg + kBurstLen, (n < kTop) ? H : kAvBeg, kBlank);
        }
    }
}

// prime the burst lock (crt_ntsc.c:325-329 / crt_ntscvhs.c:332-336): thread e < CC_SAMPLES * CC_VPER writes ccf[e / CC][e % CC]
__device__ __forceinline__ void mod_skeleton_prime(const SrcCfg &s, MonState *st, const int (*burst)[kCc], int e)
{
    const int field = s.field & 1, frame = s.frame & 1;
    const int flip = kRowCarrier ? 0 : (field == frame);
    const int row = e / kCc, x = e % kCc;
    // template / PV-1000 (crt_template.c:239, 331-335; crt_pv1k.c:236, 326-330): every video line n stores its
    // burst bytes in row (n + 3) % VPER, so row r ends up with the bytes of the lines with n % VPER == r - 3
    const int from = kRowCarrier ? posmod(row - 3, kVper) : 0;
    int p = (int) (signed char) ((kBlank + burst[from][(x + flip * 2) % kCc] * kBurst) >> 5);
    st->ccf[row][x] = kIsVhs ? 0 : p * 128;
    if (kIsVhs && e == 0) st->hsync = 0; // crt_ntscvhs.c:258-259
}

// One CTA per monitor.  (Not folded into the staged picture kernel as a ninth warp: the picture of a line shifted right
// by xoffset >= 4 spills three bytes into the next line's porch, which the reference's write order resolves.)
__global__ void __launch_bounds__(256) k_mod_skeleton_rgb(const SrcCfg *__restrict__ srcs,
                                                          MonState *__restrict__ states,
                                                          signed char *__restrict__ analog_base, int first)
{
    const SrcCfg s = srcs[blockIdx.x];
    signed char *analog = analog_base + (size_t) (first + blockIdx.x) * kSignalBytes;
    __shared__ int burst[kVper][kCc];

    if (bpp_of(s.format) == 0) return; // crt_ntsc.c:190-193
    if (threadIdx.x < kCc * kVper) {
        int b, mi, mq;
        enc_tables(s, (int) threadIdx.x / kCc, (int) threadIdx.x % kCc, b, mi, mq);
        burst[threadIdx.x / kCc][threadIdx.x % kCc] = b;
    }
    __syncthreads();
    mod_skeleton_lines(s, analog, burst, (int) (threadIdx.x >> 5), (int) (blockDim.x >> 5), (int) (threadIdx.x & 31));
    if (threadIdx.x < kCc * kVper) mod_skeleton_prime(s, &states[first + blockIdx.x], burst, (int) threadIdx.x);
}

// Picture pass.  One CTA (8 warps) per monitor; a warp owns 32 consecutive picture lines.
// Per 64-sample chunk: (A) lane-per-sample: fetch source pixels coalesced, RGB->YIQ, pack into a
// [line][sample] tile; (B) lane-per-line: the three serial band-limit IIRs, carrier mix, clamp ->
// bytes; (C) lane-per-sample: coalesced 2-byte stores into analog[].
constexpr int kModChunk = 64;
constexpr int kModTilePitch = kModChunk + 1; // words
constexpr int kModOutPitch = kModChunk / 4 + 1; // words
constexpr int kModWarpSmem = (32 * kModTilePitch + 32 * kModOutPitch) * 4;
constexpr int kModSmem = 8 * kModWarpSmem;

__device__ __forceinline__ void load_rgb(const unsigned char *data, size_t pix, int bpp, int rp, int gp, int bp,
                                         bool aligned4, int &r, int &g, int &b)
{
    if (bpp == 4 && aligned4) {
        unsigned v = __ldg(reinterpret_cast<const unsigned *>(data) + pix);
        r = (v >> (8 * rp)) & 0xff;
        g = (v >> (8 * gp)) & 0xff;
        b = (v >> (8 * bp)) & 0xff;
    } else {
        const unsigned char *p = data + pix * bpp;
        r = __ldg(p + rp);
        g = __ldg(p + gp);
        b = __ldg(p + bp);
    }
}

__host__ __device__ __forceinline__ bool mod_staged_ok(const SrcCfg &s, int destw);
template <bool STAGED> __host__ __device__ __forceinline__ bool mod_takes(const SrcCfg &s);

// (256, 2): its shared memory fits two CTAs per SM; a higher target spills the 64-bit row addresses
__global__ void __launch_bounds__(256, 2) k_mod_picture_rgb(const SrcCfg *__restrict__ srcs,
                                                         const MonCfg *__restrict__ cfgs,
                                                         signed char *__restrict__ analog_base, int first,
                                                         int skip_staged)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned *tile = reinterpret_cast<unsigned *>(smem_raw + warp * kModWarpSmem);
    unsigned *obuf = tile + 32 * kModTilePitch;

    const SrcCfg s = srcs[blockIdx.x];
    const MonCfg cfg = cfgs[first + blockIdx.x];
    signed char *analog = analog_base + (size_t) (first + blockIdx.x) * kSignalBytes;

    const int bpp = bpp_of(s.format);
    if (bpp == 0) return;
    if (skip_staged && mod_takes<true>(s)) return; // done by k_mod_picture_rgb_staged
    int destw = kDestW, desth = kDestH;
    if (s.raw) { // crt_ntsc.c:148-172
        destw = min(s.w, kDestW);
        desth = min(s.h, kDestH);
    }
    if (destw <= 0 || desth <= 0 || s.w <= 0 || s.h <= 0) return;
    const int field = s.field & 1, frame = s.frame & 1;
    const int flip = (field == frame);
    const int ph = kRowCarrier ? 1 : (flip ? -1 : 1); // the template system and the PV-1000 walk colour rows instead (below)
    const int xo_raw = kAvBeg + s.xoffset + (kAvLen - destw) / 2;
    const int xo = kRowCarrier ? xo_raw - (xo_raw % kCc) : (xo_raw & ~3); // crt_template.c:199, crt_pv1k.c:197 / crt_ntsc.c:203
    const int yo = kTop + s.yoffset + (kLines - desth) / 2;
    const int white = kWhite * cfg.white_point / 100;
    const int ire0 = kBlack + cfg.black_point;
    int rp, gp, bp;
    fmt_positions(s.format, rp, gp, bp);
    const unsigned char *data = static_cast<const unsigned char *>(s.data);
    const bool aligned4 = (((reinterpret_cast<uintptr_t>(data) | (uintptr_t) s.pitch) & 3) == 0);

    // five carrier phases (PV-1000): the phase of a sample is not a compile-time constant of the 4-sample inner
    // step, so the tables live in shared memory, [I | Q][colour row][phase]
    __shared__ int mtab[2][kVper][kCc];
    if (kCc == 5) {
        if (threadIdx.x < kCc * kVper) {
            int b;
            enc_tables(s, (int) threadIdx.x / kCc, (int) threadIdx.x % kCc, b, mtab[0][threadIdx.x / kCc][threadIdx.x % kCc],
                       mtab[1][threadIdx.x / kCc][threadIdx.x % kCc]);
        }
        __syncthreads(); // (every return above is block-uniform)
    }
    const int y = warp * 32 + lane; // this lane's picture line
    const int y0 = warp * 32;
    if (y0 >= desth) return;
    // ph * ccmodI/Q (crt_ntsc.c:174-188, 314-315); template: the tables of this lane's colour row (crt_template.c:266)
    int mI[4], mQ[4];
    const int crow = kRowCarrier ? posmod(y + yo, kVper) : 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int b;
        enc_tables(s, crow, k, b, mI[k], mQ[k]);
        mI[k] *= ph;
        mQ[k] *= ph;
    }
    const int nlines = min(32, desth - y0);
    // source row of this lane's line (crt_ntsc.c:258-266).  The reference lets row == h read one
    // row past the image (undefined); we clamp to the last row instead.
    int row = (int) (((long long) min(y, desth - 1) * s.h) / desth) + (field * s.h + desth) / desth / 2;
    if (row >= s.h) row = s.h - 1;
    if (s.compact) row = min(y, desth - 1); // crtx_frames_host staged exactly those rows, in line order (k_rows_gather)

    int hy = 0, hi = 0, hq = 0;
    for (int c0 = 0; c0 < destw; c0 += kModChunk) {
        const int nx = min(kModChunk, destw - c0);
        // (A) fetch + RGB->YIQ, two samples per lane per line
        const int xa = c0 + lane, xb = c0 + lane + 32;
        const int cola = (int) (((long long) min(xa, destw - 1) * s.w) / destw);
        const int colb = (int) (((long long) min(xb, destw - 1) * s.w) / destw);
        for (int l = 0; l < nlines; l++) {
            const unsigned char *rowp = data + row_offset(__shfl_sync(0xffffffffu, row, l), s.pitch);
#pragma unroll
            for (int half = 0; half < 2; half++) {
                int r, g, b;
                load_rgb(rowp, half ? colb : cola, bpp, rp, gp, bp, aligned4, r, g, b);
                int fy = (19595 * r + 38470 * g + 7471 * b) >> 14; // crt_ntsc.c:308-310
                int fi = (39059 * r - 18022 * g - 21103 * b) >> 14;
                int fq = (13894 * r - 34275 * g + 20382 * b) >> 14;
                tile[l * kModTilePitch + lane + 32 * half] =
                    (unsigned) fy | (((unsigned) fi & 0x7ffu) << 10) | ((unsigned) fq << 21);
            }
        }
        __syncwarp();
        // (B) serial along the line, one line per lane
        for (int x4 = 0; x4 < nx; x4 += 4) {
            unsigned packed = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                unsigned w = tile[lane * kModTilePitch + min(x4 + k, kModChunk - 1)];
                int fy = (int) (w & 0x3ffu);
                int fi = ((int) (w << 11)) >> 21;
                int fq = ((int) w) >> 21;
                hy += wmul(fy - hy, kIirY) >> 11; // iirf, crt_ntsc.c:117-126
                hi += wmul(fi - hi, kIirI) >> 11;
                hq += wmul(fq - hq, kIirQ) >> 11;
                // (x + xo) & 3 == k: xo and c0 + x4 are multiples of 4; with five phases (x + xo) % 5 == x % 5
                const int p5 = (c0 + x4 + k) % kCc;
                int ci = wmul(hi, kCc == 5 ? mtab[0][crow][p5] : mI[k]) >> 4;
                int cq = wmul(hq, kCc == 5 ? mtab[1][crow][p5] : mQ[k]) >> 4;
                int ire = ire0 + (wmul(hy + ci + cq, white) >> 10);
                ire = __vimin_s32_relu(ire, 110); // clamp to 0..110 in one instruction
                packed |= (unsigned) ire << (8 * k);
            }
            obuf[lane * kModOutPitch + (x4 >> 2)] = packed;
        }
        __syncwarp();
        // (C) coalesced stores, 2 bytes per lane per line
        for (int l = 0; l < nlines; l++) {
            signed char *dst = analog + (c0 + xo) + (y0 + l + yo) * kHres;
            unsigned w = obuf[l * kModOutPitch + (lane >> 1)];
            unsigned two = (w >> (16 * (lane & 1))) & 0xffffu;
            // the pair is 2-byte aligned when xo is even: always with four carrier phases (xo is a multiple of 4 and
            // CRT_HRES is even), not with the PV-1000's five (xo is a multiple of 5)
            if (2 * lane + 1 < nx && (kCc == 4 || ((c0 + xo) & 1) == 0)) {
                *reinterpret_cast<unsigned short *>(dst + 2 * lane) = (unsigned short) two;
            } else if (2 * lane < nx) {
                dst[2 * lane] = (signed char) (two & 0xff);
                if (2 * lane + 1 < nx) dst[2 * lane + 1] = (signed char) (two >> 8);
            }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------
// Picture pass, staged variant (the one that normally runs).  Same arithmetic as above, different
// data movement: a lane owns a picture line for the whole pass (the IIRs are serial along it), and
// the stretch of its source row that a 32-sample chunk maps to is brought into shared memory by a
// 1-D TMA bulk copy (one per lane, double buffered), so the serial loop reads pixels at
// shared-memory latency and no transposition of the input is needed.  Which source pixel a sample
// reads is tabulated once per CTA.  Finished samples are packed 4 to a word and written back in
// windows aligned to 32-byte sectors (put, below).
// Usable when the chunk's source span fits a stage row; other monitors return at once and are
// handled by k_mod_picture_rgb (gather variant), which in turn skips the ones done here.
// The source image must be readable up to the next 16-byte boundary past its last pixel
// (true of any cudaMalloc / torch allocation; include/crtx_batch.h).  A row's copy covers the 16-byte aligned superset
// of its span, which may take in bytes of the padding between rows: they land in the stage and are never used.
// ---------------------------------------------------------------------------------------
constexpr int kModSChunk = 32;                     // samples per chunk
constexpr int kModSSpan = 192;                     // largest staged span the kernel accepts (incl. alignment slack)
// Stage bytes per line per chunk.  Every lane reads "its row, same column" at once, and rows start on
// 16-byte boundaries, so the pitch decides the bank conflicts: 192 B (48 words) put all 32 lanes on 2
// banks (16-way); 176 B (44 words) spreads them over 8 (4-way,
// the best a 16-byte granular pitch can do).  176 is also exactly the largest copy an accepted span needs.
constexpr int kModSRow = 176;
constexpr int kModSOutPitch = 2 * kModSChunk / 4 + 1;  // words: a ring of two chunks' output per line
constexpr int kModSWarpSmem = 2 * 32 * kModSRow + 32 * kModSOutPitch * 4;
// Behind the eight warps' areas: their mbarriers, then the monitor's column table -- the byte offset of sample x's source
// pixel from the first pixel of x's chunk, for whole chunks -- and each chunk's first and last source column.
constexpr int kModSCols = (kDestW + kModSChunk - 1) / kModSChunk * kModSChunk;
constexpr int kModSSmem = 8 * kModSWarpSmem + 8 * 2 * 8 + kModSCols * 4 + kModSCols / kModSChunk * 8;

__host__ __device__ __forceinline__ bool mod_staged_ok(const SrcCfg &s, int destw)
{
    const int bpp = bpp_of(s.format);
    if (bpp == 0 || destw <= 0 || s.w <= 0 || (kCc != 4 && kCc != 5)) return false; // (four or five samples per carrier period)
    // widest source span of a chunk: ceil(32 * w / destw) + 1 pixels, plus 15 bytes of alignment
    const long long span = ((long long) kModSChunk * s.w + destw - 1) / destw + 1;
    // 4-byte pixels are read from the stage as words: every row must start on a 4-byte boundary
    return span * bpp + 15 + 16 <= kModSSpan && s.w <= 65535
        && (bpp != 4 || ((reinterpret_cast<uintptr_t>(s.data) | (uintptr_t) s.pitch) & 3) == 0);
}

template <bool STAGED>
__host__ __device__ __forceinline__ bool mod_takes(const SrcCfg &s)
{
    int destw = kDestW;
    if (s.raw) destw = s.w < kDestW ? s.w : kDestW;
    return mod_staged_ok(s, destw) == STAGED;
}


// cr * R + cg * G + cb * B of a 4-byte pixel whose channels sit in bytes RP, GP, BP (crt_ntsc.c:308-310) as two-way dot
// products on the pixel word itself (IDP.2A, crt_ptx.cuh): the coefficients of bytes (0, 1) and of bytes (2, 3) are packed as
// 16-bit pairs at compile time.  A pair of non-negative coefficients takes the unsigned form (up to 65535), a pair within
// +-32767 the signed one, and a pair with a coefficient outside both (39059 next to a negative one, -34275) is split into two
// signed halves.  Exact: the sum is the same 32-bit integer the three multiplications give.
constexpr bool fits_s16(int c) { return c >= -32768 && c <= 32767; }
constexpr unsigned pack_h2(int c0, int c1) { return ((unsigned) c0 & 0xffffu) | (((unsigned) c1 & 0xffffu) << 16); }
template <int C0, int C1, bool HI> struct YiqDotPair { // coefficients of bytes (0, 1) or (2, 3), pinned in registers by init()
    static constexpr int kKind = (C0 == 0 && C1 == 0) ? 0 : (C0 >= 0 && C1 >= 0) ? 1 : (fits_s16(C0) && fits_s16(C1)) ? 2 : 3;
    static constexpr int A0 = C0 / 2, B0 = C0 - A0, A1 = C1 / 2, B1 = C1 - A1; // the two signed halves (kind 3)
    static_assert(C0 <= 65535 && C1 <= 65535 && fits_s16(A0) && fits_s16(B0) && fits_s16(A1) && fits_s16(B1), "16-bit coefficients");
    unsigned a, b;
    // `zero` is a 0 the compiler cannot know to be one: OR-ing it in keeps the constants in registers -- ptxas otherwise
    // re-materialises each of them with a move at every use, six issue slots per four samples in the encoder's loop
    __device__ __forceinline__ void init(unsigned zero)
    {
        a = b = 0u;
        if (kKind == 1 || kKind == 2) a = pack_h2(C0, C1) | zero;
        if (kKind == 3) {
            a = pack_h2(A0, A1) | zero;
            b = pack_h2(B0, B1) | zero;
        }
    }
    __device__ __forceinline__ int dot(unsigned v, int acc) const
    {
        if (kKind == 1) return dp2a_u8<HI, false>(a, v, acc);
        if (kKind == 2) return dp2a_u8<HI, true>(a, v, acc);
        if (kKind == 3) return dp2a_u8<HI, true>(b, v, dp2a_u8<HI, true>(a, v, acc));
        return acc;
    }
};
template <int CR, int CG, int CB, int RP, int GP, int BP> struct YiqDot {
    static constexpr int c0 = (RP == 0) ? CR : (GP == 0) ? CG : (BP == 0) ? CB : 0;
    static constexpr int c1 = (RP == 1) ? CR : (GP == 1) ? CG : (BP == 1) ? CB : 0;
    static constexpr int c2 = (RP == 2) ? CR : (GP == 2) ? CG : (BP == 2) ? CB : 0;
    static constexpr int c3 = (RP == 3) ? CR : (GP == 3) ? CG : (BP == 3) ? CB : 0;
    YiqDotPair<c0, c1, false> lo;
    YiqDotPair<c2, c3, true> hi;
    __device__ __forceinline__ void init(unsigned zero)
    {
        lo.init(zero);
        hi.init(zero);
    }
    __device__ __forceinline__ int operator()(unsigned v) const { return hi.dot(v, lo.dot(v, 0)); }
};

// FMT / COLOR are launch-uniform (the host groups monitors by them) so byte extraction and the
// chroma path compile to straight-line code; monitors that do not match return at once.
template <int FMT, bool COLOR>
__global__ void __launch_bounds__(256, 2) k_mod_picture_rgb_staged(const SrcCfg *__restrict__ srcs,
                                                                   const MonCfg *__restrict__ cfgs,
                                                                   signed char *__restrict__ analog_base, int first)
{
    phase_mark(2, 0);
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const SrcCfg s = srcs[blockIdx.x];
    if (!mod_takes<true>(s) || s.format != FMT || (s.as_color != 0) != COLOR) return;
    const MonCfg cfg = cfgs[first + blockIdx.x];
    signed char *analog = analog_base + (size_t) (first + blockIdx.x) * kSignalBytes;

    unsigned char *stage = smem_raw + warp * kModSWarpSmem;
    unsigned *obuf = reinterpret_cast<unsigned *>(stage + 2 * 32 * kModSRow);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + 8 * kModSWarpSmem) + 2 * warp;
    unsigned *coltab = reinterpret_cast<unsigned *>(smem_raw + 8 * kModSWarpSmem + 8 * 2 * 8);
    uint2 *spans = reinterpret_cast<uint2 *>(coltab + kModSCols);

    constexpr int bpp = (FMT <= 1) ? 3 : 4;
    constexpr int rp = (FMT == 0 || FMT == 3) ? 0 : (FMT == 2) ? 1 : (FMT == 4) ? 3 : 2; // crt_core.h:62-67
    constexpr int gp = (FMT == 2 || FMT == 4) ? 2 : 1;
    constexpr int bp = (FMT == 0 || FMT == 3) ? 2 : (FMT == 2) ? 3 : (FMT == 4) ? 1 : 0;
    int destw = kDestW, desth = kDestH;
    if (s.raw) { // crt_ntsc.c:148-172
        destw = min(s.w, kDestW);
        desth = min(s.h, kDestH);
    }
    if (desth <= 0 || s.h <= 0) return;
    const int nchunks = (destw + kModSChunk - 1) / kModSChunk;
    // sample x reads source column (x * w) / destw (crt_ntsc.c:272), which depends on the monitor alone: tabulated once here
    // as a byte offset from the first pixel of x's chunk (samples past destw repeat the last column), with every chunk's
    // span of columns, instead of a division per lane per chunk in every warp
    for (int x = (int) threadIdx.x; x < nchunks * kModSChunk; x += (int) blockDim.x) {
        const unsigned col = (unsigned) min(x, destw - 1) * (unsigned) s.w / (unsigned) destw;
        const unsigned f0 = (unsigned) (x & ~(kModSChunk - 1)) * (unsigned) s.w / (unsigned) destw;
        coltab[x] = (col - f0) * bpp;
        if ((x & (kModSChunk - 1)) == kModSChunk - 1) spans[x / kModSChunk] = make_uint2(f0, col);
    }
    // five carrier phases (PV-1000): the phase of a sample is not a compile-time constant of the 4-sample inner step, so the
    // tables live in shared memory, [I | Q][colour row][phase], as in the gather kernel
    __shared__ int mtab[2][kVper][kCc];
    if (kCc == 5 && threadIdx.x < kCc * kVper) {
        int b;
        enc_tables(s, (int) threadIdx.x / kCc, (int) threadIdx.x % kCc, b, mtab[0][threadIdx.x / kCc][threadIdx.x % kCc],
                   mtab[1][threadIdx.x / kCc][threadIdx.x % kCc]);
    }
    __syncthreads(); // (every return above is block-uniform)
    const int y0 = warp * 32;
    if (y0 >= desth) return;
    const int nlines = min(32, desth - y0);
    if (lane == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
    }
    __syncwarp();
    const int field = s.field & 1, frame = s.frame & 1;
    const int flip = (field == frame);
    const int ph = kRowCarrier ? 1 : (flip ? -1 : 1); // the template system and the PV-1000 walk colour rows instead (below)
    const int xo_raw = kAvBeg + s.xoffset + (kAvLen - destw) / 2;
    const int xo = kRowCarrier ? xo_raw - (xo_raw % kCc) : (xo_raw & ~3); // crt_template.c:199, crt_pv1k.c:197 / crt_ntsc.c:203
    const int yo = kTop + s.yoffset + (kLines - desth) / 2;
    const int white = kWhite * cfg.white_point / 100;
    const int ire0 = kBlack + cfg.black_point;
    const unsigned char *data = static_cast<const unsigned char *>(s.data);
    constexpr bool color = COLOR;

    const bool active = lane < nlines;
    const int y = y0 + min(lane, nlines - 1);
    // ph * ccmodI/Q (crt_ntsc.c:174-188, 314-315); template: the tables of this lane's colour row (crt_template.c:266)
    int mI[4], mQ[4];
    const int crow = kRowCarrier ? posmod(y + yo, kVper) : 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int b;
        mI[k] = mQ[k] = 0;
        if (color) {
            enc_tables(s, crow, k, b, mI[k], mQ[k]);
            mI[k] *= ph;
            mQ[k] *= ph;
        }
    }
    // source row of this lane's line (crt_ntsc.c:258-266); row == h (one past the image, undefined in
    // the reference) is clamped to the last row
    int row = (int) (((long long) y * s.h) / desth) + (field * s.h + desth) / desth / 2;
    if (row >= s.h) row = s.h - 1;
    if (s.compact) row = y; // crtx_frames_host staged exactly those rows, in line order (k_rows_gather)
    const unsigned char *rowp = data + row_offset(row, s.pitch);

    // chunk c covers samples [32c, 32c + 32); its span of source columns f0..f1 is staged from the 16-byte aligned address
    // at or below pixel f0.  Returns the offset of pixel f0 from that address.
    auto issue = [&](int c) {
        const uint2 sp = spans[c];
        const int bytes = (int) (sp.y - sp.x + 1) * bpp;
        const unsigned char *p = rowp + (size_t) sp.x * bpp;
        const int a = (int) (reinterpret_cast<uintptr_t>(p) & 15);
        const unsigned copy = (unsigned) ((a + bytes + 15) & ~15);
        unsigned char *dst = stage + (c & 1) * 32 * kModSRow + lane * kModSRow;
        // rows may sit at different 16-byte phases, so the copies differ in size: sum them up
        unsigned total = active ? copy : 0;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) total += __shfl_xor_sync(0xffffffffu, total, d);
        if (lane == 0) mbar_expect_tx(&bars[c & 1], total);
        __syncwarp();
        if (active) tma_load_1d(dst, p - a, copy, &bars[c & 1]);
        return a;
    };

    // the rows of the RGB -> YIQ matrix (crt_ntsc.c:308-310) for 4-byte pixels, see YiqDot
    YiqDot<19595, 38470, 7471, rp, gp, bp> dot_y;
    YiqDot<39059, -18022, -21103, rp, gp, bp> dot_i;
    YiqDot<13894, -34275, 20382, rp, gp, bp> dot_q;
    if (bpp == 4) {
        const unsigned zero = (unsigned) first >> 31; // (0: the host keeps first in [0, 2^31))
        dot_y.init(zero);
        if (color) {
            dot_i.init(zero);
            dot_q.init(zero);
        }
    }
    // Stores.  A line's finished bytes go out in windows that end on a 32-byte boundary of analog[]: eight lanes write one
    // line's window as aligned words, four lines per instruction, so every sector but the first and last of a line is
    // written whole, once.  (Partly written sectors cost the memory system a read of the sector; 2-byte stores per chunk
    // left two of them per line and chunk.)  put(c) writes the window [e - 32, e) whose end e lies in (32c, 32c + 32],
    // cut to [0, destw): after chunk c all of it is in the line's 64-byte ring, chunk c - 1 in one half, chunk c in the other.
    auto put = [&](int c) {
        const int t = lane & 7;
#pragma unroll
        for (int i = 0; i < 32 / 4; i++) {
            const int L = 4 * i + (lane >> 3);
            if (L >= nlines) continue;
            signed char *ln = analog + (y0 + L + yo) * kHres + xo;
            const int e0 = (int) ((0u - (unsigned) reinterpret_cast<uintptr_t>(ln)) & 31u);
            const int x = c * kModSChunk + (e0 ? e0 : 32) - 32 + 4 * t; // ln + x is a multiple of 4
            if (x >= destw || x + 4 <= 0) continue;
            const unsigned *ring = obuf + L * kModSOutPitch;
            const int pos = x & (2 * kModSChunk - 1);
            const unsigned long long two = ring[pos >> 2] | ((unsigned long long) ring[((pos >> 2) + 1) & (2 * kModSChunk / 4 - 1)] << 32);
            const unsigned v = (unsigned) (two >> (8 * (pos & 3)));
            if (x >= 0 && x + 4 <= destw) {
                *reinterpret_cast<unsigned *>(ln + x) = v;
            } else {
                for (int b = 0; b < 4; b++)
                    if (x + b >= 0 && x + b < destw) ln[x + b] = (signed char) (v >> (8 * b));
            }
        }
    };
    int hy = 0, hi = 0, hq = 0;
    int a_cur = issue(0);
#pragma unroll 1
    for (int c = 0; c < nchunks; c++) {
        const int a_nxt = (c + 1 < nchunks) ? issue(c + 1) : 0;
        const int c0 = c * kModSChunk;
        mbar_wait(&bars[c & 1], (c >> 1) & 1);
        __syncwarp();
        const unsigned char *srow = stage + (c & 1) * 32 * kModSRow + lane * kModSRow + a_cur;
        a_cur = a_nxt;
        int p5 = c0 % 5; // carrier phase of the chunk's first sample (five-phase systems)
        // The whole chunk, straight-line: no sample's fetch or RGB -> YIQ waits for the IIR chains of the samples before it,
        // so the compiler overlaps them with those chains.  The last chunk runs whole as well: the samples past destw read
        // the last column (the table repeats it), move nothing but this line's IIR state after its last stored sample, and
        // are not stored.
        const uint4 *offs = reinterpret_cast<const uint4 *>(coltab + c0);
        unsigned packed[kModSChunk / 4];
#pragma unroll
        for (int g = 0; g < kModSChunk / 4; g++) {
            const uint4 o4 = offs[g];
            const unsigned off4[4] = {o4.x, o4.y, o4.z, o4.w};
            unsigned word = 0;
            int rr[4], gg[4], bb[4];
            unsigned pix[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int off = (int) off4[k];
                if (bpp == 4) {
                    pix[k] = *reinterpret_cast<const unsigned *>(srow + off);
                } else {
                    rr[k] = srow[off + rp];
                    gg[k] = srow[off + gp];
                    bb[k] = srow[off + bp];
                }
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                int fy, fi = 0, fq = 0; // crt_ntsc.c:308-310
                if (bpp == 4) { // the matrix rows as dot products straight on the pixel word: no byte is ever extracted
                    fy = dot_y(pix[k]) >> 14;
                    if (color) {
                        fi = dot_i(pix[k]) >> 14;
                        fq = dot_q(pix[k]) >> 14;
                    }
                } else {
                    const int r = rr[k], g = gg[k], b = bb[k];
                    fy = (19595 * r + 38470 * g + 7471 * b) >> 14;
                    if (color) {
                        fi = (39059 * r - 18022 * g - 21103 * b) >> 14;
                        fq = (13894 * r - 34275 * g + 20382 * b) >> 14;
                    }
                }
                hy += wmul(fy - hy, kIirY) >> 11; // iirf, crt_ntsc.c:117-126
                int sum = hy;
                if (color) {
                    hi += wmul(fi - hi, kIirI) >> 11;
                    hq += wmul(fq - hq, kIirQ) >> 11;
                    if (kCc == 5) { // (x + xo) % 5 == x % 5: xo is a multiple of 5; p5 walks 0 .. 4 along the line
                        sum += (wmul(hi, mtab[0][crow][p5]) >> 4) + (wmul(hq, mtab[1][crow][p5]) >> 4);
                        p5 = (p5 == 4) ? 0 : p5 + 1;
                    } else { // (x + xo) & 3 == k: xo and c0 are multiples of 4
                        sum += (wmul(hi, mI[k]) >> 4) + (wmul(hq, mQ[k]) >> 4);
                    }
                }
                int ire = ire0 + (wmul(sum, white) >> 10);
                ire = __vimin_s32_relu(ire, 110); // clamp to 0..110 in one instruction
                word |= (unsigned) ire << (8 * k);
            }
            packed[g] = word;
        }
#pragma unroll
        for (int g = 0; g < kModSChunk / 4; g++) obuf[lane * kModSOutPitch + (c & 1) * (kModSChunk / 4) + g] = packed[g];
        __syncwarp();
        put(c);
        __syncwarp();
    }
    put(nchunks); // the rest of every line
    phase_mark(2, 14);
    phase_mark(2, 12, 7 * 32);
}

#endif // RGB systems

// =======================================================================================
// encoder, NES (fully parallel: no recurrence along the line)
// =======================================================================================
#if (CRT_SYSTEM == CRT_SYSTEM_NES)

__constant__ int c_nes_level[16] = { -12042, 0,     34406,  81427,  -17203, -8028, 19497, 57342,
                                     43581,  75693, 112965, 112965, 26951,  52181, 83721, 83721 };
__constant__ int c_nes_emph[6] = { 0300, 0100, 0500, 0400, 0600, 0200 };

__device__ __forceinline__ int nes_square(int p, int phase) // crt_nes.c:21-61
{
    int hue = p & 15;
    if (hue >= 14) return 0;
    int emph = ((p & 0700) & c_nes_emph[(phase >> 1) % 6]) > 0;
    int high = (hue == 0) ? 1 : ((hue == 13) ? 0 : (((hue + phase) % 12) < 6));
    return c_nes_level[high * 8 + emph * 4 + ((p >> 4) & 3)];
}

// The composite level of a picture sample depends only on the 9-bit PPU pixel and the chroma phase
// modulo 12 (square_sample is periodic in phase: (hue + phase) % 12 and (phase >> 1) % 6), plus the
// monitor's black / white points.  k_nes_table tabulates all 512 x 12 finished sample bytes per monitor
// (crt_nes.c:21-61, 182-190) together with the burst rows; k_mod_nes then turns every sample into an
// index computation and one table read, written with coalesced byte stores.
constexpr int kNesTabBytes = 512 * 12 + 16; // + 12 burst bytes (3 rows x 4 phases) + pad
constexpr int kNesParts = 8;               // CTAs per monitor in k_mod_nes

__global__ void __launch_bounds__(256) k_nes_table(const SrcCfg *__restrict__ srcs, const MonCfg *__restrict__ cfgs,
                                                   MonState *__restrict__ states, signed char *__restrict__ tabs,
                                                   int first)
{
    const int m = blockIdx.x, tid = threadIdx.x;
    const SrcCfg s = srcs[m];
    const MonCfg cfg = cfgs[first + m];
    signed char *tab = tabs + (size_t) (first + m) * kNesTabBytes;
    for (int e = tid; e < 512 * 12; e += 256) {
        const int p = e / 12, phase = e - p * 12;
        int ire = kBlack + cfg.black_point;
        ire += nes_square(p, phase) + nes_square(p, phase + 1) + nes_square(p, phase + 2) + nes_square(p, phase + 3);
        tab[e] = (signed char) ((wmul(ire, cfg.white_point) / 100) >> 12);
    }
    if (tid < 12) { // burst rows (crt_nes.c:123-130) and the primed burst lock (crt_nes.c:196-200)
        const int row = tid >> 2, x = tid & 3;
        int sn, cs;
        const int deg = (s.hue + x * 90 + (row + s.dot_crawl_offset) * 120 + 33) % 360;
        sincos14_d(sn, cs, deg * 8192 / 180);
        const signed char v = (signed char) ((kBlank + (sn >> 10) * kBurst) >> 5);
        tab[512 * 12 + tid] = v;
        states[first + m].ccf[row][x] = (int) v * 128;
    }
}

// grid (kNesParts, n): each CTA takes every kNesParts-th chunk of the monitor's work
__global__ void __launch_bounds__(256) k_mod_nes(const SrcCfg *__restrict__ srcs, const signed char *__restrict__ tabs,
                                                 signed char *__restrict__ analog_base, int first)
{
    __shared__ __align__(16) signed char tab[kNesTabBytes];
    const int m = blockIdx.y, part = blockIdx.x, tid = threadIdx.x;
    const SrcCfg s = srcs[m];
    signed char *analog = analog_base + (size_t) (first + m) * kSignalBytes;
    const int xo = (kAvBeg + s.xoffset) & ~3, yo = kTop + s.yoffset;
    {
        const uint4 *src4 = reinterpret_cast<const uint4 *>(tabs + (size_t) (first + m) * kNesTabBytes);
        for (int e = tid; e < kNesTabBytes / 16; e += 256) reinterpret_cast<uint4 *>(tab)[e] = __ldg(src4 + e);
    }
    __syncthreads();
    const signed char *burst = tab + 512 * 12;

    // this CTA's share: lines n with n % kNesParts == part (skeleton), picture lines y likewise
    if (s.reinit) { // setup_field, crt_nes.c:81-104: every line whole; picture lines are done below
        for (int n = part; n < kVres; n += kNesParts) {
            if (n >= yo && n < yo + kLines) continue; // written (skeleton first) by the CTA that owns the line
            const int sync_end = (n >= 259) ? kNesVsyncEnd : kBwBeg;
            for (int t = tid; t < kHres; t += 256)
                analog[n * kHres + t] = (signed char) ((t >= kSyncBeg && t < sync_end) ? kSync : kBlank);
        }
    }
    const unsigned char *data = static_cast<const unsigned char *>(s.data);
    for (int y = part; y < kLines; y += kNesParts) {
        const int n = y + yo;
        // every byte of a picture line is written by this one CTA, in order: skeleton, burst, picture
        if (s.reinit) {
            const int sync_end = (n >= 259) ? kNesVsyncEnd : kBwBeg;
            for (int t = tid; t < kHres; t += 256)
                analog[n * kHres + t] = (signed char) ((t >= kSyncBeg && t < sync_end) ? kSync : kBlank);
            __syncthreads();
        }
        if (tid < kBurstLen) { // crt_nes.c:174-178
            const int t = kCbBeg + tid;
            analog[n * kHres + t] = burst[(n % 3) * 4 + (t & 3)];
        }
        int row = (y * s.h) / kLines;
        if (row >= s.h) row = s.h - 1; // the reference reads one row past the image here (undefined)
        if (row < 0) row = 0;
        // (the pitch is read per line: held in a register for the whole kernel it takes the kernel past 32 registers,
        // and 8 CTAs per SM to 6)
        const unsigned short *src_row = reinterpret_cast<const unsigned short *>(data + row_offset(row, __ldg(&srcs[m].pitch)));
        const int phase0 = ((y + yo + s.dot_crawl_offset) % 3) * 4;
        for (int x = tid; x < kAvLen; x += 256) { // crt_nes.c:180-193
            const int p = __ldg(src_row + (x * s.w) / kAvLen) & 0x1ff;
            analog[n * kHres + xo + x] = tab[p * 12 + (phase0 + 3 * x) % 12];
        }
    }
}

#endif // NES

// =======================================================================================
// encoder, SNES (crt_snes.c:125-327): the NTSC encoder's structure on the NES line layout, a burst and
// carrier phase that walk a 3-line cycle (+ dot_crawl_offset), and NO band-limit (CRT_DO_BANDLIMITING 0,
// crt_snes.h:84) -- so, unlike crt_ntsc.c, every sample is independent.
// =======================================================================================
#if (CRT_SYSTEM == CRT_SYSTEM_SNES)

constexpr int kSnesParts = 8; // CTAs per monitor; CTA p owns signal lines n with n % kSnesParts == p

__global__ void __launch_bounds__(256) k_mod_snes(const SrcCfg *__restrict__ srcs, const MonCfg *__restrict__ cfgs,
                                                  MonState *__restrict__ states, signed char *__restrict__ analog_base,
                                                  int first)
{
    __shared__ int modI[3][4], modQ[3][4], burst[3][4];
    const int m = blockIdx.y, part = blockIdx.x, tid = threadIdx.x;
    const SrcCfg s = srcs[m];
    const int bpp = bpp_of(s.format);
    if (bpp == 0) return; // crt_snes.c:189-192
    const MonCfg cfg = cfgs[first + m];
    signed char *analog = analog_base + (size_t) (first + m) * kSignalBytes;

    if (tid < 12) { // crt_snes.c:170-187
        const int row = tid >> 2, x = tid & 3;
        int bI = 0, bQ = 0, bB = 0;
        if (s.as_color) {
            const int step = 360 / 4;
            const int n = (row + s.dot_crawl_offset) * (360 / kVper) + s.hue + x * step;
            int sn, cs;
            sincos14_d(sn, cs, (n - step + 210) * 8192 / 180); // HUE_OFFSET, crt_snes.h:99
            bB = sn >> 10;
            sincos14_d(sn, cs, n * 8192 / 180);
            bI = sn >> 10;
            sincos14_d(sn, cs, (n - 90) * 8192 / 180); // Q_OFFSET, crt_snes.h:97
            bQ = sn >> 10;
        }
        modI[row][x] = bI;
        modQ[row][x] = bQ;
        burst[row][x] = bB;
        // crt_snes.c:246-248, 322-326: every video line re-primes the lock of its own row with its burst bytes
        if (part == 0) states[first + m].ccf[row][x] = (int) (signed char) ((kBlank + bB * kBurst) >> 5) * 128;
    }
    __syncthreads();

    int destw = kDestW, desth = kDestH; // crt_snes.c:129-130, 144-168
    if (s.raw) {
        destw = min(s.w, kDestW);
        desth = min(s.h, kDestH);
    }
    int xo = kAvBeg + s.xoffset + (kAvLen - destw) / 2;
    const int yo = kTop + s.yoffset + (kLines - desth) / 2;
    xo = xo - (xo % 4); // crt_snes.c:201
    const int white = kWhite * cfg.white_point / 100;
    const int ire0 = kBlack + cfg.black_point;
    int rp, gp, bp;
    fmt_positions(s.format, rp, gp, bp);
    const unsigned char *data = static_cast<const unsigned char *>(s.data);
    const bool word_pixels = (bpp == 4) && (((reinterpret_cast<uintptr_t>(data) | (uintptr_t) s.pitch) & 3) == 0);

    for (int n = part; n < kVres; n += kSnesParts) {
        signed char *line = analog + n * kHres;
        // ---- sync / blank / burst of line n (crt_snes.c:203-250)
        const bool equ = (n <= 2) || (n >= 7 && n <= 9);
        const bool vsy = (n >= 3 && n <= 6);
        for (int t = tid; t < kHres; t += 256) {
            int v;
            bool write = true;
            if (equ) {
                v = (t < 4 * kHres / 100 || (t >= 50 * kHres / 100 && t < 54 * kHres / 100)) ? kSync : kBlank;
            } else if (vsy) {
                v = (t < 46 * kHres / 100 || (t >= 50 * kHres / 100 && t < 96 * kHres / 100)) ? kSync : kBlank;
            } else {
                v = (t >= kSyncBeg && t < kBwBeg) ? kSync : kBlank;
                write = (t < kAvBeg) || (n < kTop);
                if (t >= kCbBeg && t < kCbBeg + kBurstLen) v = (kBlank + burst[n % kVper][t & 3] * kBurst) >> 5;
            }
            if (write) line[t] = (signed char) v;
        }
        // ---- picture line y = n - yo, after the line's own template (crt_snes.c:252-320)
        const int y = n - yo;
        if (y < 0 || y >= desth || s.h <= 0 || s.w <= 0) continue;
        // the picture normally starts at or after AV_BEG on a line whose template stops there; only when the
        // two overlap (negative offsets, picture above the first active line) must the template land first
        if (xo < kAvBeg || n < kTop) __syncthreads(); // block-uniform condition
        int sy = (y * s.h) / desth;
        if (sy >= s.h) sy = s.h - 1; // (never taken for y < desth; the reference clamps to one row past the image)
        const unsigned char *src_row = data + row_offset(sy, s.pitch);
        const int ph = n % kVper;
        constexpr int kPer = (kAvLen + 255) / 256; // samples per thread and line
        unsigned px[kPer];
#pragma unroll
        for (int q = 0; q < kPer; q++) { // all of a thread's pixel fetches first
            const int x = tid + q * 256;
            px[q] = 0;
            if (x < destw) {
                const unsigned char *pix = src_row + (size_t) (((unsigned) x * (unsigned) s.w) / (unsigned) destw) * bpp;
                if (word_pixels) px[q] = __ldg(reinterpret_cast<const unsigned *>(pix));
                else px[q] = (unsigned) pix[0] | (unsigned) pix[1] << 8 | (unsigned) pix[2] << 16 | (bpp == 4 ? (unsigned) pix[3] << 24 : 0u);
            }
        }
#pragma unroll
        for (int q = 0; q < kPer; q++) {
            const int x = tid + q * 256;
            if (x >= destw) continue;
            const int r = (px[q] >> (8 * rp)) & 0xff, g = (px[q] >> (8 * gp)) & 0xff, b = (px[q] >> (8 * bp)) & 0xff;
            const int fy = (19595 * r + 38470 * g + 7471 * b) >> 14;
            int fi = (39059 * r - 18022 * g - 21103 * b) >> 14;
            int fq = (13894 * r - 34275 * g + 20382 * b) >> 14;
            const int xoff = (x + xo) % 4;
            fi = wmul(fi, modI[ph][xoff]) >> 4;
            fq = wmul(fq, modQ[ph][xoff]) >> 4;
            int ire = ire0 + (wmul(fy + fi + fq, white) >> 10);
            ire = __vimin_s32_relu(ire, 110);
            line[x + xo] = (signed char) ire;
        }
    }
}

#endif // SNES

// =======================================================================================
// encoder, NES-RGB (crt_nesrgb.c:19-172): the NES sync template (written once per stream) and 3-line burst
// cycle around an RGB picture encoded like the SNES one (no band-limit: samples are independent).
// =======================================================================================
#if (CRT_SYSTEM == CRT_SYSTEM_NESRGB)

constexpr int kNesRgbParts = 8; // CTAs per monitor; CTA p owns signal lines n with n % kNesRgbParts == p

// (256, 8): the kernel fits 32 registers without spilling, and keeps 8 CTAs per SM
__global__ void __launch_bounds__(256, 8) k_mod_nesrgb(const SrcCfg *__restrict__ srcs, const MonCfg *__restrict__ cfgs,
                                                    MonState *__restrict__ states, signed char *__restrict__ analog_base,
                                                    int first)
{
    __shared__ int modI[3][4], modQ[3][4], burst[3][4];
    const int m = blockIdx.y, part = blockIdx.x, tid = threadIdx.x;
    const SrcCfg s = srcs[m];
    const int bpp = bpp_of(s.format);
    const MonCfg cfg = cfgs[first + m];
    signed char *analog = analog_base + (size_t) (first + m) * kSignalBytes;

    if (tid < 12) { // crt_nesrgb.c:68-79
        const int row = tid >> 2, x = tid & 3;
        const int n = (row + s.dot_crawl_offset) * (360 / kVper) + x * (360 / 4);
        int sn, cs;
        sincos14_d(sn, cs, (s.hue + 90 + n + 33) * 8192 / 180);
        burst[row][x] = sn >> 10;
        sincos14_d(sn, cs, n * 8192 / 180);
        modI[row][x] = sn >> 10;
        sincos14_d(sn, cs, (n - 90) * 8192 / 180);
        modQ[row][x] = sn >> 10;
        // crt_nesrgb.c:106-110, 166-170: every picture line re-primes the lock of its row with its burst bytes
        if (part == 0 && bpp != 0) states[first + m].ccf[row][x] = (int) (signed char) ((kBlank + burst[row][x] * kBurst) >> 5) * 128;
    }
    __syncthreads();

    const int xo = (kAvBeg + s.xoffset) & ~3, yo = kTop + s.yoffset; // crt_nesrgb.c:86-90
    const int white = kWhite * cfg.white_point / 100;
    const int ire0 = kBlack + cfg.black_point;
    int rp, gp, bp;
    fmt_positions(s.format, rp, gp, bp);
    const unsigned char *data = static_cast<const unsigned char *>(s.data);
    const bool word_pixels = (bpp == 4) && (((reinterpret_cast<uintptr_t>(data) | (uintptr_t) s.pitch) & 3) == 0);

    for (int n = part; n < kVres; n += kNesRgbParts) {
        signed char *line = analog + n * kHres;
        if (s.reinit) { // setup_field, crt_nesrgb.c:19-47 -- before the pixel-format check of crt_nesrgb.c:81-84
            const int sync_end = (n >= 259) ? kNesVsyncEnd : kBwBeg;
            for (int t = tid; t < kHres; t += 256) line[t] = (signed char) ((t >= kSyncBeg && t < sync_end) ? kSync : kBlank);
        }
        const int y = n - yo;
        if (bpp == 0 || y < 0 || y >= kLines || s.h <= 0 || s.w <= 0) continue;
        if (s.reinit) __syncthreads(); // (block-uniform) template before burst and picture
        if (tid < kBurstLen) { // crt_nesrgb.c:104-110
            const int t = kCbBeg + tid;
            line[t] = (signed char) ((kBlank + burst[n % kVper][t & 3] * kBurst) >> 5);
        }
        int sy = (y * s.h) / kLines;
        if (sy >= s.h) sy = s.h - 1; // (never taken; the reference clamps to one row past the image)
        const unsigned char *src_row = data + row_offset(sy, s.pitch);
        const int ph = n % kVper;
        constexpr int kPer = (kAvLen + 255) / 256;
        unsigned px[kPer];
#pragma unroll
        for (int q = 0; q < kPer; q++) { // all of a thread's pixel fetches first
            const int x = tid + q * 256;
            px[q] = 0;
            if (x < kAvLen) {
                const unsigned char *pix = src_row + (size_t) (((unsigned) x * (unsigned) s.w) / (unsigned) kAvLen) * bpp;
                if (word_pixels) px[q] = __ldg(reinterpret_cast<const unsigned *>(pix));
                else px[q] = (unsigned) pix[0] | (unsigned) pix[1] << 8 | (unsigned) pix[2] << 16 | (bpp == 4 ? (unsigned) pix[3] << 24 : 0u);
            }
        }
#pragma unroll
        for (int q = 0; q < kPer; q++) {
            const int x = tid + q * 256;
            if (x >= kAvLen) continue;
            const int r = (px[q] >> (8 * rp)) & 0xff, g = (px[q] >> (8 * gp)) & 0xff, b = (px[q] >> (8 * bp)) & 0xff;
            const int fy = (19595 * r + 38470 * g + 7471 * b) >> 14;
            int fi = (39059 * r - 18022 * g - 21103 * b) >> 14;
            int fq = (13894 * r - 34275 * g + 20382 * b) >> 14;
            const int xoff = (x + xo) % 4;
            fi = wmul(fi, modI[ph][xoff]) >> 4;
            fq = wmul(fq, modQ[ph][xoff]) >> 4;
            int ire = ire0 + (wmul(fy + fi + fq, white) >> 10);
            ire = __vimin_s32_relu(ire, 110);
            line[x + xo] = (signed char) ire;
        }
    }
}

#endif // NES-RGB

// =======================================================================================
// noise pass (crt_core.c:346-367), LCG variant, run inside k_sync.  16 samples per vector, 128-bit accesses;
// the generator state of sample i is rn0 advanced i + 1 steps, reached by two table look-ups.
// =======================================================================================
constexpr int kNoiseVec = 16;
constexpr int kNoiseThreads = (kInputSize + kNoiseVec - 1) / kNoiseVec; // 16-sample vectors of inp[]
constexpr int kJumpLo = 128; // lo[k] = jump(16 * k), hi[k] = jump(16 * 128 * k)
constexpr int kJumpHi = (kNoiseThreads + kJumpLo - 1) / kJumpLo + 1;

#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
// VHS noise pass with the per-sample noise term drawn elsewhere (crt_core.c:343-366): the drop-in
// path draws from the process's libc rand() on the host, exactly as the reference does, and hands
// the resulting terms over; this kernel only adds and clamps.
__global__ void __launch_bounds__(256) k_noise_terms(const MonCfg *__restrict__ cfgs,
                                                     const signed char *__restrict__ analog_base,
                                                     signed char *__restrict__ inp_base,
                                                     const short *__restrict__ terms, int first)
{
    const int m = first + blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= kInputSize || cfgs[m].bpp == 0) return;
    const signed char *analog = analog_base + (size_t) m * kSignalBytes;
    signed char *inp = inp_base + (size_t) m * kSignalBytes;
    int s = analog[i] + terms[(size_t) blockIdx.y * kInputSize + i];
    inp[i] = (signed char) clampi(s, -127, 127);
}
#endif

} // namespace crt

#include "crt_sync.cuh"
#include "crt_lines.cuh"
#include "crt_lines2.cuh"
#include "crt_lines_fir.cuh"
#include "crt_bloom.cuh"
#include "crt_vhs.cuh"
