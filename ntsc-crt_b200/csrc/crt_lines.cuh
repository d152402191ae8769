// crt_lines.cuh -- k_lines, the line pass of crt_demodulate (crt_core.c:511-664): Y/I/Q equalisers
// along each decoded scanline, horizontal resample, YIQ->RGB, contrast, clamp, optional blend with
// the previous image, row duplication.  This is the kernel the roofline figure is quoted on.
//
// Shape.  The three equalisers are 8 cascaded one-pole stages that round at every step, so a line
// cannot be scanned in parallel: ONE LANE CARRIES ONE SCANLINE, 32 lines per warp, 8 warps (one
// monitor = 240 lines) per CTA.  Everything that is warp-uniform (sample index, pixel index, the
// resampling phase, geometry) comes from kernel arguments so the compiler keeps it on the uniform
// datapath and the per-lane instruction stream is almost pure filter + pixel arithmetic.
//   in : each lane's 753-sample window of inp[] arrives in shared memory through 1-D TMA bulk copies
//        (cp.async.bulk + mbarrier), 64 samples per stage, double buffered;
//   out: finished pixels go to a [line][16 px] shared-memory tile; every 16 pixels the warp turns
//        the tile around and writes 64-byte row segments with 128-bit stores (4 lanes per row, 8
//        rows per instruction), blending with the previous image and replicating duplicated rows.
#pragma once

#include "crt_kernels.cuh"

namespace crt {

struct Eq { // crt_core.c:158-164
    int l0, l1, l2, l3;
    int h0, h1, h2, h3;
    int s1, s2, s3; // input history, s3 oldest
};

__device__ __forceinline__ void eq_reset(Eq &f) { f.l0 = f.l1 = f.l2 = f.l3 = f.h0 = f.h1 = f.h2 = f.h3 = f.s1 = f.s2 = f.s3 = 0; }

// One one-pole stage (crt_core.c:211-217): f += (C * (in - f) + 32768) >> 16.  `rnd` is 32768 held in a
// register the compiler cannot see through, so the coefficient becomes the instruction's immediate
// (IMAD d, C, rnd) instead of being re-materialised into a register for every stage.
template <int C>
__device__ __forceinline__ int pole(int f, int in, int rnd)
{
    return wadd(f, wadd(wmul(wsub(in, f), C), rnd) >> 16);
}

// One eqf() step (crt_core.c:205-233).
// FAST is exact when every Q16 gain of 65536 is an identity and no product wraps, i.e. every band
// stays below 32768 in magnitude.  k_sync guarantees that per monitor from max|s| * |wave| >> 9 <= 16382
// (chroma inputs <= 16383; |s| <= 127 inside inp[], 128 for a line whose window reaches the struct tail behind it; a one-pole stage with 0 < c <= 65536 never leaves the range of its inputs,
// so |fH3 - fL3| < 32768) and |bright| <= 4096 (luma; the hf = 79824 cascade overshoots by at most 1.558^4).  Then for I and Q
// r0 + r1 == fH[3] exactly -- their low cascades cancel and are not evaluated at all -- and Y's
// middle gain 8192 is an arithmetic shift by 3.
template <int LF, int HF, int G1, int G2, bool FAST, bool IS_Y>
__device__ __forceinline__ int eq_step(Eq &f, int s, int rnd)
{
    f.h0 = pole<HF>(f.h0, s, rnd);
    f.h1 = pole<HF>(f.h1, f.h0, rnd);
    f.h2 = pole<HF>(f.h2, f.h1, rnd);
    f.h3 = pole<HF>(f.h3, f.h2, rnd);
    int r;
    if (FAST && !IS_Y) {
        r = f.h3;
        if (G2 != 0) r = wadd(r, wmul(wsub(f.s3, f.h3), G2) >> 16);
    } else {
        f.l0 = pole<LF>(f.l0, s, rnd);
        f.l1 = pole<LF>(f.l1, f.l0, rnd);
        f.l2 = pole<LF>(f.l2, f.l1, rnd);
        f.l3 = pole<LF>(f.l3, f.l2, rnd);
        if (FAST) {
            // the middle band: gain 8192 is an arithmetic shift; the PV-1000's 12192 (crt_core.c:282) a product that
            // cannot wrap inside the fast path's range (|fH3 - fL3| * 12192 < 2^31)
            const int mid = (G1 == 8192) ? (wsub(f.h3, f.l3) >> 3) : (wmul(wsub(f.h3, f.l3), G1) >> 16);
            r = wadd(wadd(f.l3, mid), wmul(wsub(f.s3, f.h3), G2) >> 16);
        } else {
            const int r0 = wmul(f.l3, 65536) >> 16;
            const int r1 = wmul(wsub(f.h3, f.l3), G1) >> 16;
            const int r2 = wmul(wsub(f.s3, f.h3), G2) >> 16;
            r = wadd(wadd(r0, r1), r2);
        }
    }
    if (G2 != 0 || !FAST) { // Q's history is never read on the fast path (gain 0)
        f.s3 = f.s2;
        f.s2 = f.s1;
        f.s1 = s;
    }
    return r;
}

// crt_core.c:573-581 -> 0x00RRGGBB.  (Shifts and clamps stay on the ALU pipe: IMAD.HI and I2I.SAT are slower-rate
// instructions.)
// HALF: every channel already halved, as the blend needs it -- floor(clamp(v >> 8, 0, 255) / 2) == clamp(v >> 9, 0, 127)
template <bool HALF = false>
__device__ __forceinline__ unsigned yiq_to_rgb(int y, int i, int q, int contrast)
{
    constexpr int sh = HALF ? 9 : 8, top = HALF ? 127 : 255;
    int r = wmul(wadd(wadd(y, wmul(3879, i)), wmul(2556, q)) >> 12, contrast) >> sh;
    int g = wmul(wsub(wsub(y, wmul(1126, i)), wmul(2605, q)) >> 12, contrast) >> sh;
    int b = wmul(wadd(wsub(y, wmul(4530, i)), wmul(7021, q)) >> 12, contrast) >> sh;
    r = __vimin_s32_relu(r, top); // max(min(r, 255), 0) in one VIMNMX.RELU
    g = __vimin_s32_relu(g, top);
    b = __vimin_s32_relu(b, top);
    return (unsigned) (r << 16 | g << 8 | b);
}

// crt_core.c:559-581, literal (wrap-exact) form
template <bool HALF = false>
__device__ __forceinline__ unsigned yiq_pixel(int ay, int ai, int aq, int by, int bi, int bq, int R, int L, int contrast)
{
    const int y = wadd(wmul(ay, L) >> 2, wmul(by, R) >> 2);
    const int i = wadd(wmul(ai, L) >> 14, wmul(bi, R) >> 14);
    const int q = wadd(wmul(aq, L) >> 14, wmul(bq, R) >> 14);
    return yiq_to_rgb<HALF>(y, i, q, contrast);
}

constexpr int kLinesWarps = 8;                // 256 lane-lines per CTA = one monitor
constexpr int kSub = 3 * kCc;                 // samples filtered between two pixel passes: a multiple of
                                              // 4 (carrier phase; 5 for the PV-1000) and 3 (equaliser history), so
                                              // the unrolled block needs no register rotation at all
constexpr int kStageSamples = (kCc == 4) ? 96 : 240; // samples per staged chunk (8 / 16 sub-chunks): fewer, larger
                                              // bulk copies -- 32 per warp per stage -- keep the TMA unit ahead
constexpr int kStageRow = ((kStageSamples + 15 + 15) / 16) * 16; // bytes per line per stage: the 16-byte
                                              // aligned superset of a window at any byte phase
constexpr int kStageBytes = 32 * kStageRow;   // per warp per stage
constexpr int kTilePitch = 20;                // words: 16 pixel columns per line, pitch/4 odd
constexpr int kTileBytes = 32 * kTilePitch * 4;
// The line is filtered in whole sub-chunks: up to kSub - 1 samples past AV_LEN are run through the
// equalisers (they exist in the padded signal buffer) but no pixel ever reads them, because the
// resampler stops at sample AV_LEN - 1 (crt_core.c:529, 555).
constexpr int kSamplesPadded = ((kAvLen + kSub - 1) / kSub) * kSub;
constexpr int kNumStages = (kSamplesPadded + kStageSamples - 1) / kStageSamples;
static_assert(kStageRow % 16 == 0 && kStageSamples % 16 == 0 && kStageSamples % kSub == 0 && kSub % kCc == 0 && kSub % 3 == 0,
              "stage layout: TMA source offsets and destinations are multiples of 16; carrier phase == t % kCc");

// Per-lane row of decoded Y/I/Q for the current sub-chunk: slot 0 carries the last sample of the
// previous sub-chunk, slots 1..kSub the new ones.  FAST packs a sample into 8 bytes (Y | I:Q as
// 16-bit halves, both provably in range there), the generic path keeps three full words (16 bytes).
// An odd pitch in entries makes "all lanes, same slot" accesses bank-conflict free.
template <bool FAST> struct YiqRow {
    static constexpr int kEntryBytes = FAST ? 8 : 16;
    static constexpr int kPitch = (kSub + 1) | 1; // entries, odd
    static constexpr int kBytes = 32 * kPitch * kEntryBytes;
};
template <bool FAST> constexpr int lines_warp_smem() { return 2 * kStageBytes + kTileBytes + YiqRow<FAST>::kBytes; }
template <bool FAST> constexpr int lines_smem() { return kLinesWarps * lines_warp_smem<FAST>() + kLinesWarps * 2 * 8; }

// MAXP == 2 instantiations need dx >= 2048, i.e. outw <= kTwoPixelOutw; anything wider (up to
// kMaxOutw, where a single sample can still not overrun the 32-column tile ring) takes MAXP == 0.
constexpr int kMaxOutw = 8192;

struct LinesGeom { // uniform over a launch: host groups monitors by these (crtx.cu)
    int outw, out_format, bpp, blend;
    int pitch; // bytes between output rows (MonCfg::out_pitch, shared by every monitor of the launch)
    int pass; // -1: every line; -2: only the last line of each shared-row run; >= 0: lines at this run position
    int rnd; // 32768, passed as an argument so that it lives in a register (see pole())
    int dx;  // ((AV_LEN - 1) << 12) / outw (crt_core.c:527), computed by the host: no division in the kernels
    int line_lo, line_hi; // decoded lines [lo, hi) this launch may touch (scanline-block sharding across ranks)
};

// The 16-byte row path of k_lines and k_lines_fir (and a condition of k_lines2): 4-byte pixels, rows of whole 16-byte
// groups that start on 16-byte boundaries (the image's address and its pitch multiples of 16).  crtx_get_paths reports it.
__host__ __device__ inline bool rows16_ok(const void *out, int pitch, int outw, int bpp)
{
    return bpp == 4 && (outw & 3) == 0 && ((reinterpret_cast<uintptr_t>(out) | (uintptr_t) pitch) & 15) == 0;
}

// Write `cnt` (<= 16) finished pixels [k0, k0 + cnt) of every active line of this warp
// (crt_core.c:584-664).  The tile holds 16 pixel columns per line; pixels are already in storage byte
// order and, when blending, pre-halved with the alpha byte forced to 0xff, so the blend is
// (old >> 1 & mask) + new on whole words.
//
// 128-bit path (4-byte pixels, rows that start on 16-byte boundaries: image address and pitch multiples of 16): 4 lanes per row, 8 rows per pass, 4 passes.  Each
// lane keeps, for its 4 (row, quad) slots, the row pointer and the number of rows to write
// (crt_core.c:662-664), and -- when blending -- the previous image's pixels of the NEXT 16-pixel block,
// fetched right after this block is written so that the DRAM latency hides behind a whole sub-chunk
// of filter work instead of stalling the flush.
struct RowSlots {
    unsigned char *ptr[4]; // row start of line it * 8 + (lane >> 2), plus this lane's quad offset
    int rows[4];           // rows to write, 0 = slot inactive
};

template <bool BLEND>
__device__ __forceinline__ void load_old(const RowSlots &rs, int k0, int cnt, int lane, uint4 (&oldv)[4])
{
    if (!BLEND) return;
#pragma unroll
    for (int it = 0; it < 4; it++)
        if (rs.rows[it] > 0 && 4 * (lane & 3) < cnt)
            oldv[it] = *reinterpret_cast<const uint4 *>(rs.ptr[it] + (size_t) k0 * 4);
}

template <bool BLEND>
__device__ __forceinline__ void flush16_vec(const unsigned *tile, const RowSlots &rs, int pitch, int k0, int cnt,
                                            int lane, unsigned blend_mask, const uint4 (&oldv)[4])
{
    __syncwarp();
#pragma unroll
    for (int it = 0; it < 4; it++) {
        if (rs.rows[it] > 0 && 4 * (lane & 3) < cnt) {
            uint4 v = *reinterpret_cast<const uint4 *>(tile + (it * 8 + (lane >> 2)) * kTilePitch + 4 * (lane & 3));
            if (BLEND) {
                v.x += (oldv[it].x >> 1) & blend_mask;
                v.y += (oldv[it].y >> 1) & blend_mask;
                v.z += (oldv[it].z >> 1) & blend_mask;
                v.w += (oldv[it].w >> 1) & blend_mask;
            }
            unsigned char *p = rs.ptr[it] + (size_t) k0 * 4;
            for (int r = 0; r < rs.rows[it]; r++) *reinterpret_cast<uint4 *>(p + (size_t) r * pitch) = v;
        }
    }
    __syncwarp();
}

// scalar path: 3-byte pixels, or rows that are not 16-byte aligned; 16 lanes per row, 2 rows per pass
__device__ __forceinline__ void flush16_scalar(const unsigned *tile, const LinesGeom &geo, unsigned char *out, int k0,
                                               int cnt, int lane, int beg, int nrows, unsigned blend_mask)
{
    const int pitch = geo.pitch;
    int rp, gp, bp;
    fmt_positions(geo.out_format, rp, gp, bp);
    const int j = lane & 15;
    __syncwarp();
#pragma unroll 1
    for (int it = 0; it < 16; it++) {
        const int l = it * 2 + (lane >> 4);
        const int lbeg = __shfl_sync(0xffffffffu, beg, l);
        const int lrows = __shfl_sync(0xffffffffu, nrows, l);
        if (lbeg >= 0 && j < cnt) {
            unsigned v = tile[l * kTilePitch + j];
            unsigned char *p = out + (size_t) lbeg * pitch + (size_t) (k0 + j) * geo.bpp;
            if (geo.bpp == 4) {
                if (geo.blend) v += (*reinterpret_cast<const unsigned *>(p) >> 1) & blend_mask;
                for (int r = 0; r < lrows; r++) *reinterpret_cast<unsigned *>(p + (size_t) r * pitch) = v;
            } else { // 3 bytes per pixel: the tile word is 0x00RRGGBB (pre-halved when blending)
                if (geo.blend) {
                    const unsigned old = (unsigned) p[rp] << 16 | (unsigned) p[gp] << 8 | (unsigned) p[bp];
                    v += (old >> 1) & 0x7f7f7fu;
                }
                for (int r = 0; r < lrows; r++) {
                    unsigned char *d = p + (size_t) r * pitch;
                    d[rp] = (unsigned char) (v >> 16);
                    d[gp] = (unsigned char) (v >> 8);
                    d[bp] = (unsigned char) v;
                }
            }
        }
    }
    __syncwarp();
}

// Template axes (chosen by the host per launch, so every branch on them is compile-time):
//   FAST  see eq_step; the other instantiation takes the monitors k_sync flagged as generic
//   MODE  0: 4-byte pixels, no blend; 1: 4-byte pixels, blend; 2: 3-byte pixels (blend at run time)
//   FMT   the CRT_PIX_FORMAT of the 4-byte modes (byte order and alpha position become immediates);
//         ignored (0) for MODE 2
//
// Per warp, per 16-sample sub-chunk: (F) one straight-line filter block per sample writes packed
// Y/I/Q into the lane's own shared-memory row; (P) a uniform loop walks the output pixels whose two
// source samples are now available, reading slots by a warp-uniform index -- so neither phase has
// per-sample control flow and the register allocator sees two simple loops.
template <bool FAST, int MODE, int FMT>
__global__ void __launch_bounds__(kLinesWarps * 32, (FAST && kCc == 4) ? 2 : 1) // (the PV-1000 stages fill shared memory: one CTA per SM)
k_lines(const MonCfg *__restrict__ cfgs, const MonState *__restrict__ states, const LineRec *__restrict__ lines_base,
        const signed char *__restrict__ inp_base, int first, const LinesGeom geo)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int kWarpSmem = lines_warp_smem<FAST>();
    constexpr int kEntry = YiqRow<FAST>::kEntryBytes;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = first + blockIdx.x;
    if ((states[m].generic != 0) == FAST) return; // the other instantiation handles this monitor
    if (geo.bpp == 0 || geo.outw <= 0) return;

    unsigned char *stage = smem_raw + warp * kWarpSmem;
    unsigned *tile = reinterpret_cast<unsigned *>(stage + 2 * kStageBytes);
    unsigned char *yiq = stage + 2 * kStageBytes + kTileBytes + lane * (YiqRow<FAST>::kPitch * kEntry);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + kLinesWarps * kWarpSmem) + 2 * warp;
    if (lane == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
    }
    __syncwarp();

    const int kline = warp * 32 + lane; // decoded line of this lane
    LineRec rec;
    rec.pos = 0; rec.wave0 = rec.wave1 = 0; rec.beg = -1; rec.end = -1; rec.hsync = 0;
    if (kline < kLines) rec = lines_base[(size_t) m * kLines + kline];
    const bool active = (kline < kLines) && rec.beg >= 0 && kline >= geo.line_lo && kline < geo.line_hi
                     && (geo.pass == -1 || (geo.pass == -2 ? rec.pad1 != 0 : rec.pad0 == geo.pass));
    const unsigned active_mask = __ballot_sync(0xffffffffu, active);
    if (active_mask == 0) return;
    const unsigned nactive = __popc(active_mask);

    // per-monitor scalars (data only; nothing below branches on them)
    const MonCfg *cfg = &cfgs[m];
    const int contrast = cfg->contrast;
    const int bright = cfg->brightness - (kBlack + cfg->black_point); // crt_core.c:304
    unsigned char *out = cfg->out;
    const int beg = active ? rec.beg : -1;
    const int nrows = active ? max(1, rec.end - cfg->scanlines - rec.beg) : 0; // crt_core.c:662-664
    const bool vec = (MODE != 2) && rows16_ok(out, geo.pitch, geo.outw, 4);
    LinesGeom fgeo = geo; // what the scalar flush branches on, pinned to the template mode
    fgeo.bpp = (MODE == 2) ? 3 : 4;
    if (MODE != 2) fgeo.blend = (MODE == 1);
    const int pitch = geo.pitch;
    RowSlots rs;
    uint4 oldv[4];
#pragma unroll
    for (int it = 0; it < 4; it++) {
        const int l = it * 8 + (lane >> 2);
        const int lbeg = __shfl_sync(0xffffffffu, beg, l);
        const int lrows = __shfl_sync(0xffffffffu, nrows, l);
        rs.ptr[it] = out + (size_t) max(lbeg, 0) * pitch + (size_t) (lane & 3) * 16;
        rs.rows[it] = (vec && lbeg >= 0) ? lrows : 0;
        oldv[it] = make_uint4(0u, 0u, 0u, 0u);
    }

    // storage byte order of 0x00RRGGBB (+ alpha 0xff) for the 4-byte formats (crt_core.h:62-67)
    constexpr unsigned sel_store = (FMT == CRT_PIX_FORMAT_RGBA) ? 0x4012u : (FMT == CRT_PIX_FORMAT_ARGB) ? 0x0124u
                                 : (FMT == CRT_PIX_FORMAT_ABGR) ? 0x2104u : 0x4210u;
    constexpr unsigned alpha_ff = (FMT == CRT_PIX_FORMAT_ARGB || FMT == CRT_PIX_FORMAT_ABGR) ? 0x000000ffu : 0xff000000u;
    constexpr unsigned blend_mask = (MODE != 2) ? (0x7f7f7f7fu & ~(alpha_ff >> 1) & ~alpha_ff) : 0x7f7f7fu;

    const int dx = geo.dx; // crt_core.c:527
    // carrier value that multiplies sample i for I and for Q, by i % kCc
    int wi[5], wq[5];
    if (kCc == 4) { // wave[(i + 0) & 3] feeds I, wave[(i + 3) & 3] feeds Q (crt_core.c:538-543)
        const int nw0 = wsub(0, rec.wave0), nw1 = wsub(0, rec.wave1);
        wi[0] = rec.wave0; wi[1] = rec.wave1; wi[2] = nw0; wi[3] = nw1; wi[4] = 0;
        wq[0] = nw1; wq[1] = rec.wave0; wq[2] = rec.wave1; wq[3] = nw0; wq[4] = 0;
    } else { // waveI[i % 5], waveQ[i % 5] from the record's dci / dcq (crt_core.c:497-508, 545-549)
        pv1k_waves(rec.wave0, rec.wave1, cfg->hue, cfg->saturation, wi, wq);
    }
    const int rnd = geo.rnd;

    const signed char *inp = inp_base + (size_t) m * kSignalBytes;
    const int a = rec.pos & 15; // byte offset of the window inside its 16-byte aligned stage row
    const signed char *src = inp + (rec.pos & ~15);
    const signed char *row_base = reinterpret_cast<const signed char *>(stage) + lane * kStageRow + a;
    unsigned *tile_row = tile + lane * kTilePitch;

    auto issue = [&](int c) {
        unsigned char *dst = stage + (c & 1) * kStageBytes + lane * kStageRow;
        if (lane == 0) mbar_expect_tx(&bars[c & 1], nactive * kStageRow);
        __syncwarp();
        if (active) tma_load_1d(dst, src + c * kStageSamples, kStageRow, &bars[c & 1]);
    };

    // slot access.  FAST stores {Y, I | Q << 16} with Y NOT yet scaled by 16: there
    // (Y*16*L >> 2) + (Y'*16*R >> 2) == 4*(Y*L + Y'*R) exactly (no bits are lost, nothing wraps), so the
    // pixel pass folds the scale into its weights.  The generic path keeps {Y*16, I, Q} verbatim.
    auto put = [&](int slot, int y, int ci, int cq) {
        if (FAST) {
            *reinterpret_cast<uint2 *>(yiq + slot * kEntry) =
                make_uint2((unsigned) y, __byte_perm((unsigned) ci, (unsigned) cq, 0x5410));
        } else {
            *reinterpret_cast<uint4 *>(yiq + slot * kEntry) =
                make_uint4((unsigned) wmul(y, 16), (unsigned) ci, (unsigned) cq, 0u);
        }
    };
    auto get = [&](const unsigned char *p, int &cy, int &ci, int &cq) {
        if (FAST) {
            // (one 8-byte load and an unpacking rather than 16-bit sign-extending loads of the halves: per-lane
            // rows make those 2-way bank conflicted)
            const uint2 v = *reinterpret_cast<const uint2 *>(p);
            cy = (int) v.x;
            ci = (int) (short) (unsigned short) v.y; // sign-extended low half
            cq = ((int) v.y) >> 16;
        } else {
            const uint4 v = *reinterpret_cast<const uint4 *>(p);
            cy = (int) v.x;
            ci = (int) v.y;
            cq = (int) v.z;
        }
    };

    Eq ey, ei, eq;
    eq_reset(ey);
    eq_reset(ei);
    eq_reset(eq);
    int k = 0;         // next output pixel       (uniform)
    int kdone = 0;     // pixels already flushed  (uniform, multiple of 16)
    unsigned npos = 0; // k * dx, 20.12 position  (uniform)

    auto drain = [&](int cnt) { // write pixels [kdone, kdone + cnt), then fetch the next block's old pixels
        if (vec) {
            flush16_vec<MODE == 1>(tile, rs, pitch, kdone, cnt, lane, blend_mask, oldv);
            load_old<MODE == 1>(rs, kdone + 16, min(16, geo.outw - kdone - 16), lane, oldv);
        } else {
            flush16_scalar(tile, fgeo, out, kdone, cnt, lane, beg, nrows, blend_mask);
        }
    };

    issue(0);
    if (vec) load_old<MODE == 1>(rs, 0, min(16, geo.outw), lane, oldv);
#pragma unroll 1
    for (int c = 0; c < kNumStages; c++) {
        if (c + 1 < kNumStages) issue(c + 1); // the other buffer was drained in iteration c - 1
        mbar_wait(&bars[c & 1], (c >> 1) & 1);
        const signed char *row = row_base + (c & 1) * kStageBytes;
        const int ns = min(kStageSamples, kSamplesPadded - c * kStageSamples); // a multiple of kSub
#pragma unroll 1
        for (int u = 0; u < ns; u += kSub) {
            // ---- (F) filter kSub samples, straight line; sample index i = c * kStageSamples + u + t -> slot t + 1
            const signed char *rp = row + u;
#pragma unroll
            for (int t = 0; t < kSub; t++) {
                const int s = rp[t];
                const int y = eq_step<kEqYlf, kEqYhf, kEqYg1, kEqYg2, FAST, true>(ey, s + bright, rnd);
                const int ci = eq_step<kEqIlf, kEqIhf, 65536, kEqIg2, FAST, false>(ei, wmul(s, wi[t % kCc]) >> 9, rnd) >> 3;
                const int cq = eq_step<kEqQlf, kEqQhf, 65536, 0, FAST, false>(eq, wmul(s, wq[t % kCc]) >> 9, rnd) >> 3;
                put(t + 1, y, ci, cq);
            }
            // ---- (P) every pixel whose samples (s, s + 1) are both in slots 0..kSub (crt_core.c:555-659)
            const int base = c * kStageSamples + u - 1; // sample index held by slot 0
            // pixel k (position npos = k * dx) is computable once sample (npos >> 12) + 1 <= base + kSub
            // exists, and exists at all while npos < outw * dx (<= scanR, crt_core.c:529,555)
            const unsigned lim = min((unsigned) (base + kSub) << 12, (unsigned) geo.outw * (unsigned) dx);
            const unsigned char *slot0 = yiq - base * kEntry; // slot of sample s is slot0 + s * kEntry
#pragma unroll 1
            while (npos < lim) {
                const unsigned char *sp = slot0 + (npos >> 12) * kEntry;
                const int R = (int) (npos & 0xfffu), L = 0xfff - R;
                int ay, ai, aq, by, bi, bq;
                get(sp, ay, ai, aq);
                get(sp + kEntry, by, bi, bq);
                unsigned px;
                // when blending, the channels are halved while they are clamped (see yiq_to_rgb) instead of afterwards:
                // two instructions less per pixel (59 -> 57 in the SASS of this loop)
                constexpr bool kHalved = MODE == 1;
                if (FAST) {
                    const int y = wadd(wmul(ay, 4 * L), wmul(by, 4 * R));
                    px = yiq_to_rgb<kHalved>(y, wadd(wmul(ai, L) >> 14, wmul(bi, R) >> 14),
                                             wadd(wmul(aq, L) >> 14, wmul(bq, R) >> 14), contrast);
                } else {
                    px = yiq_pixel<kHalved>(ay, ai, aq, by, bi, bq, R, L, contrast);
                }
                if (MODE != 2) {
                    px = (FMT == CRT_PIX_FORMAT_BGRA) ? (px | alpha_ff) : __byte_perm(px, 0xffu, sel_store);
                    if (MODE == 1 && !kHalved) px = ((px >> 1) & blend_mask) | alpha_ff;
                } else if (geo.blend) {
                    px = (px >> 1) & 0x7f7f7fu;
                }
                const int col = k - kdone; // 0..15: the tile restarts after every drain
                tile_row[col] = px;
                k++;
                npos += (unsigned) dx;
                if (col == 15) {
                    drain(16);
                    kdone += 16;
                }
            }
            { // carry the newest sample into slot 0 for the next sub-chunk
                if (FAST) {
                    *reinterpret_cast<uint2 *>(yiq) = *reinterpret_cast<const uint2 *>(yiq + kSub * kEntry);
                } else {
                    *reinterpret_cast<uint4 *>(yiq) = *reinterpret_cast<const uint4 *>(yiq + kSub * kEntry);
                }
            }
        }
        __syncwarp(); // all lanes are done with this stage buffer before it is refilled
    }
    if (k - kdone > 0) drain(k - kdone);
}

} // namespace crt
