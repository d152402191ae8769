// crt_lines2.cuh -- k_lines2, the line pass of crt_demodulate (crt_core.c:511-664) for the geometries the drivers
// actually use: stock equaliser gains on their exact fast path (see eq_step), 4-byte pixels, 16-byte aligned rows,
// an output about as wide as the line has samples (kL2MinDx4096 .. kL2MaxOutw).  Everything else -- 3-byte pixels,
// very narrow or very wide outputs, the wrap-exact generic equaliser, rows shared by several lines, the PV-1000 --
// stays with k_lines (crt_lines.cuh); the host picks per launch (crtx.cu: lines2_eligible).
//
// Same shape as k_lines -- one LANE carries one scanline through the equalisers -- with three changes:
//   * a CTA is 15 warps = 480 lane-lines = TWO monitors.  240 lines are 7.5 warps: k_lines leaves half a warp
//     empty per monitor (1/16 of all issued instructions);
//   * the resampler's index arithmetic is gone from the instruction stream.  Which two samples pixel k reads and
//     with what weights depends on outw only (crt_core.c:527, 559-570), so the CTA tabulates it once in shared
//     memory as 16-byte descriptors {4R, 4L, byte offset of the left sample in the lane's ring, last sample needed};
//     the pixel pass is a fully unrolled block of 8 pixels whose descriptors arrive by one broadcast LDS.128 each
//     and whose tile stores have immediate offsets: 16 integer instructions per pixel of loop control and address
//     arithmetic in k_lines (they are warp-uniform, but ptxas keeps them on the vector pipes) become 1;
//   * the filter block no longer adds the brightness to every sample: a one-pole stage is translation invariant
//     (f' - b = (f - b) + ((C * ((in - b) - (f - b)) + 32768) >> 16)), so the luma cascade runs on the raw samples
//     from the state -bright and the constant joins the pixel's first multiply-add as its addend.
// Decoded Y/I/Q go to a per-lane ring of 24 samples (two filter sub-chunks) + one guard slot that repeats slot 0,
// so "sample s + 1" is always the next slot; a block of 8 pixels is emitted as soon as its last sample is in the
// ring, which the host guarantees is before its first one is overwritten (7 * dx <= 10 * 4096).
// Nothing in the loops waits on DRAM with a register: the signal windows arrive by per-lane asynchronous copies (48
// bytes per lane and stage: three 16-byte cp.async), the previous image's pixels of the NEXT tile by cp.async into
// shared memory while the current tile is being computed, and all shared-memory traffic of the hot loops goes through
// 32-bit shared addresses held in registers.
#pragma once

#include "crt_lines.cuh"

// the builds that have this kernel: four samples per chroma period (not the PV-1000), the IIR equaliser, no bloom
#define CRTX_HAS_LINES2 ((CRT_CC_SAMPLES == 4) && (CRTX_CONV == 0) && (CRT_DO_BLOOM == 0))
#if CRTX_HAS_LINES2

namespace crt {

constexpr int kL2Warps = 15;
constexpr int kL2Threads = kL2Warps * 32;      // 480 lane-lines = two monitors (kLines == 240)
constexpr int kL2Stage = 2 * kSub;             // samples per staged chunk = 2 filter sub-chunks
constexpr int kL2StageRow = ((kL2Stage + 15 + 15) / 16) * 16; // 48 bytes: the aligned superset of a window at any byte phase
constexpr int kL2StageBytes = 32 * kL2StageRow;
constexpr int kL2Stages = (kSamplesPadded + kL2Stage - 1) / kL2Stage;
constexpr int kL2Ring = 2 * kSub;              // slots; slot of sample s is s % kL2Ring
constexpr int kL2RingPitch = kL2Ring + 1;      // + guard slot; odd => "all lanes, same slot" is conflict free
constexpr int kL2RingBytes = 32 * kL2RingPitch * 8;
constexpr int kL2Block = 8;                    // pixels per unrolled block; the tile is flushed every two blocks
constexpr int kL2OldBytes = 4 * 32 * 16;       // previous-image pixels of the next tile: [row pass][lane] x 16 bytes
constexpr int kL2WarpSmem = 2 * kL2StageBytes + kTileBytes + kL2RingBytes + kL2OldBytes;
constexpr int kL2MaxOutw = 1312;               // descriptor table: 16 bytes per pixel of shared memory, what is left of 227 KB
static_assert(kLines * 2 == kL2Threads, "two monitors per CTA");
static_assert(kL2Stage % kSub == 0 && kL2StageRow % 16 == 0 && kSamplesPadded % kSub == 0, "stage layout");
static_assert(kL2RingPitch % 2 == 1, "ring pitch");

__host__ __device__ constexpr int lines2_desc_count(int outw) { return ((outw + 15) / 16) * 16; }
__host__ __device__ constexpr int lines2_smem(int outw)
{
    return kL2Warps * kL2WarpSmem + lines2_desc_count(outw) * 16;
}
static_assert(lines2_smem(kL2MaxOutw) <= 227 * 1024, "k_lines2 shared memory");

// the geometries k_lines2 takes (the rest of the conditions -- pixel size, row alignment, fast equaliser -- are the caller's)
__host__ __device__ inline bool lines2_geometry_ok(int outw)
{
    if (kCc != 4 || outw < 16 || outw > kL2MaxOutw || (outw & 3)) return false;
    const long long dx = ((long long) (kAvLen - 1) << 12) / outw;
    return 7 * dx <= 10 * 4096; // a block's 8 pixels span at most 12 samples: its first is still in the ring (see above)
}

// Row pointers of the 16-pixel tile a warp is about to write: lane (q = lane & 3, r = lane >> 2) owns the 16-byte quad q of
// the rows of lines r, r + 8, r + 16, r + 24.  The pointers walk along the rows, 64 bytes per tile.
struct TileRows {
    unsigned char *ptr[4]; // current tile, this lane's quad
    int rows[4];           // rows to write (crt_core.c:662-664), 0 = slot inactive
};

// Write one tile (crt_core.c:584-664): 4 passes x (LDS.128 of new pixels, LDS.128 of the previous image's pixels that a
// cp.async put into shared memory a tile ago, blend on whole words, st.global.v4 to every row of the line), then move
// on to the next tile and request ITS previous pixels.  No register ever waits on DRAM.
template <bool BLEND>
__device__ __forceinline__ void flush_tile(unsigned tile_q_a, unsigned old_a, TileRows &tr, int pitch, int cnt, int cnt_next,
                                           int lane, unsigned blend_mask)
{
    __syncwarp();
    if (BLEND) cp_async_wait<0>(); // (each lane reads back only what it copied itself)
    const bool mine = 4 * (lane & 3) < cnt, mine_next = 4 * (lane & 3) < cnt_next;
#pragma unroll
    for (int it = 0; it < 4; it++) {
        if (tr.rows[it] > 0 && mine) {
            uint4 v = (it == 0) ? lds_u4<0>(tile_q_a) : (it == 1) ? lds_u4<8 * kTilePitch * 4>(tile_q_a)
                    : (it == 2) ? lds_u4<16 * kTilePitch * 4>(tile_q_a) : lds_u4<24 * kTilePitch * 4>(tile_q_a);
            if (BLEND) {
                const uint4 o = (it == 0) ? lds_u4<0>(old_a) : (it == 1) ? lds_u4<512>(old_a) : (it == 2) ? lds_u4<1024>(old_a) : lds_u4<1536>(old_a);
                v.x += (o.x >> 1) & blend_mask;
                v.y += (o.y >> 1) & blend_mask;
                v.z += (o.z >> 1) & blend_mask;
                v.w += (o.w >> 1) & blend_mask;
            }
            unsigned char *p = tr.ptr[it];
            stg_u4(p, v);
            if (tr.rows[it] > 1) {
                stg_u4(p + pitch, v);
                for (int r = 2; r < tr.rows[it]; r++) stg_u4(p + (size_t) r * pitch, v);
            }
        }
        tr.ptr[it] += 64;
        if (BLEND && tr.rows[it] > 0 && mine_next) cp_async_16a(old_a + it * 512, tr.ptr[it]);
    }
    if (BLEND) cp_async_commit();
    __syncwarp();
}

template <int MODE, int FMT> // MODE 0: no blend, 1: blend; FMT: one of the four 4-byte CRT_PIX_FORMATs
__global__ void __launch_bounds__(kL2Threads, 1)
k_lines2(const MonCfg *__restrict__ cfgs, const MonState *__restrict__ states, const LineRec *__restrict__ lines_base,
         const signed char *__restrict__ inp_base, int first, int count, const LinesGeom geo)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint4 *desc = reinterpret_cast<uint4 *>(smem_raw + kL2Warps * kL2WarpSmem);
    const int dx = geo.dx;
    phase_mark(1, 0);

    // ---- descriptor table, once per CTA (pixels past outw repeat the last one: they are computed and never stored)
    const int ndesc = lines2_desc_count(geo.outw);
    for (int k = threadIdx.x; k < ndesc; k += kL2Threads) {
        const unsigned npos = (unsigned) min(k, geo.outw - 1) * (unsigned) dx;
        const unsigned s = npos >> 12, R = npos & 0xfffu;
        desc[k] = make_uint4(4u * R, 4u * (0xfffu - R), (s % (unsigned) kL2Ring) * 8u, s + 1u);
    }
    __syncthreads();
    phase_mark(1, 1);

    const int gl = warp * 32 + lane;           // lane-line of the CTA
    const int half = gl >= kLines ? 1 : 0;
    const int kline = gl - half * kLines;      // decoded line of this lane
    const int mrel = 2 * blockIdx.x + half;
    const bool present = mrel < count;
    const int m = first + (present ? mrel : 0);

    unsigned char *stage = smem_raw + warp * kL2WarpSmem;
    // 32-bit shared-space addresses of everything the hot loops touch
    const unsigned stage_a = smem_u32(stage);
    const unsigned tile_a = stage_a + 2 * kL2StageBytes;
    const unsigned tile_row_a = tile_a + lane * (kTilePitch * 4);                                    // P phase: this lane's line
    const unsigned tile_q_a = tile_a + ((lane >> 2) * kTilePitch + 4 * (lane & 3)) * 4;             // flush: this lane's quad
    const unsigned yiq_a = tile_a + kTileBytes + lane * (kL2RingPitch * 8);
    const unsigned old_a = tile_a + kTileBytes + kL2RingBytes + lane * 16;
    const unsigned desc_a = smem_u32(desc);

    LineRec rec;
    rec.pos = 0; rec.wave0 = rec.wave1 = 0; rec.beg = -1; rec.end = -1; rec.hsync = 0; rec.pad0 = rec.pad1 = 0;
    if (present) rec = lines_base[(size_t) m * kLines + kline];
    const bool active = present && states[m].generic == 0 && rec.beg >= 0 && kline >= geo.line_lo && kline < geo.line_hi;
    const unsigned active_mask = __ballot_sync(0xffffffffu, active);
    if (active_mask == 0) return;

    const MonCfg *cfg = &cfgs[m];
    const int contrast = cfg->contrast;
    const int bright = cfg->brightness - (kBlack + cfg->black_point); // crt_core.c:304
    const int ybias = wmul(bright, 4 * 0xfff);                        // 4 * (L + R) * bright, see the header
    unsigned char *out = cfg->out;
    const int beg = active ? rec.beg : -1;
    const int nrows = active ? max(1, rec.end - cfg->scanlines - rec.beg) : 0; // crt_core.c:662-664
    const int pitch = geo.pitch;
    TileRows tr;
#pragma unroll
    for (int it = 0; it < 4; it++) {
        const int l = it * 8 + (lane >> 2);
        const int lbeg = __shfl_sync(0xffffffffu, beg, l);
        const int lrows = __shfl_sync(0xffffffffu, nrows, l);
        const unsigned long long lout = __shfl_sync(0xffffffffu, (unsigned long long) reinterpret_cast<uintptr_t>(out), l);
        tr.ptr[it] = reinterpret_cast<unsigned char *>((uintptr_t) lout) + (size_t) max(lbeg, 0) * pitch + (size_t) (lane & 3) * 16;
        tr.rows[it] = (lbeg >= 0) ? lrows : 0;
    }

    // storage byte order of 0x00RRGGBB (+ alpha 0xff) for the 4-byte formats (crt_core.h:62-67)
    constexpr unsigned sel_store = (FMT == CRT_PIX_FORMAT_RGBA) ? 0x4012u : (FMT == CRT_PIX_FORMAT_ARGB) ? 0x0124u
                                 : (FMT == CRT_PIX_FORMAT_ABGR) ? 0x2104u : 0x4210u;
    constexpr unsigned alpha_ff = (FMT == CRT_PIX_FORMAT_ARGB || FMT == CRT_PIX_FORMAT_ABGR) ? 0x000000ffu : 0xff000000u;
    constexpr unsigned blend_mask = 0x7f7f7f7fu & ~(alpha_ff >> 1) & ~alpha_ff;
    constexpr bool kHalved = MODE == 1; // when blending the channels are halved while they are clamped (yiq_to_rgb)

    // carrier value that multiplies sample i for I and for Q, by i % 4 (crt_core.c:538-543)
    int wi[4], wq[4];
    {
        const int nw0 = wsub(0, rec.wave0), nw1 = wsub(0, rec.wave1);
        wi[0] = rec.wave0; wi[1] = rec.wave1; wi[2] = nw0; wi[3] = nw1;
        wq[0] = nw1; wq[1] = rec.wave0; wq[2] = rec.wave1; wq[3] = nw0;
    }
    const int rnd = geo.rnd;

    const signed char *inp = inp_base + (size_t) m * kSignalBytes;
    // stage c holds samples [c * kL2Stage, + kL2Stage) of the window: copied from the 16-byte aligned address at or
    // below its first sample (asynchronous copies move whole 16-byte words), found at byte (pos + c * kL2Stage) & 15
    const signed char *row_base = reinterpret_cast<const signed char *>(stage) + lane * kL2StageRow;

    auto issue = [&](int c) { // request stage c: samples [c * kL2Stage, + kL2Stage) of every active lane's window
        unsigned char *dst = stage + (c & 1) * kL2StageBytes + lane * kL2StageRow;
        const signed char *src = inp + ((rec.pos + c * kL2Stage) & ~15);
        if (active) {
#pragma unroll
            for (int q = 0; q < kL2StageRow / 16; q++) cp_async_16(dst + 16 * q, src + 16 * q);
        }
        cp_async_commit();
    };

    Eq ey, ei, eq;
    eq_reset(ei);
    eq_reset(eq);
    { // luma on the raw samples: every state starts at 0 - bright
        const int nb = wsub(0, bright);
        ey.l0 = ey.l1 = ey.l2 = ey.l3 = ey.h0 = ey.h1 = ey.h2 = ey.h3 = ey.s1 = ey.s2 = ey.s3 = nb;
    }
    const int nblk = (geo.outw + kL2Block - 1) / kL2Block;
    int blk = 0;  // next pixel block (uniform)
    int sub = 0;  // filter sub-chunk counter (uniform)

    issue(0);
    if (MODE == 1) { // previous pixels of tile 0
        const bool mine0 = 4 * (lane & 3) < min(16, geo.outw);
#pragma unroll
        for (int it = 0; it < 4; it++)
            if (tr.rows[it] > 0 && mine0) cp_async_16a(old_a + it * 512, tr.ptr[it]);
        cp_async_commit();
    }
#pragma unroll 1
    for (int c = 0; c < kL2Stages; c++) {
        // stage c has had a whole stage of work to arrive
        cp_async_wait<0>();
        __syncwarp(); // ... and every lane is done with the other buffer, which is refilled now
        if (c + 1 < kL2Stages) issue(c + 1);
        const signed char *row = row_base + (c & 1) * kL2StageBytes + ((rec.pos + c * kL2Stage) & 15);
        const int ns = min(kL2Stage, kSamplesPadded - c * kL2Stage); // a multiple of kSub
#pragma unroll 1
        for (int u = 0; u < ns; u += kSub, sub++) {
            // ---- (F) filter kSub samples, straight line; sample sub * kSub + t -> ring slot (sub & 1) * kSub + t
            const signed char *rp = row + u;
            const unsigned yq_a = yiq_a + (sub & 1) * (kSub * 8);
#pragma unroll
            for (int t = 0; t < kSub; t++) {
                const int s = rp[t];
                const int y = eq_step<kEqYlf, kEqYhf, kEqYg1, kEqYg2, true, true>(ey, s, rnd);
                const int ci = eq_step<kEqIlf, kEqIhf, 65536, kEqIg2, true, false>(ei, wmul(s, wi[t % 4]) >> 9, rnd) >> 3;
                const int cq = eq_step<kEqQlf, kEqQhf, 65536, 0, true, false>(eq, wmul(s, wq[t % 4]) >> 9, rnd) >> 3;
                const uint2 e = make_uint2((unsigned) y, __byte_perm((unsigned) ci, (unsigned) cq, 0x5410));
                switch (t) { // (constant offsets: the store is one instruction)
#define CRT_L2_PUT(T) case T: sts_u2<T * 8>(yq_a, e); break;
                    CRT_L2_PUT(0) CRT_L2_PUT(1) CRT_L2_PUT(2) CRT_L2_PUT(3) CRT_L2_PUT(4) CRT_L2_PUT(5) CRT_L2_PUT(6) CRT_L2_PUT(7)
                    CRT_L2_PUT(8) CRT_L2_PUT(9) CRT_L2_PUT(10) CRT_L2_PUT(11)
#undef CRT_L2_PUT
                }
                if (t == 0 && !(sub & 1)) sts_u2<kL2Ring * 8>(yiq_a, e); // guard slot = slot 0
            }
            // ---- (P) every block of 8 pixels whose last sample is now in the ring (crt_core.c:555-659)
            const unsigned have = (unsigned) (sub * kSub + kSub - 1); // newest sample index filtered
#pragma unroll 1
            while (blk < nblk) {
                const unsigned dp_a = desc_a + blk * (kL2Block * 16);
                if (lds_u1<(kL2Block - 1) * 16 + 12>(dp_a) > have) break;
                const unsigned tp_a = tile_row_a + (blk & 1) * (kL2Block * 4);
                // software pipeline: pixel j + 1's descriptor and samples are requested before pixel j's arithmetic
                uint4 d = lds_u4<0>(dp_a);
                uint2 va = lds_u2<0>(yiq_a + d.z), vb = lds_u2<8>(yiq_a + d.z);
#define CRT_L2_PIXEL(J)                                                                                                   \
                {                                                                                                         \
                    const int R4 = (int) d.x, L4 = (int) d.y;                                                             \
                    const uint2 ca = va, cb = vb;                                                                         \
                    if (J + 1 < kL2Block) {                                                                               \
                        d = lds_u4<((J + 1) % kL2Block) * 16>(dp_a);                                                      \
                        va = lds_u2<0>(yiq_a + d.z);                                                                      \
                        vb = lds_u2<8>(yiq_a + d.z);                                                                      \
                    }                                                                                                     \
                    const int ai = (int) (short) (unsigned short) ca.y, aq = ((int) ca.y) >> 16;                          \
                    const int bi = (int) (short) (unsigned short) cb.y, bq = ((int) cb.y) >> 16;                          \
                    /* (Y*16*L >> 2) + (Y'*16*R >> 2) == 4*(Y*L + Y'*R) exactly; (I*L >> 14) == (I*4L >> 16) */           \
                    const int y = wadd(wmul((int) ca.x, L4), wadd(wmul((int) cb.x, R4), ybias));                          \
                    unsigned px = yiq_to_rgb<kHalved>(y, wadd(wmul(ai, L4) >> 16, wmul(bi, R4) >> 16),                    \
                                                      wadd(wmul(aq, L4) >> 16, wmul(bq, R4) >> 16), contrast);            \
                    px = (FMT == CRT_PIX_FORMAT_BGRA) ? (px | alpha_ff) : __byte_perm(px, 0xffu, sel_store);              \
                    sts_u1<J * 4>(tp_a, px);                                                                              \
                }
                CRT_L2_PIXEL(0) CRT_L2_PIXEL(1) CRT_L2_PIXEL(2) CRT_L2_PIXEL(3) CRT_L2_PIXEL(4) CRT_L2_PIXEL(5) CRT_L2_PIXEL(6) CRT_L2_PIXEL(7)
#undef CRT_L2_PIXEL
                blk++;
                if (!(blk & 1)) { // two blocks = one 16-pixel tile
                    const int k0 = (blk - 2) * kL2Block;
                    flush_tile<MODE == 1>(tile_q_a, old_a, tr, pitch, min(16, geo.outw - k0), min(16, geo.outw - k0 - 16), lane, blend_mask);
                }
            }
        }
    }
    if (blk & 1) { // odd number of blocks: the last tile holds one
        const int k0 = (blk - 1) * kL2Block;
        flush_tile<MODE == 1>(tile_q_a, old_a, tr, pitch, geo.outw - k0, 0, lane, blend_mask);
    }
    cp_async_wait<0>();
    phase_mark(1, 14);
    phase_mark(1, 12, 7 * 32);
}

} // namespace crt

#endif // CRTX_HAS_LINES2
