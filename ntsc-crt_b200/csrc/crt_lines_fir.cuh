// crt_lines_fir.cuh -- k_lines_fir, the line pass of crt_demodulate for the reference's
// USE_CONVOLUTION 1 build (crt_core.c:85-147 with crt_core.c:511-664): eqf() is the 7-tap kernel
// [1 4 7 8 7 4 1] >> 5 (or, by the reference's other compile-time switches, [1 3 4 4 3 1] >> 4,
// [1 2 2 2 1] >> 3, [1 1 1 1] >> 2) over a history that is zero at the start of every line.
//
// Shape.  Unlike the three-band equaliser (crt_lines.cuh) this filter has no recurrence, so the line
// itself is data parallel: ONE WARP DECODES ONE SCANLINE.
//   in : the line's window of inp[] arrives in shared memory with one 1-D TMA bulk copy (784 bytes,
//        the 16-byte aligned superset of 768 samples at any byte phase), and -- when blending -- so
//        does the previous image's row; both are requested one line ahead (each warp walks several
//        lines of its monitor), so the copies fly while the warp filters;
//   F  : every lane filters 24 consecutive samples (plus a taps - 1 sample run-in that rebuilds the filter
//        history), the kernel factored as [1 1]^(taps - 4) * [1 1 1 1] -- five additions per channel and
//        sample for 7 taps, exact because nothing is rounded before the final shift -- and writes Y/I/Q
//        into the warp's shared-memory rows;
//   P  : lane = output pixel, 32 consecutive pixels per step: resample, YIQ->RGB, contrast, clamp,
//        blend with the previous image IN PLACE in the staged row, which one lane then sends to every
//        output row the line covers (crt_core.c:662-664) as bulk stores; two row buffers alternate so
//        the stores of line n drain, and the previous image of line n + 1 arrives, behind the arithmetic.
#pragma once

#include <type_traits>

#include "crt_lines.cuh"

namespace crt {

constexpr int kFirWarps = 8;                       // lines in flight per CTA
constexpr int kFirChunk = 24;                      // samples per lane: a multiple of 8 (slot padding) and 4 (carrier)
constexpr int kFirSamples = 32 * kFirChunk;        // 768 >= AV_LEN of every system
constexpr int kFirTaps = kConvTaps ? kConvTaps : 7; // (the kernel is only launched in CRTX_CONV builds)
constexpr int kFirHalo = kFirTaps - 1;             // run-in samples that rebuild the history
constexpr int kFirShift = kFirTaps - 2;            // log2 of the weights' sum: 5, 4, 3, 2
constexpr int kFirStage = ((kFirSamples + 15 + 15) / 16) * 16; // staged bytes per line
constexpr int kFirSeg = 832;                       // output pixels staged per bulk load / store
constexpr int kFirIter = kFirSeg / 32;               // pixels per lane and segment
constexpr int kFirGroups = (kLines + kFirWarps - 1) / kFirWarps;
static_assert(!kConv || kFirSamples >= kAvLen, "one warp covers a whole line");
static_assert(kFirChunk % 8 == 0 && kFirChunk % 4 == 0, "slot padding and carrier phase are per-lane constants");
static_assert(kFirSeg % 32 == 0, "whole warp steps per segment");

// Y, I and Q rows of one line, one array per component.  Sample e lives in slot 1 + e + (e >> 3): one pad
// slot after every 8 samples makes the per-lane chunk pitch 27 entries, which spreads "all lanes, same t"
// stores over the banks; the pad slot after samples 8j..8j+7 holds a COPY of sample 8j+8, so the resampler
// always finds sample s + 1 in the slot after sample s.  FAST keeps 16-bit entries, which the resampler
// reads with sign-extending loads; they fit because the kernels have unit DC gain and k_sync only leaves
// a monitor on the FAST path when |bright| <= 4096 (|Y| <= 127 + 4096 before the x16 the pixel pass
// applies) and every chroma input (s * wave) >> 9 is within +-16383 (|I|, |Q| <= 2048 after the >> 3), counting |s| = 128 for a
// line whose window reaches the struct tail behind inp[] (crt_sync.cuh).
template <bool FAST> struct FirRow {
    using Elem = typename std::conditional<FAST, short, int>::type;
    static constexpr int kSlots = 1 + kFirSamples + kFirSamples / 8;
    static constexpr int kCompBytes = ((kSlots * (int) sizeof(Elem) + 15) / 16) * 16;
    static constexpr int kBytes = 3 * kCompBytes;
};
// per warp: two signal stages, the Y/I/Q rows, two output-row segments
template <bool FAST> constexpr int fir_warp_smem() { return 2 * kFirStage + FirRow<FAST>::kBytes + 2 * kFirSeg * 4; }
template <bool FAST> constexpr int fir_smem() { return kFirWarps * fir_warp_smem<FAST>() + kFirWarps * 4 * 8; }

// One channel of the factored kernel.  All four kernels are cascades of [1 1] stages and one box:
//   7 taps [1 4 7 8 7 4 1] = [1 1]^3 * [1 1 1 1]      6 taps [1 3 4 4 3 1] = [1 1]^2 * [1 1 1 1]
//   5 taps [1 2 2 2 1]     = [1 1]   * [1 1 1 1]      4 taps [1 1 1 1]
// (exact: nothing is rounded before the final shift); the 4-wide box is two pair sums.
struct FirChan {
    int a, b, c, d, p1, p2;
};
__device__ __forceinline__ void fir_reset(FirChan &f) { f.a = f.b = f.c = f.d = f.p1 = f.p2 = 0; }
__device__ __forceinline__ int fir_push(FirChan &f, int x)
{
    int v = x;
    if (kFirTaps >= 5) { // first [1 1]
        const int s1 = wadd(v, f.a);
        f.a = v;
        v = s1;
    }
    if (kFirTaps >= 6) { // second [1 1]
        const int s2 = wadd(v, f.b);
        f.b = v;
        v = s2;
    }
    if (kFirTaps == 7) { // third [1 1]
        const int s3 = wadd(v, f.c);
        f.c = v;
        v = s3;
    }
    const int p = wadd(v, f.d); // v[i] + v[i-1]
    f.d = v;
    const int out = wadd(p, f.p2); // + v[i-2] + v[i-3]
    f.p2 = f.p1;
    f.p1 = p;
    return out;
}

// what a warp keeps of a line record
struct FirLine {
    int pos, wave0, wave1, beg, end, run_pos, run_last, index;
};

// Grid: (CTAs per monitor, monitors).  Warp w of CTA x decodes lines (x + n * gridDim.x) * kFirWarps + w,
// n = 0, 1, ... of its monitor; the host picks gridDim.x so that the whole launch is about two waves of
// resident CTAs.  While line n is being decoded the record of line n + 2, the signal window of line
// n + 1 and (from the middle of line n on) the previous image's row of line n + 1 are on their way.
template <bool FAST, int MODE, int FMT>
__global__ void __launch_bounds__(kFirWarps * 32, FAST ? 2 : 1)
k_lines_fir(const MonCfg *__restrict__ cfgs, const MonState *__restrict__ states, const LineRec *__restrict__ lines_base,
            const signed char *__restrict__ inp_base, int first, const LinesGeom geo)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using Elem = typename FirRow<FAST>::Elem;
    constexpr int kComp = FirRow<FAST>::kCompBytes / (int) sizeof(Elem); // elements between the Y, I and Q rows
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = first + blockIdx.y;
    const LineRec *recs = lines_base + (size_t) m * kLines;
    const int stride = (int) gridDim.x * kFirWarps;

    // A record is fetched two lines before it is decoded and must not be LOOKED AT before it is needed:
    // deciding "active" at fetch time would make every line wait for this load.
    auto fetch = [&](int kl) -> FirLine { // warp-uniform
        FirLine l;
        l.pos = l.wave0 = l.wave1 = l.run_pos = l.run_last = 0;
        l.beg = l.end = -1;
        l.index = kl;
        if (kl < kLines) {
            const LineRec r = recs[kl];
            l.pos = r.pos; l.wave0 = r.wave0; l.wave1 = r.wave1; l.beg = r.beg; l.end = r.end;
            l.run_pos = r.pad0; l.run_last = r.pad1;
        }
        return l;
    };
    auto is_active = [&](const FirLine &l) -> bool {
        return l.index < kLines && l.beg >= 0 && l.index >= geo.line_lo && l.index < geo.line_hi
            && (geo.pass == -1 || (geo.pass == -2 ? l.run_last != 0 : l.run_pos == geo.pass));
    };

    // everything the first line needs from global memory, requested together
    int kline = (int) blockIdx.x * kFirWarps + warp;
    const int is_generic = states[m].generic;
    const MonCfg *cfg = &cfgs[m];
    const int contrast = cfg->contrast;
    const int bright = cfg->brightness - (kBlack + cfg->black_point); // crt_core.c:304
    const int scanlines = cfg->scanlines;
    unsigned char *out = cfg->out;
    FirLine cur = fetch(kline);
    FirLine nxt = fetch(kline + stride);
    if ((is_generic != 0) == FAST) return; // the other instantiation handles this monitor
    if (geo.bpp == 0 || geo.outw <= 0) return;

    unsigned char *stage = smem_raw + warp * fir_warp_smem<FAST>();
    Elem *yrow = reinterpret_cast<Elem *>(stage + 2 * kFirStage);
    unsigned *orow = reinterpret_cast<unsigned *>(stage + 2 * kFirStage + FirRow<FAST>::kBytes);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + kFirWarps * fir_warp_smem<FAST>()) + 4 * warp;
    if (lane == 0) {
        mbar_init(&bars[0], 1); // signal stage 0 / 1
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1); // output-row buffer 0 / 1 (previous image, for the blend)
        mbar_init(&bars[3], 1);
        mbar_fence_init();
    }
    __syncwarp();
    unsigned ph_sig = 0, ph_old = 0; // bit b: parity of the next wait on buffer b

    constexpr int bpp = (MODE == 2) ? 3 : 4;
    const int pitch = geo.outw * bpp;
    // rows go through shared memory and bulk copies when they are 16-byte granular; otherwise (3-byte
    // pixels, odd widths, unaligned images) every lane reads and writes its own pixels
    const bool bulk = (MODE != 2) && ((geo.outw & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    const bool prefetch_old = bulk && (MODE == 1);
    const signed char *inp = inp_base + (size_t) m * kSignalBytes;
    const unsigned dx = (unsigned) (((kAvLen - 1) << 12) / geo.outw); // crt_core.c:527
    const int seg0 = min(geo.outw, kFirSeg);
    constexpr unsigned sel_store = (FMT == CRT_PIX_FORMAT_RGBA) ? 0x4012u : (FMT == CRT_PIX_FORMAT_ARGB) ? 0x0124u
                                 : (FMT == CRT_PIX_FORMAT_ABGR) ? 0x2104u : 0x4210u;
    constexpr unsigned alpha_ff = (FMT == CRT_PIX_FORMAT_ARGB || FMT == CRT_PIX_FORMAT_ABGR) ? 0x000000ffu : 0xff000000u;
    constexpr unsigned blend_mask = 0x7f7f7f7fu & ~(alpha_ff >> 1) & ~alpha_ff;
    constexpr unsigned blend_even = 0xfefefefeu & ~alpha_ff; // (x & blend_even) >> 1 == (x >> 1) & blend_mask
    int rp = 0, gp = 0, bp = 0;
    if (MODE == 2) fmt_positions(geo.out_format, rp, gp, bp);

    auto request_signal = [&](const FirLine &l, int buf) { // one lane
        mbar_expect_tx(&bars[buf], kFirStage);
        tma_load_1d(stage + buf * kFirStage, inp + (l.pos & ~15), kFirStage, &bars[buf]);
    };
    auto request_old = [&](const FirLine &l, int buf, int k0, int cnt) { // one lane
        mbar_expect_tx(&bars[2 + buf], cnt * 4);
        tma_load_1d(orow + buf * kFirSeg, out + (size_t) l.beg * pitch + (size_t) k0 * 4, cnt * 4, &bars[2 + buf]);
    };

    // Where output pixel k0 + 32 u + lane reads its samples and with which weight depends only on the
    // output width: every lane keeps that for its (at most kFirIter) pixels of a segment in registers.
    int tab_slot[kFirIter], tab_r4[kFirIter];
    int tab_k0 = -1;
    auto build_table = [&](int k0) {
#pragma unroll
        for (int u = 0; u < kFirIter; u++) {
            const unsigned pos = (unsigned) (k0 + u * 32 + lane) * dx;
            const unsigned sidx = pos >> 12;
            // shared address of the sample's Y slot (clamped for pixels past outw)
            tab_slot[u] = (int) smem_u32(yrow + 1 + min(sidx + (sidx >> 3), (unsigned) (FirRow<FAST>::kSlots - 3)));
            tab_r4[u] = (int) ((pos & 0xfffu) << 2);
        }
    };
    if (bulk) {
        build_table(0);
        tab_k0 = 0;
    }

    if (lane == 0 && is_active(cur)) {
        request_signal(cur, 0);
        if (prefetch_old) request_old(cur, 0, 0, seg0);
    }

#pragma unroll 1
    for (int it = 0; kline < kLines; it++, kline += stride) {
        const int buf = it & 1;
        // line n + 1's signal window and line n + 2's record
        const bool nxt_active = is_active(nxt); // (fetched a whole line ago)
        if (lane == 0 && nxt_active) request_signal(nxt, buf ^ 1);
        const FirLine nn = fetch(kline + 2 * stride);

        if (is_active(cur)) {
            unsigned char *sigbuf = stage + buf * kFirStage;
            const int a = cur.pos & 15;
            const int nrows = max(1, cur.end - scanlines - cur.beg); // crt_core.c:662-664
            unsigned char *row0 = out + (size_t) cur.beg * pitch;
            mbar_wait(&bars[buf], (ph_sig >> buf) & 1);
            ph_sig ^= 1u << buf;
            const int nw0 = wsub(0, cur.wave0), nw1 = wsub(0, cur.wave1);
            // wave[(i + 0) & 3] feeds I, wave[(i + 3) & 3] feeds Q (crt_core.c:538-543)
            const int wi[4] = { cur.wave0, cur.wave1, nw0, nw1 };
            const int wq[4] = { nw1, cur.wave0, cur.wave1, nw0 };

            // ---- (F) samples [24 * lane - halo, 24 * lane + 24); the first ones only rebuild the history
            const int e0 = lane * kFirChunk;
            if (e0 - kFirHalo < kAvLen) {
                const signed char *sg = reinterpret_cast<const signed char *>(sigbuf) + a + e0;
                const bool head = (lane == 0); // samples before the line start are zeros, not signal (crt_core.c:534-536)
                FirChan fy, fi, fq;
                fir_reset(fy);
                fir_reset(fi);
                fir_reset(fq);
#pragma unroll
                for (int j = 0; j < kFirHalo; j++) {
                    const int i4 = (j - kFirHalo) & 3; // (e0 - halo + j) & 3, e0 a multiple of 4
                    const int s = head ? 0 : (int) sg[head ? 0 : j - kFirHalo];
                    (void) fir_push(fy, head ? 0 : wadd(s, bright));
                    (void) fir_push(fi, wmul(s, wi[i4]) >> 9);
                    (void) fir_push(fq, wmul(s, wq[i4]) >> 9);
                }
                Elem *dst = yrow + 1 + lane * (kFirChunk + kFirChunk / 8);
#pragma unroll
                for (int t = 0; t < kFirChunk; t++) {
                    const int s = sg[t];
                    // FAST keeps Y not yet scaled by 16 (see crt_lines.cuh: the pixel pass folds the scale into its
                    // weights); the generic path keeps Y * 16 verbatim.
                    const int y5 = fir_push(fy, wadd(s, bright)) >> kFirShift;
                    const Elem y = (Elem) (FAST ? y5 : wmul(y5, 16));
                    const Elem ci = (Elem) (fir_push(fi, wmul(s, wi[t & 3]) >> 9) >> (kFirShift + 3)); // (v >> shift) >> 3
                    const Elem cq = (Elem) (fir_push(fq, wmul(s, wq[t & 3]) >> 9) >> (kFirShift + 3));
                    const int slot = t + (t >> 3);
                    dst[slot] = y;
                    dst[slot + kComp] = ci;
                    dst[slot + 2 * kComp] = cq;
                    if ((t & 7) == 0) {
                        dst[slot - 1] = y;
                        dst[slot - 1 + kComp] = ci;
                        dst[slot - 1 + 2 * kComp] = cq;
                    }
                }
            }
            __syncwarp();

            // The stores of the previous line have had the whole filter pass to read their row buffer: it can
            // now receive the previous image's row of the NEXT line, which in turn has the pixel pass to arrive.
            if (bulk && lane == 0) {
                tma_store_wait_read<0>();
                if (prefetch_old && nxt_active) request_old(nxt, buf ^ 1, 0, seg0);
            }
            __syncwarp(); // no lane writes this line's row buffer before the stores that last read it are known done

            // ---- (P) pixels (crt_core.c:555-659), 32 consecutive ones per step
            const Elem *slot1 = yrow + 1; // slot of sample 0
            // 0x00RRGGBB from the two samples at `sp` and the 4x interpolation weight of the second one; when blending
            // (MODE 1) every channel comes back already halved (yiq_to_rgb<true>), which is what crt_core.c:608 adds
            auto shade = [&](unsigned sp, int R4) -> unsigned { // sp: shared address of the first sample's Y
                constexpr int E = (int) sizeof(Elem), C = FirRow<FAST>::kCompBytes;
                const int ay = lds_elem<Elem, 0>(sp), by = lds_elem<Elem, E>(sp);
                const int ai = lds_elem<Elem, C>(sp), bi = lds_elem<Elem, C + E>(sp);
                const int aq = lds_elem<Elem, 2 * C>(sp), bq = lds_elem<Elem, 2 * C + E>(sp);
                if (FAST) {
                    const int L4 = 0x3ffc - R4; // 4 * L
                    const int y = wadd(wmul(ay, L4), wmul(by, R4));
                    // (v * 4L) >> 16 == (v * L) >> 14: the two dropped bits are zeros.  (Multiply + shift rather than one
                    // IMAD.HI per term: IMAD.HI is a multi-pass instruction.)
                    return yiq_to_rgb<MODE == 1>(y, wadd(wmul(ai, L4) >> 16, wmul(bi, R4) >> 16),
                                                 wadd(wmul(aq, L4) >> 16, wmul(bq, R4) >> 16), contrast);
                } else {
                    const int R = R4 >> 2, L = 0xfff - R;
                    return yiq_pixel<MODE == 1>(ay, ai, aq, by, bi, bq, R, L, contrast);
                }
            };
            auto pixel = [&](int px) -> unsigned { // 0x00RRGGBB of output pixel px
                const unsigned pos = (unsigned) px * dx;
                const unsigned s = pos >> 12;
                return shade(smem_u32(slot1 + (s + (s >> 3))), (int) ((pos & 0xfffu) << 2));
            };

            if (bulk) {
                unsigned *ob = orow + buf * kFirSeg;
#pragma unroll 1
                for (int k0 = 0; k0 < geo.outw; k0 += kFirSeg) {
                    const int cnt = min(kFirSeg, geo.outw - k0);
                    if (k0 > 0) { // wide images: later segments reuse the buffer in place
                        __syncwarp();
                        if (lane == 0) {
                            tma_store_wait_read<0>();
                            if (MODE == 1) request_old(cur, buf, k0, cnt);
                        }
                        __syncwarp();
                    }
                    if (k0 != tab_k0) { // (only images wider than one segment ever rebuild the table)
                        build_table(k0);
                        tab_k0 = k0;
                    }
                    if (MODE == 1) {
                        mbar_wait(&bars[2 + buf], (ph_old >> buf) & 1);
                        ph_old ^= 1u << buf;
                    }
                    const int steps = (cnt + 31) >> 5; // lanes (and one whole step) past cnt compute into the unused tail
                    auto emit = [&](int u) {
                        const int j = u * 32 + lane;
                        const unsigned rgb = shade((unsigned) tab_slot[u], tab_r4[u]);
                        unsigned v = (FMT == CRT_PIX_FORMAT_BGRA) ? rgb : __byte_perm(rgb, 0u, sel_store);
                        if (MODE == 1) // crt_core.c:608 on whole words; the alpha byte is masked out and set
                            v = alpha_ff + v + ((ob[j] & blend_even) >> 1);
                        else
                            v |= alpha_ff;
                        ob[j] = v;
                    };
#pragma unroll
                    for (int u = 0; u + 1 < kFirIter; u += 2) {
                        if (u < steps) {
                            emit(u);
                            emit(u + 1);
                        }
                    }
                    if ((kFirIter & 1) && kFirIter - 1 < steps) emit(kFirIter - 1);
                    fence_async_smem();
                    __syncwarp();
                    if (lane == 0) {
                        unsigned char *d = row0 + (size_t) k0 * 4;
                        for (int r = 0; r < nrows; r++) tma_store_1d(d + (size_t) r * pitch, ob, cnt * 4);
                        tma_store_commit();
                    }
                }
            } else {
#pragma unroll 1
                for (int px = lane; px < geo.outw; px += 32) {
                    unsigned rgb = pixel(px);
                    if (MODE != 2) {
                        unsigned char *p = row0 + (size_t) px * 4;
                        unsigned v = (FMT == CRT_PIX_FORMAT_BGRA) ? (rgb | alpha_ff) : __byte_perm(rgb, 0xffu, sel_store);
                        if (MODE == 1) // (rgb is already halved, v carries the alpha byte)
                            v += (__ldcg(reinterpret_cast<const unsigned *>(p)) >> 1) & blend_mask;
                        for (int r = 0; r < nrows; r++) __stcg(reinterpret_cast<unsigned *>(p + (size_t) r * pitch), v);
                    } else {
                        unsigned char *p = row0 + (size_t) px * 3;
                        if (geo.blend) {
                            const unsigned o = (unsigned) p[rp] << 16 | (unsigned) p[gp] << 8 | (unsigned) p[bp];
                            rgb = ((rgb >> 1) & 0x7f7f7fu) + ((o >> 1) & 0x7f7f7fu);
                        }
                        for (int r = 0; r < nrows; r++) {
                            unsigned char *d = p + (size_t) r * pitch;
                            d[rp] = (unsigned char) (rgb >> 16);
                            d[gp] = (unsigned char) (rgb >> 8);
                            d[bp] = (unsigned char) rgb;
                        }
                    }
                }
            }
            __syncwarp(); // every lane is done with the Y/I/Q rows before the next line's filter pass rewrites them
        } else if (prefetch_old && lane == 0 && nxt_active) {
            // nothing was requested during this (skipped) line: the other row buffer's last reader is the
            // line before it
            tma_store_wait_read<0>();
            request_old(nxt, buf ^ 1, 0, seg0);
        }
        cur = nxt;
        nxt = nn;
    }
    if (lane == 0) tma_store_wait_read<0>(); // shared memory must outlive the stores that read it
}

} // namespace crt
