// crt_bloom.cuh -- the decoder of the reference's CRT_DO_BLOOM 1 build (crt_core.h:70; crt_core.c:399-402,
// 512-531): every decoded line gets its own width from a filtered "beam energy",
//     prev_e = prev_e * 123 / 128 + (((max_e >> 1) - sum(line)) << 10) / max_e       (serial from line to line)
//     line_w = AV_LEN * 112 / 128 + (prev_e >> 9),  dx = (line_w << 12) / outw,  scanL = ((AV_LEN / 2) - (line_w >> 1) + 8) << 12
// so the resampling step, the first filtered sample and the number of pixels a line writes differ from line to
// line, and a row may keep part of its previous content.  That does not fit the launch-uniform pixel loop of
// k_lines; this option (off in the reference's stock build) gets its own, functional-not-tuned kernels:
//   k_bloom        CTA per monitor: line sums in parallel (warp per line), the 240-step energy chain on one thread
//   k_lines_bloom  warp per line: lanes 0..2 run the Y / I / Q equalisers (same code, per-lane coefficients),
//                  then all lanes resample, convert and store pixels, and replicate duplicated rows whole
//                  (crt_core.c:662-664 copies the complete row, including what this line did not write).
#pragma once

#include "crt_lines.cuh"

namespace crt {

// The option is supported for the systems whose encoder has the option's branch (crt_ntsc.c:148-160 and the same
// lines of crt_ntscvhs.c, crt_template.c, crt_pv1k.c, crt_snes.c; crt_sys.cuh: kDestW, kDestH).  The NES and NES-RGB
// encoders have none (the reference notes "does not work for NES", crt_core.h:70).
static_assert(!kBloom || CRT_B200_BANDLIMITED || (CRT_SYSTEM == CRT_SYSTEM_SNES),
              "CRT_DO_BLOOM=1: supported for CRT_SYSTEM 0 (NTSC), 2 (PV1K), 3 (SNES), 4 (TEMP) and 5 (NTSCVHS) only");

struct BloomLine { // per decoded line, written by k_bloom
    int dx, scan_l;
};

__global__ void __launch_bounds__(256) k_bloom(const MonCfg *__restrict__ cfgs, const LineRec *__restrict__ lines_base,
                                               const signed char *__restrict__ inp_base, BloomLine *__restrict__ bloom_base,
                                               int first)
{
    __shared__ int energy[kLines];
    const int m = first + blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const MonCfg cfg = cfgs[m];
    if (cfg.bpp == 0 || cfg.outw <= 0) return;
    const LineRec *recs = lines_base + (size_t) m * kLines;
    const signed char *inp = inp_base + (size_t) m * kSignalBytes;
    BloomLine *bloom = bloom_base + (size_t) m * kLines;
    for (int k = warp; k < kLines; k += 8) { // crt_core.c:513-516
        const int beg = recs[k].beg, pos = recs[k].pos;
        int s = 0;
        if (beg >= 0)
            for (int i = lane; i < kAvLen; i += 32) s += inp[pos + i];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
        if (lane == 0) energy[k] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int max_e = (128 + (cfg.noise / 2)) * kAvLen; // crt_core.c:400-401
        int prev_e = 16384 / 8;
        for (int k = 0; k < kLines; k++) {
            BloomLine b;
            b.dx = 0;
            b.scan_l = 0;
            if (recs[k].beg >= 0 && max_e != 0) { // skipped lines leave the chain alone (crt_core.c:431)
                prev_e = (prev_e * 123 / 128) + ((((max_e >> 1) - energy[k]) << 10) / max_e); // crt_core.c:518
                const int line_w = (kAvLen * 112 / 128) + (prev_e >> 9);
                b.dx = (line_w << 12) / cfg.outw;
                b.scan_l = ((kAvLen / 2) - (line_w >> 1) + 8) << 12;
            }
            bloom[k] = b;
        }
    }
}

constexpr int kBloomWarps = 8;
constexpr int kBloomRow = kAvLen + 1;                       // ints per component and line
constexpr int kBloomSmem = kBloomWarps * 3 * kBloomRow * 4; // Y, I, Q rows of the lines in flight
constexpr int kBloomGroups = (kLines + kBloomWarps - 1) / kBloomWarps;

__global__ void __launch_bounds__(kBloomWarps * 32) k_lines_bloom(const MonCfg *__restrict__ cfgs,
                                                                 const LineRec *__restrict__ lines_base,
                                                                 const signed char *__restrict__ inp_base,
                                                                 const BloomLine *__restrict__ bloom_base, int first,
                                                                 const LinesGeom geo)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = first + blockIdx.y;
    const int k = blockIdx.x * kBloomWarps + warp; // decoded line of this warp
    if (k >= kLines || geo.bpp == 0 || geo.outw <= 0) return;
    const LineRec rec = lines_base[(size_t) m * kLines + k];
    if (!line_in_launch(k, rec, geo)) return; // (warp-uniform)
    const MonCfg cfg = cfgs[m];
    const BloomLine bl = bloom_base[(size_t) m * kLines + k];
    int *comp = reinterpret_cast<int *>(smem_raw) + warp * 3 * kBloomRow;
    int *yy = comp, *ii = comp + kBloomRow, *qq = comp + 2 * kBloomRow;
    const signed char *sig = inp_base + (size_t) m * kSignalBytes + rec.pos;
    const unsigned scan_l = (unsigned) bl.scan_l, scan_r = (unsigned) ((kAvLen - 1) << 12);
    const int f_lo = (int) (scan_l >> 12), f_hi = (int) (scan_r >> 12); // crt_core.c:524-525: sample AV_LEN - 1 is NOT filtered

    // ---- equalisers (crt_core.c:534-543, literal wrap-exact form): lane 0 = Y, 1 = I, 2 = Q
    if (lane < 3 && f_lo >= 0) {
        const int lf = lane == 0 ? kEqYlf : lane == 1 ? kEqIlf : kEqQlf;
        const int hf = lane == 0 ? kEqYhf : lane == 1 ? kEqIhf : kEqQhf;
        const int g1 = lane == 0 ? kEqYg1 : 65536;
        const int g2 = lane == 0 ? kEqYg2 : lane == 1 ? kEqIg2 : 0;
        const int bright = cfg.brightness - (kBlack + cfg.black_point);
        const int off = lane == 2 ? 3 : 0; // wave[(i + 0) & 3] feeds I, wave[(i + 3) & 3] feeds Q
        int w5[5] = { 0, 0, 0, 0, 0 };      // five carrier phases (PV-1000): this lane's table, waveI or waveQ
        if (kCc == 5) {
            int wi5[5], wq5[5];
            pv1k_waves(rec.wave0, rec.wave1, cfg.hue, cfg.saturation, wi5, wq5);
#pragma unroll
            for (int q = 0; q < 5; q++) w5[q] = (lane == 2) ? wq5[q] : wi5[q];
        }
        int l0 = 0, l1 = 0, l2 = 0, l3 = 0, h0 = 0, h1 = 0, h2 = 0, h3 = 0, s1 = 0, s2 = 0, s3 = 0;
        int *dst = comp + lane * kBloomRow;
        for (int i = f_lo; i < f_hi; i++) {
            const int s = sig[i];
            int in;
            if (lane == 0) {
                in = s + bright;
            } else if (kCc == 5) { // waveI[i % 5] / waveQ[i % 5] (crt_core.c:545-549)
                const int ph = i % 5;
                const int w = ph == 0 ? w5[0] : ph == 1 ? w5[1] : ph == 2 ? w5[2] : ph == 3 ? w5[3] : w5[4];
                in = wmul(s, w) >> 9;
            } else {
                const int ph = (i + off) & 3;
                const int w = (ph & 1) ? rec.wave1 : rec.wave0;
                in = wmul(s, (ph & 2) ? wsub(0, w) : w) >> 9;
            }
            l0 = wadd(l0, wadd(wmul(wsub(in, l0), lf), 32768) >> 16); // crt_core.c:211-217
            l1 = wadd(l1, wadd(wmul(wsub(l0, l1), lf), 32768) >> 16);
            l2 = wadd(l2, wadd(wmul(wsub(l1, l2), lf), 32768) >> 16);
            l3 = wadd(l3, wadd(wmul(wsub(l2, l3), lf), 32768) >> 16);
            h0 = wadd(h0, wadd(wmul(wsub(in, h0), hf), 32768) >> 16);
            h1 = wadd(h1, wadd(wmul(wsub(h0, h1), hf), 32768) >> 16);
            h2 = wadd(h2, wadd(wmul(wsub(h1, h2), hf), 32768) >> 16);
            h3 = wadd(h3, wadd(wmul(wsub(h2, h3), hf), 32768) >> 16);
            const int r0 = wmul(l3, 65536) >> 16; // crt_core.c:219-232
            const int r1 = wmul(wsub(h3, l3), g1) >> 16;
            const int r2 = wmul(wsub(s3, h3), g2) >> 16;
            s3 = s2;
            s2 = s1;
            s1 = in;
            const int r = wadd(wadd(r0, r1), r2);
            dst[i] = lane == 0 ? wmul(r, 16) : (r >> 3);
        }
        // never filtered with bloom on, and the reference's static scratch array holds its initial zero there
        dst[kAvLen - 1] = 0;
    }
    __syncwarp();

    // ---- pixels (crt_core.c:551-664)
    const int bpp = geo.bpp, pitch = geo.pitch;
    int rp, gp, bp;
    fmt_positions(geo.out_format, rp, gp, bp);
    const int ap = (bpp == 4) ? (6 - rp - gp - bp) : -1; // the remaining byte of a 4-byte pixel
    unsigned char *row = cfg.out + (size_t) rec.beg * pitch;
    const int nrows = rows_written(rec, cfg.scanlines);
    for (int j = lane; j < geo.outw; j += 32) {
        const unsigned pos = scan_l + (unsigned) j * (unsigned) bl.dx;
        const bool wr = f_lo >= 0 && pos < scan_r; // the written pixels are a prefix of the row (crt_core.c:555)
        unsigned char *p = row + (size_t) j * bpp;
        unsigned char px[4];
        px[0] = p[0]; px[1] = p[1]; px[2] = p[2]; px[3] = (bpp == 4) ? p[3] : 0;
        if (wr) {
            const int s = (int) (pos >> 12), R = (int) (pos & 0xfffu), L = 0xfff - R;
            unsigned rgb = yiq_pixel(yy[s], ii[s], qq[s], yy[s + 1], ii[s + 1], qq[s + 1], R, L, cfg.contrast);
            if (geo.blend) { // crt_core.c:584-609
                const unsigned old = (unsigned) px[rp] << 16 | (unsigned) px[gp] << 8 | (unsigned) px[bp];
                rgb = ((rgb & 0xfefeffu) >> 1) + ((old & 0xfefeffu) >> 1);
            }
            px[rp] = (unsigned char) (rgb >> 16);
            px[gp] = (unsigned char) (rgb >> 8);
            px[bp] = (unsigned char) rgb;
            if (ap >= 0) px[ap] = 0xff;
        }
        for (int r = wr ? 0 : 1; r < nrows; r++) { // row `beg` itself only where the line wrote
            unsigned char *d = p + (size_t) r * pitch;
            d[0] = px[0]; d[1] = px[1]; d[2] = px[2];
            if (bpp == 4) d[3] = px[3];
        }
    }
}

} // namespace crt
