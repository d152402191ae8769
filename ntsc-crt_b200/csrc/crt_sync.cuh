// crt_sync.cuh -- k_sync, the sync pre-pass of crt_demodulate (crt_core.c:379-479).
//
// What is serial in the reference and stays serial here (the values are exact integers with
// truncation at every step, so there is no closed form):
//   * the hsync chain: line k searches a 2W-sample window positioned by line k-1's result;
//   * the colour-burst lock: ccr[p] = ccr[p] * 127 / 128 + sample, 10 steps per phase per line, carried
//     from line to line (and, with CRT_CC_VPER = 3, along three interleaved rows).
// What this kernel does about it: one CTA of 4 warps per monitor;
//   1. all warps copy the head of every signal line (the only bytes either chain can touch while
//      sync holds) into shared memory with coalesced loads -- the chains then run at shared-memory
//      latency instead of L2 latency;
//   2. the 2W vsync candidates are integrated in parallel, 4 lines at a time, one per warp;
//   3. the hsync chain is solved by verified speculation (parallel sweeps to a fixed point, see 3a);
//      one warp then runs the burst-lock chain, 4 lanes per colour row, next line prefetched;
//   4. all threads emit the per-line records k_lines consumes.
// Lines whose windows leave the staged heads (sync lost, |hsync| large) fall back to global loads.
#pragma once

#include "crt_kernels.cuh"

namespace crt {

constexpr int kHeadBefore = 16;                 // staged bytes before each line start
constexpr int kHeadAfter = ((kCbBeg + kBurstLen + 40 + 15) / 16) * 16; // ... and after it
constexpr int kHeadWords = (kHeadBefore + kHeadAfter) / 4 + 1;        // +1: start is aligned down to 4
constexpr int kCandWords = (kHres + 3) / 4 + 1;                     // a whole line from a 4-aligned start
// One head more than there are signal lines: with hsync in the second half of a line (the steady state of the
// NTSC timing, ~898) the search window of the LAST signal line sits on the start of the line after it.  Those
// bytes are the padding after inp[] (the reference reads past its array there); staging them keeps that one
// line off the 16-dependent-loads fall-back, which would hold every sweep's barrier.
constexpr int kHeadLines = kVres + 1;
constexpr int kSyncSmem = (kHeadLines * kHeadWords + 2 * kVsyncWindow * kCandWords) * 4;
constexpr int kSyncThreads = 256;

// CRT_CC_SAMPLES == 5 (crt_core.c:497-508): carrier tables rotated by the hue knob, one I and one Q value per phase
__device__ __forceinline__ void pv1k_waves(int dci, int dcq, int hue, int saturation, int (&wi)[5], int (&wq)[5])
{
    int ang = hue % 360;
#pragma unroll
    for (int i = 0; i < 5; i++) {
        int sn, cs;
        sincos14_d(sn, cs, ang * 8192 / 180);
        wi[i] = wmul(wadd(wmul(dci, cs), wmul(dcq, sn)) >> 15, saturation);
        sincos14_d(sn, cs, (ang + 90) * 8192 / 180);
        wq[i] = wmul(wadd(wmul(dci, cs), wmul(dcq, sn)) >> 15, saturation);
        ang += 360 / 5;
    }
}

// The rows the decoded lines spread over, as the reference computes them (crt_core.c:428-429): outh + v_fac in 32-bit
// unsigned arithmetic (v_fac is unsigned), so a "negative" v_fac shrinks the span and may wrap it to anything.
__host__ __device__ inline unsigned row_span(const MonCfg &c) { return (unsigned) c.outh + c.v_fac; }
// Up to this span (k + 1) * span does not wrap for any line: beg and end never decrease from one line to the next.
// Above it lines far apart can share rows, and the line passes take them one level at a time (k_sync, crtx.cu).
constexpr unsigned kMonotonicSpan = 0xffffffffu / (unsigned) kLines;
// The rows a decoded line writes, from `beg` on (crt_core.c:662-664): `l` is anything with the line's beg and end.
template <class Line> __device__ __forceinline__ int rows_written(const Line &l, int scanlines) { return max(1, l.end - scanlines - l.beg); }

struct SyncLine { // what depends only on k, vsync and the detected field (not on the chains)
    short jl;   // signal line the decoded line reads: posmod(top + k + vsync, vres)
    short row;  // colour row: ypos % CC_VPER
    int ypos;   // posmod(top + k + vsync + 3, vres)
    int beg, end; // output rows, beg = -1 when the line is skipped (crt_core.c:428-432)
};

struct SyncShared {
    SyncLine ln[kLines];
    int hs[kLines];     // hsync after each decoded line's search
    int ccr[kLines][kCc]; // burst-lock accumulator of the line's colour row after its 10 steps
    uint4 burst[kLines][kCc]; // the burst samples each decoded line locks onto, by carrier phase: bytes 0 .. 9 of [line][phase]
    union {
        short rowlist[kVper > 3 ? kVper : 3][kLines]; // decoded lines of each colour row, in order (step 3b)
        short level[kLines]; // spans above kMonotonicSpan: the line pass each line runs in (filled after step 3b)
    };
    int rowcount[kVper > 3 ? kVper : 3];
    int vs_found[2 * kVsyncWindow]; // per vsync candidate: crossing index or -1
    int generic;
    int noise_next; // next chunk of the noise pass to hand out (kFusedNoise)
    int need_max;   // some line of this pass needed its signal lines' largest sample
    int need_inp;   // some line's window runs past inp[] into the struct tail, which must be read unclamped: inp[] after all
    int linemax[kVres + 2]; // largest |sample| of each signal line of inp[], measured by the noise pass when MonState::track_max says so
};

// hsync search of one decoded line given the hsync it enters with (crt_core.c:437-447):
// integrate 2W samples starting W before the expected sync edge, stop at the threshold.
template <typename FetchByte>
__device__ __forceinline__ int hsync_step(const unsigned *heads, FetchByte fetch_byte, int jl, int hs)
{
    const int p0 = jl * kHres + hs + kSyncBeg - kHsyncWindow; // first window sample
    const int j = (hs > kHres / 2) ? jl + 1 : jl;             // line whose staged head holds the window
    const int off = p0 - ((j * kHres - kHeadBefore) & ~3);
    int i = 2 * kHsyncWindow, acc = 0;
    if (j < kHeadLines && off >= 0 && off + 2 * kHsyncWindow <= kHeadWords * 4) {
        const signed char *hb = reinterpret_cast<const signed char *>(heads + j * kHeadWords) + off;
#pragma unroll
        for (int t = 0; t < 2 * kHsyncWindow; t++) {
            acc += hb[t];
            if (acc <= kHsyncLevel && i == 2 * kHsyncWindow) i = t;
        }
    } else { // window outside the staged heads (sync lost): plain loads
        for (int t = 0; t < 2 * kHsyncWindow; t++) {
            acc += fetch_byte(p0 + t);
            if (acc <= kHsyncLevel && i == 2 * kHsyncWindow) i = t;
        }
    }
    hs += i - kHsyncWindow;
    if (hs < 0) hs += kHres; // POSMOD(i + hsync, HRES), |i| <= W
    else if (hs >= kHres) hs -= kHres;
    return hs;
}

// In the reference inp[] is followed, inside struct CRT, by outw, outh, out_format and four bytes of padding
// (crt_core.h:74-92; crt_init zeroes the struct).  A sync search or decode window that runs a few samples past the
// end of inp[] -- the PV-1000 does that in ordinary operation: its picture ends one sample before the end of the
// line and hsync settles above 4 -- reads those bytes.  They are deterministic, so they are reproduced: 16 bytes
// behind each signal buffer (the kernels stage from analog[] when the noise pass is fused, from inp[] otherwise).
// What follows them in the reference is the `out` pointer; windows that reach it are outside the parity domain.
__global__ void __launch_bounds__(64) k_struct_tail(const MonCfg *__restrict__ cfgs, signed char *__restrict__ analog_base,
                                                    signed char *__restrict__ inp_base, int first, int count)
{
    const int i = blockIdx.x * 64 + threadIdx.x;
    if (i >= count) return;
    const MonCfg c = cfgs[first + i];
    const int v[4] = { c.outw, c.outh, c.out_format, 0 };
    signed char *a = analog_base + (size_t) (first + i) * kSignalBytes + kInputSize;
    signed char *b = inp_base + (size_t) (first + i) * kSignalBytes + kInputSize;
    for (int k = 0; k < 16; k++) { // (byte stores: CRT_INPUT_SIZE is not a multiple of 4 in every system)
        const signed char byte = (signed char) ((unsigned) v[k >> 2] >> (8 * (k & 3)));
        a[k] = byte;
        b[k] = byte;
    }
}

// max(b, -127) on four packed samples (the clamp of crt_core.c:363-364 when the noise term is zero: only -128 moves).
// A byte is 0x80 iff its top bit is set and its low seven bits are zero; (low7 + 0x7f) carries into the top bit iff they are not.
__device__ __forceinline__ unsigned clamp127_4(unsigned x)
{
    const unsigned nz = (x & 0x7f7f7f7fu) + 0x7f7f7f7fu;
    return x | ((x & ~nz & 0x80808080u) >> 7);
}
__device__ __forceinline__ uint4 clamp127_v(uint4 v)
{
    return make_uint4(clamp127_4(v.x), clamp127_4(v.y), clamp127_4(v.z), clamp127_4(v.w));
}

// The noise pass (crt_core.c:346-367) at noise != 0: sample i of inp[] is analog[i] plus the noise term of the LCG state
// advanced i + 1 steps from the call's seed rn0, clamped to +-127.  noise_state: the state before sample 16 t, from the
// jump tables; noise_word: four samples from the state before them, which it advances past them.
__device__ __forceinline__ unsigned noise_state(int t, unsigned rn0, const Affine *__restrict__ jump_lo, const Affine *__restrict__ jump_hi)
{
    const Affine lo = jump_lo[t % kJumpLo], hi = jump_hi[t / kJumpLo];
    return (rn0 * hi.mul + hi.add) * lo.mul + lo.add;
}
__device__ __forceinline__ unsigned noise_word(unsigned w, unsigned &rn, int noise)
{
    unsigned o = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
        rn = rn * kLcgMul + kLcgAdd;
        const int v = (int) (signed char) (w >> (8 * b)) + (wmul((int) ((rn >> 16) & 0xff) - 0x7f, noise) >> 8);
        o |= ((unsigned) clampi(v, -127, 127) & 0xffu) << (8 * b);
    }
    return o;
}

// Vector t of inp[] (samples 16 t .. 16 t + 15) from the same 16 bytes of analog[].  Its bytes past inp[] (the last vector
// runs over) are noised like the rest: its callers store and measure only the bytes inside.
__device__ __forceinline__ uint4 noisy_vec(uint4 v, int t, int noise, unsigned rn0, const Affine *__restrict__ jump_lo,
                                           const Affine *__restrict__ jump_hi)
{
    if (noise == 0) return clamp127_v(v);
    unsigned rn = noise_state(t, rn0, jump_lo, jump_hi);
    v.x = noise_word(v.x, rn, noise);
    v.y = noise_word(v.y, rn, noise);
    v.z = noise_word(v.z, rn, noise);
    v.w = noise_word(v.w, rn, noise);
    return v;
}

// The same rule for the four samples starting at the 4-aligned index p, from the word `w` of analog[] there, for what k_sync
// stages and reads.  Beyond inp[] lie the bytes k_struct_tail put there (what follows inp[] inside the reference's struct
// CRT), identical after analog[] and after inp[], and never touched by the noise pass: they are kept raw.  Kept apart from
// the load so that callers can issue a batch of loads before touching any.
__device__ __forceinline__ unsigned noisy_apply(unsigned w, int p, int noise, unsigned rn0,
                                                const Affine *__restrict__ jump_lo, const Affine *__restrict__ jump_hi)
{
    const unsigned raw = w;
    if (noise == 0) {
        w = clamp127_4(w);
    } else {
        unsigned rn = noise_state(p / kNoiseVec, rn0, jump_lo, jump_hi);
        for (int k = 0; k < (p % kNoiseVec); k++) rn = rn * kLcgMul + kLcgAdd;
        w = noise_word(w, rn, noise);
    }
    if (p + 4 > kInputSize) {
        const unsigned keep = (p >= kInputSize) ? 0u : (0xffffffffu >> (8 * (p + 4 - kInputSize))); // bytes still inside inp[]
        w = (w & keep) | (raw & ~keep);
    }
    return w;
}

__device__ __forceinline__ unsigned noisy_word(const signed char *__restrict__ analog, int p, int noise, unsigned rn0,
                                               const Affine *__restrict__ jump_lo, const Affine *__restrict__ jump_hi)
{
    return noisy_apply(__ldg(reinterpret_cast<const unsigned *>(analog + p)), p, noise, rn0, jump_lo, jump_hi);
}

// |b| of four packed samples in -127 .. 127, and the larger of two such words byte by byte (values <= 127: bit 7 is free to
// catch the borrow of a per-byte subtraction)
__device__ __forceinline__ unsigned abs127_4(unsigned x)
{
    const unsigned neg = (x >> 7) & 0x01010101u;
    return (x ^ (neg * 0xffu)) + neg; // ~b + 1 where b < 0: at most 127, no carry leaves the byte
}
__device__ __forceinline__ unsigned max127_4(unsigned a, unsigned b)
{
    const unsigned ge = (((a | 0x80808080u) - b) >> 7) & 0x01010101u; // 1 where a >= b
    const unsigned sel = ge * 0xffu;
    return (a & sel) | (b & ~sel);
}

// Writes vector t of inp[] (noisy_vec's result): in the last vector only the bytes inside inp[] (behind it lie the bytes of
// k_struct_tail, the same in both buffers)
__device__ __forceinline__ void store_inp_vec(signed char *inp, int t, uint4 v)
{
    signed char *d = inp + t * kNoiseVec;
    if ((t + 1) * kNoiseVec <= kInputSize) {
        *reinterpret_cast<uint4 *>(d) = v;
    } else {
#pragma unroll
        for (int b = 0; b < kNoiseVec; b++) {
            const unsigned w = (b < 4) ? v.x : (b < 8) ? v.y : (b < 12) ? v.z : v.w;
            if (t * kNoiseVec + b < kInputSize) d[b] = (signed char) (w >> (8 * (b & 3)));
        }
    }
}

// inp[] of the monitors whose last k_sync left it unwritten (MonState::inp_late), one CTA per monitor: what the host runs
// before it hands inp[] out or lets analog[] change (crtx.cu: inp_from_analog)
__global__ void __launch_bounds__(256) k_inp_from_analog(const MonState *__restrict__ states, const signed char *__restrict__ analog_base,
                                                         signed char *__restrict__ inp_base, int first)
{
    const int m = first + blockIdx.x;
    if (!states[m].inp_late) return;
    const signed char *analog = analog_base + (size_t) m * kSignalBytes;
    signed char *inp = inp_base + (size_t) m * kSignalBytes;
    for (int t = threadIdx.x; t < kNoiseThreads; t += 256) store_inp_vec(inp, t, clamp127_v(__ldg(reinterpret_cast<const uint4 *>(analog) + t)));
}

// The LCG systems' noise pass is fused into this kernel (kFusedNoise): it reads analog[], applies the noise itself to what it
// stages, and writes the whole inp[].  That copy is pure memory traffic and the burst-lock chain pure latency on one
// warp, so they overlap: while the last warp runs the chain the other seven copy, 4 KB chunks handed out by a counter in shared
// memory (the chain warp joins when it is through).  The overlap is not free: on the H100 the chain takes about 40 us beside
// the copy and about 24 us without it (DESIGN.md, k_sync), so at noise 0 it is left out where it can be (inp_late).
// VHS, whose noise comes from rand(): inp[] was written by k_noise_vhs, and this kernel reads it.
constexpr bool kFusedNoise = !kIsVhs;
constexpr int kNoiseNB = 8;                                   // 16-byte loads in flight per thread
constexpr int kNoiseChunkVecs = 32 * kNoiseNB;                // vectors per chunk (one warp, kNoiseNB rounds)
constexpr int kNoiseChunks = (kNoiseThreads + kNoiseChunkVecs - 1) / kNoiseChunkVecs;
constexpr int kChainWarp = kSyncThreads / 32 - 1;             // the arbiter favours the highest warp id: the serial chain gets it
constexpr int kBurstSteps = kBurstLen / kCc;                  // burst samples per carrier phase and line (10)
static_assert(kBurstSteps <= 16 && kBurstLen % kCc == 0, "one 16-byte record per (line, phase)");
// staging (phase 1) moves 16-byte vectors: a head row is covered by kHeadVecs of them from the 16-byte aligned address at or
// below its first word, a vsync candidate line by kCandVecs
constexpr int kHeadVecs = (12 + 4 * kHeadWords + 15) / 16;
constexpr int kCandVecs = (12 + 4 * kCandWords + 15) / 16;
constexpr int kStageVecs = kHeadLines * kHeadVecs + 2 * kVsyncWindow * kCandVecs;
constexpr int kStageBatch = (kStageVecs + kSyncThreads - 1) / kSyncThreads; // vector loads per thread, all in flight at once

__global__ void __launch_bounds__(kSyncThreads, 2) k_sync(const MonCfg *__restrict__ cfgs, MonState *__restrict__ states,
                                                          LineRec *__restrict__ lines_base,
                                                          const signed char *__restrict__ analog_base,
                                                          signed char *__restrict__ inp_base,
                                                          const Affine *__restrict__ jump_lo,
                                                          const Affine *__restrict__ jump_hi, int first,
                                                          int force_generic)
{
    phase_mark(0, 0);
    extern __shared__ __align__(16) unsigned heads[]; // [kHeadLines][kHeadWords]
    __shared__ SyncShared sh;
    const int m = first + blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const MonCfg cfg = cfgs[m];
    if (cfg.bpp == 0) return; // crt_core.c:312-315
    MonState *st = &states[m];
    const signed char *analog = analog_base + (size_t) m * kSignalBytes;
    signed char *inp_w = inp_base + (size_t) m * kSignalBytes;
    const signed char *inp = inp_w; // VHS reads; fall-back loads when sync is lost (see below)
    LineRec *lines = lines_base + (size_t) m * kLines;
    const unsigned rn0 = (unsigned) st->rn;
    const int noise = cfg.noise;
    auto fetch = [&](int p) { // one staged word
        if (p < 0) return 0u;
        if (kFusedNoise) return noisy_word(analog, p, noise, rn0, jump_lo, jump_hi);
        return __ldg(reinterpret_cast<const unsigned *>(inp + p));
    };
    auto fetch_byte = [&](int p) { // a single sample outside the staged regions (sync lost)
        const unsigned w = fetch(p & ~3);
        return (int) (signed char) (w >> (8 * (p & 3)));
    };
    const int track = kFusedNoise ? st->track_max : 0; // measure every signal line's largest sample during the copy (see step 4)
    // At noise 0 inp[] is max(analog[], -127).  For a monitor that k_lines2 decodes (MonCfg::lines2) the copy is not made:
    // k_lines2 reads its windows from analog[] with that clamp, and the host produces inp[] when a caller asks for it
    // (crtx.cu: inp_from_analog).  The copy would slow the burst-lock chain, which runs beside it on the same SM.  A monitor
    // that turns out to need the generic equaliser (k_lines, which reads inp[]), or a window that reads the struct tail
    // behind inp[] (bytes that may be -128 and are not clamped), gets it at the end after all.
    bool inp_late = kFusedNoise && cfg.lines2 && noise == 0 && !track;
    if (tid == 0) {
        sh.noise_next = 0;
        sh.need_max = 0;
        sh.need_inp = 0;
    }
    if (track)
        for (int l = tid; l < kVres + 2; l += kSyncThreads) sh.linemax[l] = 0;

    // ---- 1. stage line heads (heads[j][w] = the aligned word at ((j * H - 16) & ~3) + 4w) and the 2W
    // vsync candidate lines in full (cand[c][w] = aligned words covering line posmod(vsync + c - W)).  The signal is
    // read in 16-byte vectors, kStageBatch of them in flight per thread (word-sized loads in batches would spend most of
    // the time on index arithmetic), the noise applied, and the four words land at their places in the row.
    unsigned *cand = heads + kHeadLines * kHeadWords; // [2W][kCandWords]
    const int vs_in = st->vsync;
    // candidate c is line posmod(vsync + c - W, VRES) (crt->vsync is the caller's to poke: any value); one modulo per thread
    const int cand0 = posmod(vs_in - kVsyncWindow, kVres);
    auto cand_line = [&](int c) { return (cand0 + c >= kVres) ? cand0 + c - kVres : cand0 + c; };
    {
        const signed char *from = kFusedNoise ? analog : inp;
        // where staged vector idx comes from and which row words it feeds (computed twice -- for the load and again for the
        // stores -- rather than kept: with every load of the phase in flight at once the registers belong to the data)
        auto place = [&](int idx, int &pos, int &w0, int &nw) -> unsigned * {
            int start4, i;
            unsigned *row;
            if (idx < kHeadLines * kHeadVecs) {
                const int j = idx / kHeadVecs;
                i = idx - j * kHeadVecs;
                start4 = (j * kHres - kHeadBefore) & ~3;
                row = heads + j * kHeadWords;
                nw = kHeadWords;
            } else {
                const int q = idx - kHeadLines * kHeadVecs, c = q / kCandVecs;
                i = q - c * kCandVecs;
                start4 = (cand_line(c) * kHres) & ~3;
                row = cand + c * kCandWords;
                nw = (idx < kStageVecs) ? kCandWords : 0;
            }
            pos = (start4 & ~15) + 16 * i; // (arithmetic "& ~15": also right for the negative start of line 0)
            w0 = (pos - start4) >> 2;      // row word the vector's first word is (-3 .. nw)
            return row;
        };
        // CRT_DO_VSYNC 0: the candidates are searched in analog[], before any noise (crt_core.c:323-337); heads keep it
        auto raw_cand = [&](int idx) { return !kDoVsync && idx >= kHeadLines * kHeadVecs; };
        uint4 v[kStageBatch];
#pragma unroll
        for (int b = 0; b < kStageBatch; b++) {
            int pos, w0, nw;
            (void) place(b * kSyncThreads + tid, pos, w0, nw);
            v[b] = make_uint4(0u, 0u, 0u, 0u);
            const signed char *src = raw_cand(b * kSyncThreads + tid) ? analog : from;
            if (nw > 0 && pos >= 0) v[b] = __ldg(reinterpret_cast<const uint4 *>(src + pos));
        }
#pragma unroll
        for (int b = 0; b < kStageBatch; b++) {
            int pos, w0, nw;
            unsigned *row = place(b * kSyncThreads + tid, pos, w0, nw);
            if (nw == 0) continue;
            unsigned w[4] = { v[b].x, v[b].y, v[b].z, v[b].w };
            if (kFusedNoise && pos >= 0 && !raw_cand(b * kSyncThreads + tid)) {
                if (noise == 0 && pos + 16 <= kInputSize) {
                    const uint4 c = clamp127_v(v[b]);
                    w[0] = c.x;
                    w[1] = c.y;
                    w[2] = c.z;
                    w[3] = c.w;
                } else {
#pragma unroll 1
                    for (int e = 0; e < 4; e++) w[e] = noisy_apply(w[e], pos + 4 * e, noise, rn0, jump_lo, jump_hi);
                }
            }
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int wi = w0 + e;
                if (wi >= 0 && wi < nw) row[wi] = w[e];
            }
        }
    }
    // |bright| bound of the fast equaliser path (crt_lines.cuh); halved for the PV-1000, whose luma cascade
    // (hf = 80024) is only proven wrap-free up to there.  bright wraps as in the reference (crt_core.c:304), and its
    // magnitude is taken in 64 bits: abs(INT_MIN) is INT_MIN, which would pass the bound
    if (tid == 0) sh.generic = force_generic || llabs((long long) wsub(cfg.brightness, wadd(kBlack, cfg.black_point))) > (kCc == 5 ? 2048 : 4096);
    __syncthreads();
    phase_mark(0, 1);

    // ---- 2. vsync (crt_core.c:379-396): candidate c = line posmod(vsync + c - W); first crossing wins
    constexpr int kSeg = (kHres + 31) / 32;
    for (int c = warp; c < 2 * kVsyncWindow; c += kSyncThreads / 32) {
        const int lstart = cand_line(c) * kHres;
        const signed char *sig = reinterpret_cast<const signed char *>(cand + c * kCandWords) + (lstart & 3);
        const int b0 = lane * kSeg, b1 = min(kHres, b0 + kSeg);
        int sum = 0;
        for (int t = b0; t < b1; t++) sum += sig[t];
        int acc = warp_scan_incl(sum, lane) - sum, idx = -1;
        for (int t = b0; t < b1; t++) {
            acc += sig[t];
            if (idx < 0 && acc <= kVsyncLevel) idx = t;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, idx >= 0);
        const int j = hit ? __shfl_sync(0xffffffffu, idx, __ffs(hit) - 1) : -1;
        if (lane == 0) sh.vs_found[c] = j;
    }
    __syncthreads();
    phase_mark(0, 2);
    int vs = posmod(vs_in + kVsyncWindow - 1, kVres), jcross = kHres; // "gave up" defaults
    for (int c = 0; c < 2 * kVsyncWindow; c++) {
        if (sh.vs_found[c] >= 0) {
            vs = cand_line(c);
            jcross = sh.vs_found[c];
            break;
        }
    }
    if (!kDoVsync) vs = -3; // crt_core.c:341: the search only gave the field
    int field = (jcross > kHres / 2);
    const int ratio = (((cfg.outh << 16) / kLines) + 32768) >> 16; // crt_core.c:404-407
    field *= ratio / 2;
    const int hs_in = st->hsync;
    for (int k = tid; k < kLines; k += kSyncThreads) { // chain-independent per-line geometry
        SyncLine g;
        int beg = (int) ((unsigned) k * ((unsigned) cfg.outh + cfg.v_fac) / (unsigned) kLines + (unsigned) field);
        int end = (int) ((unsigned) (k + 1) * ((unsigned) cfg.outh + cfg.v_fac) / (unsigned) kLines + (unsigned) field);
        if (beg >= cfg.outh) beg = end = -1; // crt_core.c:431
        else if (end > cfg.outh) end = cfg.outh;
        g.jl = (short) posmod(kTop + k + vs, kVres);
        g.ypos = posmod(kTop + k + vs + 3, kVres);
        g.row = (short) (g.ypos % kVper);
        g.beg = beg;
        g.end = end;
        sh.ln[k] = g;
        sh.hs[k] = hs_in; // initial guess of the chain
    }
    __syncthreads();
    phase_mark(0, 3);
    // Decoded lines of each colour row, in order (skipped lines do not touch ccf).  Warp r compacts row r
    // with ballots, 32 lines per step -- a 240-iteration loop on one thread per row here would make every other
    // thread wait at the next barrier.
    if (warp < kVper) {
        int n = 0;
        for (int k0 = 0; k0 < kLines; k0 += 32) {
            const int k = k0 + lane;
            const bool mine = (k < kLines) && sh.ln[k].beg >= 0 && sh.ln[k].row == warp;
            const unsigned mm = __ballot_sync(0xffffffffu, mine);
            if (mine) sh.rowlist[warp][n + __popc(mm & ((1u << lane) - 1u))] = (short) k;
            n += __popc(mm);
        }
        if (lane == 0) sh.rowcount[warp] = n;
    }

    // ---- 3a. hsync chain hs[k] = f_k(hs[k-1]) (crt_core.c:437-450) by verified speculation: every line
    // is evaluated in parallel from the current guess of its predecessor; a sweep that changes nothing
    // proves hs[] is the chain's unique solution.  The sync edge recaptures the search from any start
    // within the window, so this takes a handful of sweeps instead of 240 dependent steps.
    // CRT_DO_HSYNC 0 (crt_core.c:446-450): the search's result is dropped and hsync is 0 after every decoded line.  A skipped
    // line keeps its predecessor's, so hs_in lasts until the first decoded line; warp 0 finds it with ballots, no sweeps.
    if (!kDoHsync) {
        if (warp == 0) {
            bool seen = false;
            for (int k0 = 0; k0 < kLines; k0 += 32) {
                const int k = k0 + lane;
                const unsigned dec = __ballot_sync(0xffffffffu, k < kLines && sh.ln[k].beg >= 0);
                if (k < kLines && (seen || (dec & (0xffffffffu >> (31 - lane))) != 0)) sh.hs[k] = 0;
                seen = seen || dec != 0;
            }
        }
        __syncthreads();
    }
    for (int sweep = 0; kDoHsync && sweep <= kLines; sweep++) {
        int nh[(kLines + kSyncThreads - 1) / kSyncThreads];
        int changed = 0;
#pragma unroll
        for (int q = 0; q < (kLines + kSyncThreads - 1) / kSyncThreads; q++) {
            const int k = tid + q * kSyncThreads;
            nh[q] = 0;
            if (k < kLines) {
                const int prev = (k == 0) ? hs_in : sh.hs[k - 1];
                nh[q] = (sh.ln[k].beg >= 0) ? hsync_step(heads, fetch_byte, sh.ln[k].jl, prev) : prev; // crt_core.c:431
                changed |= (nh[q] != sh.hs[k]);
            }
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < (kLines + kSyncThreads - 1) / kSyncThreads; q++) {
            const int k = tid + q * kSyncThreads;
            if (k < kLines) sh.hs[k] = nh[q];
        }
        if (!__syncthreads_or(changed)) break;
    }
    phase_mark(0, 4);

    // ---- 3b. burst lock (crt_core.c:456-467): ccr = ccr * 127 / 128 + sample, 10 samples per phase per line.
    // First one thread per decoded line gathers the line's 40 burst samples (their position depends on hsync, now known)
    // into shared memory, sorted by carrier phase -- sample t belongs to phase (t + CB_BEG) % CC, step t / CC -- so that the
    // serial chain below is nothing but one 16-byte load per line and the recurrence.
    for (int k = tid; k < kLines; k += kSyncThreads) {
        if (sh.ln[k].beg < 0) continue; // (never on a colour row's list)
        const int hs = sh.hs[k], jl = sh.ln[k].jl;
        const int p = jl * kHres + (hs - hs % kCc) + kCbBeg; // crt_core.c:458-462 (hs >= 0: "& ~3" when kCc == 4)
        const int j = (hs > kHres / 2) ? jl + 1 : jl;
        const int off = p - ((j * kHres - kHeadBefore) & ~3);
        signed char *dst = reinterpret_cast<signed char *>(&sh.burst[k][0]);
        if (j < kHeadLines && off >= 0 && off + kBurstLen <= kHeadWords * 4) {
            const signed char *hb = reinterpret_cast<const signed char *>(heads + j * kHeadWords) + off;
#pragma unroll
            for (int t = 0; t < kBurstLen; t++) dst[((t + kCbBeg) % kCc) * 16 + t / kCc] = hb[t];
        } else {
            for (int t = 0; t < kBurstLen; t++) dst[((t + kCbBeg) % kCc) * 16 + t / kCc] = (signed char) fetch_byte(p + t);
        }
    }
    __syncthreads();
    phase_mark(0, 5);
    if (warp == kChainWarp) {
        // Lane = kCc * row + phase walks its own colour row's lines (at most 5 x 5 = 25 lanes).
        static_assert(kCc * kVper <= 32, "one lane per (colour row, phase)");
        const bool chain_lane = lane < kCc * kVper;
        const int row = chain_lane ? lane / kCc : 0, phase = chain_lane ? lane % kCc : 0;
        int x = chain_lane ? st->ccf[row][phase] : 0;
        const int count = chain_lane ? sh.rowcount[row] : 0;
        const short *rl = sh.rowlist[row];
        // One line, exactly.  C's x * 127 / 128 truncates towards zero; while the product cannot wrap it equals
        // x - ((x + (x >= 0 ? 127 : 0)) >> 7): ceil(x / 128) for x >= 0, floor for x < 0.
        auto exact_line = [&](int v, const int (&b)[kBurstSteps]) {
            if (abs(v) < (1 << 23)) {
#pragma unroll
                for (int q = 0; q < kBurstSteps; q++) v = v - ((v + ((v >= 0) ? 127 : 0)) >> 7) + b[q];
            } else {
#pragma unroll
                for (int q = 0; q < kBurstSteps; q++) v = wadd(wmul(v, 127) / 128, b[q]);
            }
            return v;
        };
        // The serial part proper.  floor and ceil differ by a sign: with v = -x while x >= 0 (and the samples subtracted) and
        // v = x while x < 0, BOTH cases are v -= v >> 7 (v <= 0: floor(v / 128)), then the sample -- a step is shift,
        // three-input add, two dependent instructions, for as long as v stays <= 0, which it does: the sign of x almost never
        // changes, within a line or from one line to the next.  Whether a line kept it (the largest v after any step: one
        // max per step, beside the chain) and was small enough for the shortcut is looked at one line LATE, so that no branch
        // waits for the end of a chain; a line that did not is redone exactly together with its successor.
        auto samples = [&](const uint4 &c, int (&b)[kBurstSteps]) {
            const unsigned cw[4] = { c.x, c.y, c.z, c.w };
#pragma unroll
            for (int q = 0; q < kBurstSteps; q++) b[q] = (int) (signed char) (cw[q >> 2] >> (8 * (q & 3)));
        };
        int mode = (x >= 0) ? 1 : 0; // 1: v = -x
        int v = mode ? -x : x;
        int pend_k = 0, pend_x = 0, pend_verdict = -1; // the line before the current one: record, starting x, >= 0 = redo
        // the line after the current one is loaded while the current one's ten dependent steps run
        int k = (count > 0) ? rl[0] : 0, k1 = (count > 1) ? rl[1] : k;
        uint4 cur = sh.burst[k][phase];
        for (int n = 0; n < count; n++) {
            const uint4 nxt = sh.burst[k1][phase];
            const int k2 = (n + 2 < count) ? rl[n + 2] : k1;
            int bs[kBurstSteps];
            samples(cur, bs);
            const int v0 = v;
            int vv = v, top = -0x7fffffff - 1; // (the largest v after any step)
            // (one instruction stream for both directions -- the lanes of a warp differ in theirs: the samples take the sign)
            const int sg = mode ? -1 : 1;
            int be[kBurstSteps];
#pragma unroll
            for (int q = 0; q < kBurstSteps; q++) {
                be[q] = mode ? -bs[q] : bs[q]; // (not "* sg": ptxas folds a multiplication into the chain's add, a third dependent instruction per step)
            }
#pragma unroll
            for (int q = 0; q < kBurstSteps; q++) {
                vv = vv - (vv >> 7) + be[q];
                top = max(top, vv);
            }
            // negative: the shortcut held for this line (no step started from a v > 0) and holds for the start of the next.
            // v == 0 is fine -- floor and ceil agree there -- and must be: a carrier phase that samples the burst at its zero
            // crossing (the NES has one) keeps its accumulator at exactly 0.
            const int verdict = (top <= 0 && v0 > -(1 << 23)) ? -1 : 0;
            if (pend_verdict >= 0) { // (rare) the previous line's did not: this line started from a wrong value
                int pb[kBurstSteps];
                samples(sh.burst[pend_k][phase], pb);
                x = exact_line(pend_x, pb);
                sh.ccr[pend_k][phase] = x;
                x = exact_line(x, bs);
                sh.ccr[k][phase] = x;
                mode = (x >= 0) ? 1 : 0;
                v = mode ? -x : x;
                pend_verdict = -1;
            } else {
                sh.ccr[k][phase] = wmul(vv, sg); // (provisional if this line's verdict says so: rewritten next time round)
                pend_k = k;
                pend_x = wmul(v0, sg);
                pend_verdict = verdict;
                v = vv;
            }
            k = k1;
            k1 = k2;
            cur = nxt;
        }
        if (pend_verdict >= 0) {
            int pb[kBurstSteps];
            samples(sh.burst[pend_k][phase], pb);
            x = exact_line(pend_x, pb);
            sh.ccr[pend_k][phase] = x;
        } else {
            x = mode ? -v : v;
        }
        if (chain_lane) st->ccf[row][phase] = x;
        if (lane == 0) {
            st->vsync = vs;
            st->hsync = sh.hs[kLines - 1];
            st->field = field;
            if (!kIsVhs) st->rn = (int) (rn0 * kLcgField.mul + kLcgField.add); // crt_core.c:367
        }
        phase_mark(0, 6, kChainWarp * 32);
    }
    // ---- 3c. the noise pass proper (crt_core.c:346-367): analog -> inp, 16 samples per thread per round, 128-bit accesses,
    // by the seven warps that would otherwise wait for the chain (which joins them when it is through)
    if (kFusedNoise && !inp_late) {
        for (;;) {
            int c = 0;
            if (lane == 0) c = atomicAdd(&sh.noise_next, 1);
            c = __shfl_sync(0xffffffffu, c, 0);
            if (c >= kNoiseChunks) break;
            const int t0 = c * kNoiseChunkVecs + lane;
            // largest |sample| of the vector's 16 bytes (already clamped to +-127), credited to the signal line(s) they lie in
            auto track_vec = [&](uint4 v, int i0) {
                unsigned a = max127_4(max127_4(abs127_4(v.x), abs127_4(v.y)), max127_4(abs127_4(v.z), abs127_4(v.w)));
                a = max127_4(a, a >> 16);
                const int mx = (int) (max127_4(a, a >> 8) & 0xffu);
                const int l0 = i0 / kHres, l1 = min(i0 + kNoiseVec - 1, kInputSize - 1) / kHres;
                if (mx > sh.linemax[l0]) atomicMax(&sh.linemax[l0], mx);
                if (l1 != l0 && mx > sh.linemax[l1]) atomicMax(&sh.linemax[l1], mx);
            };
            auto inside_inp = [&](uint4 v, int i0) { // the vector's bytes inside inp[], 0 behind it (not signal)
                unsigned w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int left = kInputSize - i0 - 4 * e; // bytes of word e inside inp[]
                    w[e] = (left <= 0) ? 0u : (left >= 4) ? w[e] : (w[e] & (0xffffffffu >> (8 * (4 - left))));
                }
                return make_uint4(w[0], w[1], w[2], w[3]);
            };
            if (noise == 0 && (c + 1) * kNoiseChunkVecs * kNoiseVec <= kInputSize) { // whole vectors, no noise term: the stock case
                uint4 in[kNoiseNB];
#pragma unroll
                for (int u = 0; u < kNoiseNB; u++) in[u] = *reinterpret_cast<const uint4 *>(analog + (t0 + 32 * u) * kNoiseVec);
#pragma unroll
                for (int u = 0; u < kNoiseNB; u++) {
                    if ((t0 + 32 * u + 1) * kNoiseVec > kInputSize) __builtin_unreachable(); // (a whole chunk: no partial vector)
                    in[u] = clamp127_v(in[u]);
                    store_inp_vec(inp_w, t0 + 32 * u, in[u]);
                }
                if (track) {
#pragma unroll
                    for (int u = 0; u < kNoiseNB; u++) track_vec(in[u], (t0 + 32 * u) * kNoiseVec);
                }
                continue;
            }
#pragma unroll 2
            for (int u = 0; u < kNoiseNB; u++) {
                const int t = t0 + 32 * u;
                if (t >= kNoiseThreads) continue;
                const int i0 = t * kNoiseVec;
                uint4 v = noisy_vec(*reinterpret_cast<const uint4 *>(analog + i0), t, noise, rn0, jump_lo, jump_hi);
                store_inp_vec(inp_w, t, v);
                if (track) track_vec(i0 + kNoiseVec <= kInputSize ? v : inside_inp(v, i0), i0);
            }
        }
        phase_mark(0, 7);
    }
    __syncthreads();
    phase_mark(0, 8);

    // Spans above kMonotonicSpan (a v_fac near 2^31, or one that wraps outh + v_fac to a huge span): beg and end wrap, so
    // a line's rows may overlap those of any earlier line, not only of its neighbours.  The reference applies such lines
    // in order.  Line k's level is 1 + the highest level of an earlier line whose written rows [beg, beg + nrows) overlap
    // its own (0 if none does).  Lines of one level write disjoint rows, and the host runs one line pass per level, in
    // order.  One warp walks the lines; it is a pathological geometry and this is not a fast path.
    const bool by_level = row_span(cfg) > kMonotonicSpan;
    if (by_level) {
        if (warp == 0) {
            for (int k = 0; k < kLines; k++) {
                const SyncLine g = sh.ln[k];
                if (g.beg < 0) continue;
                const int e = g.beg + rows_written(g, cfg.scanlines);
                int lv = -1;
                for (int j = lane; j < k; j += 32) {
                    const SyncLine h = sh.ln[j];
                    if (h.beg >= 0 && h.beg < e && g.beg < h.beg + rows_written(h, cfg.scanlines)) lv = max(lv, (int) sh.level[j]);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) lv = max(lv, __shfl_xor_sync(0xffffffffu, lv, o));
                if (lane == 0) sh.level[k] = (short) (lv + 1);
                __syncwarp();
            }
        }
        __syncthreads();
    }

    // ---- 4. per-line records for k_lines (crt_core.c:452-454, 469-479), all threads
    int huesn, huecs;
    {
        int sn, cs;
        sincos14_d(sn, cs, ((cfg.hue % 360) + 33) * 8192 / 180); // crt_core.c:318-320
        huesn = sn >> 11;
        huecs = cs >> 11;
    }
    for (int k = tid; k < kLines; k += kSyncThreads) {
        const SyncLine g = sh.ln[k];
        const int hs = sh.hs[k];
        LineRec rec;
        // When the output has fewer rows than there are decoded lines, consecutive lines land on the same
        // row and the reference applies them in order (each one blending onto, or overwriting, its
        // predecessor).  run_pos = position of this line within its run, run_last = 1 for the run's last line;
        // the host then launches the line kernel once per position (crtx.cu: line_passes).  Spans above kMonotonicSpan:
        // run_pos = level.
        int rank = 0;
        if (by_level) rank = (g.beg >= 0) ? sh.level[k] : 0;
        else for (int j = k - 1; j >= 0 && g.beg >= 0 && sh.ln[j].beg == g.beg; j--) rank++;
        rec.run_pos = rank;
        rec.run_last = (k == kLines - 1 || sh.ln[k + 1].beg != g.beg) ? 1 : 0;
        rec.hsync = hs;
        rec.beg = g.beg;
        rec.end = g.end;
        rec.pos = 0;
        rec.wave0 = rec.wave1 = 0;
        if (g.beg >= 0) {
            rec.pos = posmod(kAvBeg + hs - 3, kHres) + g.ypos * kHres;
            long long wmax;
            if (kCc == 4) {
                const int pa = hs & 3;
                const int dci = wsub(sh.ccr[k][(pa + 1) & 3], sh.ccr[k][(pa + 3) & 3]);
                const int dcq = wsub(sh.ccr[k][(pa + 2) & 3], sh.ccr[k][pa]);
                rec.wave0 = wmul(wsub(wmul(dci, huecs), wmul(dcq, huesn)) >> 4, cfg.saturation);
                rec.wave1 = wmul(wadd(wmul(dcq, huecs), wmul(dci, huesn)) >> 4, cfg.saturation);
                wmax = max(llabs((long long) rec.wave0), llabs((long long) rec.wave1));
            } else { // crt_core.c:480-509: the record carries dci / dcq, the line kernel rebuilds the ten carrier values
                const int pa = hs % kCc, peak = pa + kCc / 4;
                const int *ccr = sh.ccr[k];
                const int dci = wsub(ccr[peak % kCc], wadd(ccr[(peak + kCc / 2) % kCc], ccr[(peak + kCc / 2 + 1) % kCc]) / 2);
                const int dcq = wsub(ccr[(pa + kCc / 2) % kCc], ccr[pa % kCc]);
                rec.wave0 = dci;
                rec.wave1 = dcq;
                int wi[5], wq[5];
                pv1k_waves(dci, dcq, cfg.hue, cfg.saturation, wi, wq);
                wmax = 0;
#pragma unroll
                for (int i = 0; i < 5; i++) wmax = max(wmax, max(llabs((long long) wi[i]), llabs((long long) wq[i])));
            }
            // The fast equaliser path of k_lines is exact while every chroma input (s * wave) >> 9 stays
            // within +-16383 (crt_lines.cuh).  The line reads samples [pos, pos + AV_LEN).  Inside inp[] |s| <= 127 (the
            // clamp of crt_core.c:363-364); a window that runs past the end of inp[] (the PV-1000's last signal line, in
            // ordinary operation) also reads the struct tail behind it (k_struct_tail), bytes that are neither clamped nor
            // measured below, and -128 whenever a byte of outw or outh is 0x80 (outw = 640): such a line counts |s| = 128.
            // With the stock saturation that bound already passes and nothing more is needed; only a line whose carrier is
            // large enough to fail it needs the real maximum of its two signal lines.  Measuring that costs about as much as
            // the copy itself, so it is done only for monitors that needed it the last time (MonState::track_max: the NES and
            // NES-RGB systems at their stock saturation, nothing else at stock settings), inside the copy that runs beside the
            // burst-lock chain; the first pass of such a monitor scans the two lines here instead, one thread per line, slowly.
            const int stail = (rec.pos + kAvLen > kInputSize) ? 128 : 0;
            if (stail && inp_late) sh.need_inp = 1;
            int smax = max(127, stail);
            if (kFusedNoise && ((smax * wmax) >> 9) + 1 > 16383) {
                sh.need_max = 1; // (the next pass of this monitor measures while it copies)
                if (track) {
                    smax = max(sh.linemax[g.ypos], sh.linemax[g.ypos + 1]);
                } else {
                    const int lo = (g.ypos * kHres) & ~15, hi = min((g.ypos + 2) * kHres, kInputSize);
                    int mx = 0;
                    const signed char *sig = inp_late ? analog : inp_w; // (the clamp: inp[] not written yet)
                    for (int i = lo; i < hi; i++) mx = max(mx, abs(max((int) sig[i], -127)));
                    smax = mx;
                }
                smax = max(smax, stail);
            }
            if (((smax * wmax) >> 9) + 1 > 16383) sh.generic = 1;
        }
        lines[k] = rec;
    }
    __syncthreads();
    if (inp_late && (sh.generic || sh.need_inp)) {
        for (int t = tid; t < kNoiseThreads; t += kSyncThreads) store_inp_vec(inp_w, t, clamp127_v(__ldg(reinterpret_cast<const uint4 *>(analog) + t)));
        inp_late = false;
    }
    if (tid == 0) {
        st->generic = sh.generic;
        st->inp_late = inp_late;
        if (kFusedNoise) st->track_max = sh.need_max;
    }
    phase_mark(0, 14);
}

} // namespace crt
