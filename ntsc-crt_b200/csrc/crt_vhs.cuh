// crt_vhs.cuh -- the VHS variant's noise pass in the batch interface (crt_core.c:343-367).
//
// The reference draws its VHS noise from libc rand(): one draw per call for the wobble, then per
// sample one draw for the noise value, one for the first bound of the "bottom of frame" band and --
// short-circuit && -- a third only when the first test passed.  The drop-in calls (crt_dropin.cu) keep
// drawing from the process's libc on the host; the batch interface carries, per monitor, a replica of
// glibc's TYPE_3 generator (o[n] = o[n-31] + o[n-3] mod 2^32, output o[n] >> 1; glibc 2.39
// stdlib/random_r.c) seeded by crtx_seed, and this kernel reproduces the reference's draw order exactly:
//
//   bulk   samples [0, kVhsBulk): the first test can never pass there (it needs i > INPUT_SIZE - 25 lines),
//          so every sample costs exactly two draws.  256 threads each own a contiguous run of samples; the
//          generator state at the start of every run comes from jump-ahead matrices (powers of the
//          31 x 31 transition matrix, doubling tree), then each thread steps the recurrence in registers.
//   tail   the last ~26.5 lines, where the draw count is data dependent.  The raw stream for the whole
//          tail is generated in parallel the same way; the walk "sample -> position of its first draw" is
//          then resolved per signal line by pointer jumping (within a line the tests' thresholds are
//          constant, so next(p) = p + 2 + [test1(raw[p + 1])] is a function of p alone): 10 doubling
//          rounds give every sample its position, after which all samples of the line are evaluated in
//          parallel with the reference's literal expressions.
// Round 2: runs of 868 samples = 7 blocks of 124 (four generator periods), so that every thread's share of a block is
// 31 aligned 32-bit words: the terms meet the signal 4 samples per lane with word loads and stores.  The two regions run as
// two CTAs per monitor at once (blockIdx.y: 0 tail, 1 bulk) -- the tail's start state is the
// bulk's 256 runs applied as two level-7 jumps -- and the tail only builds tables where the count is really data
// dependent: within signal line L the first test of sample x >= 1 is (draw % 20) >= 256 - L, so lines up to 236 always
// take two draws and lines from 256 on always three (closed-form positions); for the 19 lines in between the successor
// table is doubled five times (1, 2, 4, 8, 16, 32 steps) instead of nine, one thread walks the 29 chunk starts with
// the 32-step table, and a sample finishes with five look-ups.  The generator state after the call goes to a second
// array that k_vhs_commit copies back, because the bulk CTA of the same monitor may not have read the old one yet.
#pragma once

#include "crt_kernels.cuh"

#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)

namespace crt {

constexpr int kVhsThreads = 256;
constexpr int kVhsPeriods = 4;                        // generator periods (31 samples, 62 draws) per block of a run
constexpr int kVhsSlice = 31 * kVhsPeriods;           // 124 samples: a thread's share of one block -- a whole number of 32-bit words
constexpr int kVhsRun = kVhsSlice * 7;                // 868 samples per run (2 draws each); every slice starts 4-byte aligned
constexpr int kVhsRuns = 248;                         // runs = generating threads of the bulk CTA (the doubling tree makes 256 states)
constexpr int kVhsBulk = kVhsRuns * kVhsRun;          // 215 264 <= INPUT_SIZE - 25 lines
constexpr int kVhsTailSamples = kInputSize - kVhsBulk;
constexpr int kVhsTailRun = 310;                      // raw values per thread for the tail (10 x 31)
constexpr int kVhsTailRaw = kVhsThreads * kVhsTailRun; // 79 360 >= 3 draws x tail samples
constexpr int kVhsWin = 2752;                         // raw values visible to one line's walk (>= 3 * 910 + 3)
constexpr int kVhsLevels = 8;                         // doubling levels: 2^8 = 256 runs
constexpr int kVhsJLevels = 6;                        // tail walk: successor tables for 1, 2, 4, 8, 16, 32 steps
constexpr int kVhsChunk = 1 << (kVhsJLevels - 1);     // samples per chunk of the walk (32)
constexpr int kVhsChunks = (kHres + kVhsChunk - 1) / kVhsChunk + 1;
static_assert(kVhsBulk <= kInputSize - 25 * kHres, "bulk region must stay clear of the data-dependent band");
static_assert(kVhsRun % 4 == 0 && kVhsSlice % 4 == 0 && kVhsRuns <= kVhsThreads, "bulk slices are whole aligned words");
static_assert(kVhsTailRaw >= 3 * kVhsTailSamples + 64 && kVhsWin >= 3 * kHres + 8, "tail stream sizes");

struct VhsRand { // generator state: the last 31 raw values, oldest first
    unsigned hist[31];
    unsigned pad;
};

struct VhsJump { // powers of the transition matrix, [level][row][col], applied as new = A * old
    unsigned bulk[kVhsLevels][31][31]; // (M^(2 * kVhsRun))^(2^level)
    unsigned tail[kVhsLevels][31][31]; // (M^kVhsTailRun)^(2^level)
    unsigned field[2][31][31];         // M^(ab + 1 + 2 * kVhsBulk): a field's draws before its tail, ab = the aberration draw
};

// one draw on a chronological state held in shared/global memory (used for the odd single draws)
__device__ __forceinline__ unsigned vhs_draw_mem(unsigned *h)
{
    const unsigned v = h[0] + h[28];
    for (int j = 0; j < 30; j++) h[j] = h[j + 1];
    h[30] = v;
    return v >> 1;
}

// states[t + 2^k] = A_k * states[t] for t < 2^k, k = 0 .. kVhsLevels - 1: after it states[0 .. 256]
// hold the generator state at the start of every run (and, at [256], after the last one).
__device__ __forceinline__ void vhs_spread_states(unsigned (*states)[32], const unsigned (*A)[31][31], int tid,
                                                  unsigned *Am /* shared, 31 * 31 words */)
{
    const int warp = tid >> 5, lane = tid & 31;
    for (int k = 0; k <= kVhsLevels; k++) {
        const int half = 1 << k; // states [0, half) known; fill [half, 2 * half) (level 8 fills only [256])
        if (k < kVhsLevels) { // this level's matrix into shared memory (row stride 31: conflict-free rows)
            const unsigned *src = &A[k][0][0];
            for (int e = tid; e < 31 * 31; e += kVhsThreads) Am[e] = __ldg(src + e);
            __syncthreads();
        } // level 8 reuses A^(128), still resident
        const int todo = (k < kVhsLevels) ? half : 1;
        for (int t = warp; t < todo; t += kVhsThreads / 32) {
            const int from = (k < kVhsLevels) ? t : 128, to = (k < kVhsLevels) ? t + half : 256;
            if (lane < 31) {
                unsigned acc = 0;
#pragma unroll
                for (int j = 0; j < 31; j++) acc += Am[lane * 31 + j] * states[from][j];
                states[to][lane] = acc;
            }
        }
        __syncthreads();
    }
}

// the reference's literal tests (crt_core.c:350-351) for sample i given the two draws
__device__ __forceinline__ bool vhs_test1(int i, unsigned a) { return i > (kInputSize - kHres * (16 + ((int) (a % 20u) - 10))); }
__device__ __forceinline__ bool vhs_test2(int i, unsigned b) { return i < (kInputSize - kHres * (5 + ((int) (b % 8u) - 4))); }

// new = A * old on chronological states in shared memory (warp 0 computes, everybody synchronises)
__device__ __forceinline__ void vhs_apply(unsigned *to, const unsigned (*A)[31], const unsigned *from, int tid, unsigned *Am)
{
    const unsigned *src = &A[0][0];
    for (int e = tid; e < 31 * 31; e += kVhsThreads) Am[e] = __ldg(src + e);
    __syncthreads();
    if (tid < 31) {
        unsigned acc = 0;
#pragma unroll
        for (int j = 0; j < 31; j++) acc += Am[tid * 31 + j] * from[j];
        to[tid] = acc;
    }
    __syncthreads();
}

// draws per regular sample (x >= 1) of signal line `line` where that number does not depend on the data, else 0: within
// the line the first test of sample x >= 1 is (draw % 20) >= need (crt_core.c:350 with i = line * HRES + x)
__device__ __forceinline__ int vhs_fixed_draws(int line)
{
    const int need = (kInputSize / kHres - 6) - line;
    return (need > 19) ? 2 : (need <= 0) ? 3 : 0;
}

// One line of the tail walk, samples xa .. kHres - 1 of signal line `line` (i0 = line * kHres + xa), whose first draw is
// raw[D]: win = raw[D ..], *s_start = the position of its first regular sample in win, and where the line's draw count
// depends on the data, jt[k][p] = the position 2^k regular samples after position p (k < kVhsJLevels).  Within a line
// the first test is the same function of its draw for every sample except x == 0 (its bound is a multiple of the line
// length), so x == 0 is stepped on its own and the regular samples start at x0 = 1 (or at xa > 0).  k_vhs_skip walks
// with these tables; k_noise_vhs runs the same steps inline, interleaved with its chunk table, which keeps its machine
// code as it was (the compiler schedules the shared version differently there).
__device__ __forceinline__ void vhs_line_tables(unsigned *win, unsigned short *jt, int *s_start, const unsigned *raw, int D,
                                                int i0, int xa, int line, int fixed, int tid)
{
    { // all of a thread's window loads in flight together
        constexpr int kPer = (kVhsWin + 8 + kVhsThreads - 1) / kVhsThreads;
        unsigned v[kPer];
#pragma unroll
        for (int u = 0; u < kPer; u++) {
            const int q = tid + u * kVhsThreads;
            v[u] = (q < kVhsWin + 8 && D + q < kVhsTailRaw) ? raw[D + q] : 0u;
        }
#pragma unroll
        for (int u = 0; u < kPer; u++) {
            const int q = tid + u * kVhsThreads;
            if (q < kVhsWin + 8) win[q] = v[u];
        }
    }
    __syncthreads();
    if (tid == 0) {
        int p = 0;
        if (xa == 0) p = 2 + (vhs_test1(i0, win[1] >> 1) ? 1 : 0);
        *s_start = p; // position of the first "regular" sample
    }
    if (!fixed) {
        const int irep = line * kHres + 1;
        for (int p = tid; p < kVhsWin + 8; p += kVhsThreads)
            jt[p] = (unsigned short) ((p + 3 < kVhsWin) ? p + 2 + (vhs_test1(irep, win[p + 1] >> 1) ? 1 : 0) : kVhsWin);
        __syncthreads();
        for (int k = 1; k < kVhsJLevels; k++) { // jt[k][p] = 2^k-th successor
            unsigned short *prev = jt + (k - 1) * (kVhsWin + 8), *cur = jt + k * (kVhsWin + 8);
#pragma unroll 4
            for (int p = tid; p < kVhsWin + 8; p += kVhsThreads) cur[p] = prev[min((int) prev[p], kVhsWin)];
            __syncthreads();
        }
    }
}

// The tail CTA's raw stream: from the state at the start of the tail in states[0], raw[0 .. kVhsTailRaw) = the next
// kVhsTailRaw raw values of the generator (jumps of kVhsTailRun values spread the start states over the threads).
// Ends with the block synchronised; `states` may then be overlaid.
__device__ __forceinline__ void vhs_tail_stream(unsigned (*states)[32], const VhsJump *jump, unsigned *raw, int tid, unsigned *Am)
{
    vhs_spread_states(states, jump->tail, tid, Am);
    {
        unsigned h[31];
#pragma unroll
        for (int j = 0; j < 31; j++) h[j] = states[tid][j];
        for (int it = 0; it < kVhsTailRun / 31; it++) {
#pragma unroll
            for (int d = 0; d < 31; d++) {
                h[d] += h[(d + 28) % 31];
                raw[tid * kVhsTailRun + it * 31 + d] = h[d];
            }
        }
    }
    __syncthreads(); // (block-wide: the stream is visible to every thread; `states` may now be overlaid)
}

__global__ void __launch_bounds__(kVhsThreads, 4) k_noise_vhs(const MonCfg *__restrict__ cfgs, MonState *__restrict__ states_mon,
                                                           const VhsRand *__restrict__ rands, VhsRand *__restrict__ rands_next,
                                                           const VhsJump *__restrict__ jump,
                                                           unsigned *__restrict__ raw_base,
                                                           const signed char *__restrict__ analog_base,
                                                           signed char *__restrict__ inp_base, int first)
{
    extern __shared__ __align__(16) unsigned char vsm[];
    unsigned (*states)[32] = reinterpret_cast<unsigned (*)[32]>(vsm);                 // [257][32]
    // the tail's tables overlay the run states, which are dead once the raw stream is generated
    unsigned *win = reinterpret_cast<unsigned *>(vsm);                                  // tail: [kVhsWin + 8]
    unsigned short *jt = reinterpret_cast<unsigned short *>(win + kVhsWin + 8);         // tail: [kVhsJLevels][kVhsWin + 8]
    int *cs = reinterpret_cast<int *>(jt + kVhsJLevels * (kVhsWin + 8));                // tail: [kVhsChunks] chunk start positions
    __shared__ int s_wobble, s_adv, s_start;
    __shared__ unsigned s_mat[31 * 31];
    const int m = first + blockIdx.x, tid = threadIdx.x;
    const bool tail_role = blockIdx.y == 0; // (the tail CTAs are the longer ones: they are scheduled first)
    if (cfgs[m].bpp == 0) { // crt_core.c:312-315: no draws, the generator state stays
        if (tail_role && tid < 32) reinterpret_cast<unsigned *>(&rands_next[m])[tid] = reinterpret_cast<const unsigned *>(&rands[m])[tid];
        return;
    }
    const int noise = cfgs[m].noise;
    const signed char *analog = analog_base + (size_t) m * kSignalBytes;
    signed char *inp = inp_base + (size_t) m * kSignalBytes;
    unsigned *raw = raw_base + (size_t) blockIdx.x * kVhsTailRaw;
    const VhsRand *rs = &rands[m];

    // ---- the wobble draw (crt_core.c:344), then the run start states
    if (tid == 0) {
        unsigned h[31];
        for (int j = 0; j < 31; j++) h[j] = rs->hist[j];
        s_wobble = ((int) (vhs_draw_mem(h) % 8u) - 4) + 14;
        for (int j = 0; j < 31; j++) states[0][j] = h[j];
    }
    __syncthreads();

    if (!tail_role) {
        vhs_spread_states(states, jump->bulk, tid, s_mat);
        // ---- bulk: thread t < kVhsRuns owns samples [t * kVhsRun, (t + 1) * kVhsRun), two draws each.  Per block of
        // kVhsSlice samples: (1) every thread generates its slice's noise terms into shared memory, (2) the CTA adds
        // them to the signal -- slice by slice, 31 lanes x one aligned 32-bit word (4 samples) each, so global traffic
        // is whole words and coalesced although a thread's slices lie kVhsRun bytes apart.
        unsigned h[31];
#pragma unroll
        for (int j = 0; j < 31; j++) h[j] = states[min(tid, kVhsRuns - 1)][j];
        __syncthreads(); // the run states are in registers: the terms buffer may overlay them
        short *terms = reinterpret_cast<short *>(vsm); // [kVhsRuns][kVhsSlice]
        constexpr int kSlicesPerWarp = (kVhsRuns + 7) / 8; // 31 slices per warp per block
        const int warp = tid >> 5, lane = tid & 31;
        for (int it = 0; it < kVhsRun / kVhsSlice; it++) {
            if (tid < kVhsRuns) {
#pragma unroll
                for (int pr = 0; pr < kVhsPeriods; pr++) {
#pragma unroll
                    for (int d = 0; d < 62; d++) { // draw d of a period uses slot d % 31 (31-periodic alignment)
                        const int slot = d % 31;
                        h[slot] += h[(slot + 28) % 31];
                        if ((d & 1) == 0) { // the noise draw; the odd draw feeds the never-true first test
                            const int rn = (int) (h[slot] >> 1);
                            int t = wmul(((rn >> 16) & 0xff) - 0x7f, noise) >> 8;
                            t = clampi(t, -255, 255); // analog is within [-128, 127]: beyond +-255 the sum saturates anyway
                            terms[tid * kVhsSlice + pr * 31 + (d >> 1)] = (short) t;
                        }
                    }
                }
            }
            __syncthreads();
            // apply: eight slices per batch, their signal words requested together (the register budget of the whole kernel
            // is what lets every CTA of a launch be resident at once)
#pragma unroll 1
            for (int q0 = 0; q0 < kSlicesPerWarp; q0 += 8) {
                unsigned sig[8];
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const int u = warp + 8 * (q0 + q);
                    sig[q] = (q0 + q < kSlicesPerWarp && u < kVhsRuns && lane < kVhsSlice / 4)
                                 ? __ldg(reinterpret_cast<const unsigned *>(analog + u * kVhsRun + it * kVhsSlice) + lane) : 0u;
                }
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const int u = warp + 8 * (q0 + q);
                    if (q0 + q < kSlicesPerWarp && u < kVhsRuns && lane < kVhsSlice / 4) {
                        const uint2 tw = *reinterpret_cast<const uint2 *>(terms + u * kVhsSlice + 4 * lane);
                        const unsigned tws[2] = { tw.x, tw.y };
                        unsigned o = 0;
#pragma unroll
                        for (int b = 0; b < 4; b++) {
                            const int sg = (int) (signed char) (sig[q] >> (8 * b));
                            const int tm = (int) (short) (tws[b >> 1] >> (16 * (b & 1)));
                            o |= ((unsigned) clampi(sg + tm, -127, 127) & 0xffu) << (8 * b);
                        }
                        reinterpret_cast<unsigned *>(inp + u * kVhsRun + it * kVhsSlice)[lane] = o;
                    }
                }
            }
            __syncthreads();
        }
        return;
    }

    // ---- tail CTA: the state after the bulk's 256 runs = two jumps of 128 runs (level 7), then the raw stream
    { // kVhsRuns = 248 = 128 + 64 + 32 + 16 + 8 runs: one jump per set bit (levels 7, 6, 5, 4, 3)
        int cur = 0;
        for (int k = kVhsLevels - 1; k >= 0; k--)
            if ((kVhsRuns >> k) & 1) {
                vhs_apply(states[cur ^ 1], jump->bulk[k], states[cur], tid, s_mat);
                cur ^= 1;
            }
        if (cur) {
            if (tid < 31) states[0][tid] = states[1][tid];
            __syncthreads();
        }
    }
    vhs_tail_stream(states, jump, raw, tid, s_mat);

    // ---- tail walk, one signal line (or the partial first one) at a time
    const int wobble = s_wobble;
    int D = 0;            // raw values consumed so far in the tail
    for (int i0 = kVhsBulk; i0 < kInputSize;) {
        const int line = i0 / kHres, xa = i0 - line * kHres, nx = kHres - xa; // samples xa .. 909 of this line
        const int fixed = vhs_fixed_draws(line);
        { // all of a thread's window loads in flight together
            constexpr int kPer = (kVhsWin + 8 + kVhsThreads - 1) / kVhsThreads;
            unsigned v[kPer];
#pragma unroll
            for (int u = 0; u < kPer; u++) {
                const int q = tid + u * kVhsThreads;
                v[u] = (q < kVhsWin + 8 && D + q < kVhsTailRaw) ? raw[D + q] : 0u;
            }
#pragma unroll
            for (int u = 0; u < kPer; u++) {
                const int q = tid + u * kVhsThreads;
                if (q < kVhsWin + 8) win[q] = v[u];
            }
        }
        __syncthreads();
        // Within a line the first test is the same function of its draw for every sample except x == 0
        // (its bound is a multiple of the line length), so x == 0 is stepped on its own.
        if (tid == 0) {
            int p = 0;
            if (xa == 0) p = 2 + (vhs_test1(i0, win[1] >> 1) ? 1 : 0);
            s_start = p; // position of the first "regular" sample
        }
        const int x0 = (xa == 0) ? 1 : xa; // first regular sample
        if (!fixed) {
            const int irep = line * kHres + 1;
            for (int p = tid; p < kVhsWin + 8; p += kVhsThreads)
                jt[p] = (unsigned short) ((p + 3 < kVhsWin) ? p + 2 + (vhs_test1(irep, win[p + 1] >> 1) ? 1 : 0) : kVhsWin);
            __syncthreads();
            for (int k = 1; k < kVhsJLevels; k++) { // jt[k][p] = 2^k-th successor
                unsigned short *prev = jt + (k - 1) * (kVhsWin + 8), *cur = jt + k * (kVhsWin + 8);
#pragma unroll 4
                for (int p = tid; p < kVhsWin + 8; p += kVhsThreads) cur[p] = prev[min((int) prev[p], kVhsWin)];
                __syncthreads();
            }
            if (tid == 0) { // chunk c starts kVhsChunk * c regular samples after the first one
                const unsigned short *far = jt + (kVhsJLevels - 1) * (kVhsWin + 8);
                int p = s_start;
                const int chunks = (kHres - x0 + kVhsChunk - 1) / kVhsChunk;
                for (int c = 0; c < chunks; c++) {
                    cs[c] = p;
                    p = far[min(p, kVhsWin)];
                }
            }
        }
        __syncthreads();
        for (int x = xa + tid; x < kHres; x += kVhsThreads) {
            const int sig = analog[line * kHres + x]; // requested before the (dependent) table walk
            int P = 0;
            if (!(xa == 0 && x == 0)) {
                const int e = x - x0;
                if (fixed) {
                    P = s_start + fixed * e;
                } else {
                    P = cs[e / kVhsChunk];
#pragma unroll
                    for (int k = 0; k < kVhsJLevels - 1; k++)
                        if ((e >> k) & 1) P = jt[k * (kVhsWin + 8) + min(P, kVhsWin)];
                }
            }
            const int i = line * kHres + x;
            const int rn = (int) (win[P] >> 1);
            int gain = noise, used = 2;
            if (vhs_test1(i, win[P + 1] >> 1)) { // crt_core.c:350-357
                used = 3;
                if (vhs_test2(i, win[P + 2] >> 1)) {
                    int sn, cs14;
                    sincos14_d(sn, cs14, ((i * wobble) / kHres) * 8192 / 180);
                    gain = cs14 >> 8;
                }
            }
            const int s = sig + (wmul(((rn >> 16) & 0xff) - 0x7f, gain) >> 8);
            inp[i] = (signed char) clampi(s, -127, 127);
            if (x == kHres - 1) { // the line's last sample closes the walk
                s_adv = P + used;
                if (i == kInputSize - 1) states_mon[m].rn = rn; // crt_core.c:367
            }
        }
        __syncthreads();
        D += s_adv;
        i0 += nx;
        __syncthreads();
    }
    // ---- the generator state after the call: the last 31 raw values consumed
    if (tid < 31) {
        // total draws: 1 + 2 * kVhsBulk + D; D >= 31 always (the tail spans > 24 000 samples)
        rands_next[m].hist[tid] = raw[D - 31 + tid];
    }
}

// rands_next -> rands for monitors [first, first + count): runs after k_noise_vhs on the same stream
__global__ void k_vhs_commit(VhsRand *__restrict__ rands, const VhsRand *__restrict__ rands_next, int first, int count)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count * 32) return;
    reinterpret_cast<unsigned *>(rands + first)[k] = reinterpret_cast<const unsigned *>(rands_next + first)[k];
}

// the aberration draw of crt_modulate (crt_ntscvhs.c:205-207), one thread per monitor
__global__ void k_vhs_aberration(SrcCfg *__restrict__ srcs, const int *__restrict__ wants, VhsRand *__restrict__ rands,
                                 int first, int count)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    int ab = 0;
    if (wants[k]) ab = ((int) (vhs_draw_mem(rands[first + k].hist) % 12u) - 8) + 14;
    srcs[first + k].aberration = ab;
}

constexpr int kVhsSmemBulk = (257 * 32 * 4 > kVhsRuns * kVhsSlice * 2) ? 257 * 32 * 4 : kVhsRuns * kVhsSlice * 2;
constexpr int kVhsSmemTail = (kVhsWin + 8) * 4 + kVhsJLevels * (kVhsWin + 8) * 2 + kVhsChunks * 4 + 16;
constexpr int kVhsSmem = (kVhsSmemBulk > kVhsSmemTail ? kVhsSmemBulk : kVhsSmemTail) > 257 * 32 * 4
                             ? (kVhsSmemBulk > kVhsSmemTail ? kVhsSmemBulk : kVhsSmemTail) : 257 * 32 * 4;
constexpr int kVhsSkipSmem = kVhsSmemTail > 257 * 32 * 4 ? kVhsSmemTail : 257 * 32 * 4; // the tail CTA's part of kVhsSmem

// Advance monitor first + b's replica by fields[b] modulate + demodulate pairs, b = blockIdx.x, without a signal: what a
// field draws depends on its own values alone, never on the images, the noise or the knobs.  Per field: the draws
// before the tail -- [the aberration draw, ab] + the wobble + two per bulk sample -- are one matrix (VhsJump::field[ab]);
// the tail's raw stream is generated as k_noise_vhs's tail CTA does, and walked line by line with the same tables: the
// line's draw count is s_start + fixed * samples where it does not depend on the data, else the position the successor
// tables give after its last sample.  The next field starts from the last 31 raw values consumed.  One CTA per monitor:
// each field's count depends on that field's values.  The state after the call goes to rands_next (k_vhs_commit).
__global__ void __launch_bounds__(kVhsThreads) k_vhs_skip(const int *__restrict__ fields, const VhsRand *__restrict__ rands,
                                                          VhsRand *__restrict__ rands_next, const VhsJump *__restrict__ jump,
                                                          unsigned *__restrict__ raw_base, int ab, int first)
{
    extern __shared__ __align__(16) unsigned char vsm[];
    unsigned (*states)[32] = reinterpret_cast<unsigned (*)[32]>(vsm);                 // [257][32]
    unsigned *win = reinterpret_cast<unsigned *>(vsm);                                  // walk: [kVhsWin + 8]
    unsigned short *jt = reinterpret_cast<unsigned short *>(win + kVhsWin + 8);         // walk: [kVhsJLevels][kVhsWin + 8]
    __shared__ unsigned s_mat[31 * 31];
    __shared__ unsigned s_cur[32]; // the generator state at the start of the next field
    __shared__ int s_start, s_adv;
    const int m = first + blockIdx.x, tid = threadIdx.x;
    unsigned *raw = raw_base + (size_t) blockIdx.x * kVhsTailRaw;
    if (tid < 32) s_cur[tid] = reinterpret_cast<const unsigned *>(&rands[m])[tid];
    __syncthreads();
    const int n = fields[blockIdx.x];
    for (int f = 0; f < n; f++) {
        vhs_apply(states[0], jump->field[ab], s_cur, tid, s_mat);
        vhs_tail_stream(states, jump, raw, tid, s_mat);
        int D = 0; // raw values consumed so far in the tail
        for (int i0 = kVhsBulk; i0 < kInputSize;) {
            const int line = i0 / kHres, xa = i0 - line * kHres;
            const int fixed = vhs_fixed_draws(line);
            const int e = kHres - ((xa == 0) ? 1 : xa); // regular samples of the line
            vhs_line_tables(win, jt, &s_start, raw, D, i0, xa, line, fixed, tid);
            if (tid == 0) { // the position after the line's last sample
                int p = s_start;
                if (fixed) {
                    p += fixed * e;
                } else {
                    const unsigned short *far = jt + (kVhsJLevels - 1) * (kVhsWin + 8);
                    for (int c = 0; c < (e >> (kVhsJLevels - 1)); c++) p = far[min(p, kVhsWin)];
#pragma unroll
                    for (int k = 0; k < kVhsJLevels - 1; k++)
                        if ((e >> k) & 1) p = jt[k * (kVhsWin + 8) + min(p, kVhsWin)];
                }
                s_adv = p;
            }
            __syncthreads();
            D += s_adv;
            i0 += kHres - xa;
            __syncthreads();
        }
        if (tid < 31) s_cur[tid] = raw[D - 31 + tid]; // D >= 31 always (the tail spans > 24 000 samples)
        __syncthreads();
    }
    if (tid < 32) reinterpret_cast<unsigned *>(&rands_next[m])[tid] = (tid < 31) ? s_cur[tid] : 0u;
}
static_assert(kInputSize % kHres == 0, "the tail's per-line test assumes whole signal lines");

} // namespace crt

#endif
