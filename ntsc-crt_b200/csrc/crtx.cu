// crtx.cu -- context, launches and the crtx_* C-ABI (include/crtx_batch.h).
//
// A context owns, in HBM, for each of its N monitors: analog[] and inp[] (CRT_INPUT_SIZE + slack,
// same flat layout as the host struct so they can be memcpy'd), the persistent decoder state, the
// per-line table the sync pre-pass hands to the line kernel, and the small configuration records.
// There is no CPU implementation behind any of these calls: a CUDA failure is reported, never
// papered over.
#include <cuda_runtime.h>

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cstddef>
#include <vector>

#include "crt_kernels.cuh"
#include "crtx_internal.h"

namespace crt {

static thread_local char g_error[512] = "";

int fail(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
    return 1;
}

#define CUDA_TRY(expr)                                                                           \
    do {                                                                                         \
        cudaError_t e_ = (expr);                                                                 \
        if (e_ != cudaSuccess) return fail("%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

static int check_range(const crtx_ctx *ctx, int first, int count)
{
    if (!ctx) return fail("null context");
    if (first < 0 || count < 0 || first + count > ctx->n) return fail("monitor range [%d, %d) outside [0, %d)", first, first + count, ctx->n);
    return 0;
}

static int upload_cfg(crtx_ctx *ctx, cudaStream_t stream)
{
    if (ctx->cfg_dirty_lo < ctx->cfg_dirty_hi) {
        const int lo = ctx->cfg_dirty_lo, hi = ctx->cfg_dirty_hi;
        // pageable source: staged before the call returns, so h_cfg may be edited right after
        CUDA_TRY(cudaMemcpyAsync(ctx->d_cfg + lo, ctx->h_cfg.data() + lo, sizeof(MonCfg) * (hi - lo),
                                 cudaMemcpyHostToDevice, stream));
        // the bytes that follow inp[] in the reference's struct CRT depend on the output geometry alone (crt_sync.cuh)
        if (ctx->tail_dirty_lo < ctx->tail_dirty_hi) {
            const int tlo = ctx->tail_dirty_lo, thi = ctx->tail_dirty_hi;
            k_struct_tail<<<(thi - tlo + 63) / 64, 64, 0, stream>>>(ctx->d_cfg, ctx->d_analog, ctx->d_inp, tlo, thi - tlo);
            ctx->launches += 1;
            ctx->tail_dirty_lo = ctx->n;
            ctx->tail_dirty_hi = 0;
        }
        ctx->cfg_dirty_lo = ctx->n;
        ctx->cfg_dirty_hi = 0;
        // a context may be driven from several streams over disjoint monitor ranges (crtx_frames_host, bench.py): the
        // others must not read d_cfg or the signal tails before this upload has landed
        if (!ctx->cfg_ready) CUDA_TRY(cudaEventCreateWithFlags(&ctx->cfg_ready, cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(ctx->cfg_ready, stream));
        ctx->cfg_stream = stream;
    } else if (ctx->cfg_ready && stream != ctx->cfg_stream) {
        CUDA_TRY(cudaStreamWaitEvent(stream, ctx->cfg_ready, 0)); // (free once the event has completed)
    }
    return 0;
}

template <bool FAST, int MODE, int FMT>
static void launch_lines_one(crtx_ctx *ctx, int count, int lo, const LinesGeom &geo, cudaStream_t stream)
{
    if constexpr (kConv) { // USE_CONVOLUTION build: one warp per decoded line (crt_lines_fir.cuh)
        // about two waves of resident CTAs (2 per SM) over the whole launch, see k_lines_fir; the generic
        // pass is normally empty and gets the smallest grid
        int gx = FAST ? (4 * ctx->sm_count + count - 1) / count : 1;
        gx = gx < 1 ? 1 : (gx > kFirGroups ? kFirGroups : gx);
        const dim3 grid(gx, count);
        k_lines_fir<FAST, MODE, FMT><<<grid, kFirWarps * 32, fir_smem<FAST>(), stream>>>(ctx->d_cfg, ctx->d_state, ctx->d_lines,
                                                                                      ctx->d_inp, lo, geo);
    } else { // (only the kernel a build uses is instantiated)
        k_lines<FAST, MODE, FMT><<<count, kLinesWarps * 32, lines_smem<FAST>(), stream>>>(ctx->d_cfg, ctx->d_state, ctx->d_lines,
                                                                                       ctx->d_inp, lo, geo);
    }
}

template <bool FAST>
static void launch_lines_mode(crtx_ctx *ctx, int count, int lo, const LinesGeom &geo, cudaStream_t stream)
{
    if (geo.bpp != 4) return launch_lines_one<FAST, 2, 0>(ctx, count, lo, geo, stream);
#define LL(F)                                                                                     \
    case F:                                                                                       \
        if (geo.blend) launch_lines_one<FAST, 1, F>(ctx, count, lo, geo, stream);                 \
        else launch_lines_one<FAST, 0, F>(ctx, count, lo, geo, stream);                           \
        break;
    switch (geo.out_format) {
        LL(CRT_PIX_FORMAT_ARGB) LL(CRT_PIX_FORMAT_RGBA) LL(CRT_PIX_FORMAT_ABGR) LL(CRT_PIX_FORMAT_BGRA)
    }
#undef LL
}

// k_lines2 (crt_lines2.cuh): two monitors per CTA, tabulated resampler.  Taken when the whole run qualifies: the stock
// IIR decoder, 4-byte pixels, every line owning its rows, a width the pixel ring covers, 16-byte aligned images.
#if CRTX_HAS_LINES2
static bool lines2_eligible(const crtx_ctx *ctx, int count, int lo, const LinesGeom &geo)
{
    if (!ctx->opt_lines2) return false;
    if (geo.bpp != 4 || geo.pass != -1 || !lines2_geometry_ok(geo.outw)) return false;
    for (int i = lo; i < lo + count; i++)
        if (reinterpret_cast<uintptr_t>(ctx->h_cfg[i].out) & 15) return false;
    return true;
}

template <int MODE, int FMT>
static void launch_lines2_one(crtx_ctx *ctx, int count, int lo, const LinesGeom &geo, cudaStream_t stream)
{
    k_lines2<MODE, FMT><<<(count + 1) / 2, kL2Threads, lines2_smem(geo.outw), stream>>>(ctx->d_cfg, ctx->d_state, ctx->d_lines,
                                                                                          ctx->d_inp, lo, count, geo);
}

static void launch_lines2(crtx_ctx *ctx, int count, int lo, const LinesGeom &geo, cudaStream_t stream)
{
#define LL(F)                                                                  \
    case F:                                                                    \
        if (geo.blend) launch_lines2_one<1, F>(ctx, count, lo, geo, stream);   \
        else launch_lines2_one<0, F>(ctx, count, lo, geo, stream);             \
        break;
    switch (geo.out_format) {
        LL(CRT_PIX_FORMAT_ARGB) LL(CRT_PIX_FORMAT_RGBA) LL(CRT_PIX_FORMAT_ABGR) LL(CRT_PIX_FORMAT_BGRA)
    }
#undef LL
}

static cudaError_t lines2_attr_all()
{
    cudaError_t e = cudaSuccess;
#define LA(M, T)                                                                                               \
    if (e == cudaSuccess)                                                                                      \
        e = cudaFuncSetAttribute(k_lines2<M, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, lines2_smem(kL2MaxOutw));
#define LF(T) LA(0, T) LA(1, T)
        LF(CRT_PIX_FORMAT_ARGB) LF(CRT_PIX_FORMAT_RGBA) LF(CRT_PIX_FORMAT_ABGR) LF(CRT_PIX_FORMAT_BGRA)
#undef LF
#undef LA
    return e;
}
#else
static bool lines2_eligible(const crtx_ctx *, int, int, const LinesGeom &) { return false; }
static void launch_lines2(crtx_ctx *, int, int, const LinesGeom &, cudaStream_t) {}
static cudaError_t lines2_attr_all() { return cudaSuccess; }
#endif

static void launch_lines(crtx_ctx *ctx, int count, int lo, const LinesGeom &geo, cudaStream_t stream)
{
    if (kBloom) { // CRT_DO_BLOOM build: per-line resampling step, one kernel for every format (crt_bloom.cuh)
        k_lines_bloom<<<dim3(kBloomGroups, count), kBloomWarps * 32, kBloomSmem, stream>>>(
            ctx->d_cfg, ctx->d_lines, ctx->d_inp, static_cast<const BloomLine *>(ctx->d_bloom), lo, geo);
        return;
    }
    if (lines2_eligible(ctx, count, lo, geo)) {
        launch_lines2(ctx, count, lo, geo, stream);
        ctx->lines2_launches += 1;
    } else {
        launch_lines_mode<true>(ctx, count, lo, geo, stream);
    }
    launch_lines_mode<false>(ctx, count, lo, geo, stream); // the monitors k_sync flagged for the wrap-exact equaliser
}

template <bool FAST, int MODE, int FMT>
static cudaError_t lines_attr()
{
    if constexpr (kConv)
        return cudaFuncSetAttribute(k_lines_fir<FAST, MODE, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    fir_smem<FAST>());
    else
        return cudaFuncSetAttribute(k_lines<FAST, MODE, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    lines_smem<FAST>());
}

static cudaError_t lines_attr_all()
{
    cudaError_t e = cudaSuccess;
#define LA(F, M, T)                                  \
    if (e == cudaSuccess) e = lines_attr<F, M, T>();
#define LF(T) LA(true, 0, T) LA(true, 1, T) LA(false, 0, T) LA(false, 1, T)
    LF(CRT_PIX_FORMAT_ARGB) LF(CRT_PIX_FORMAT_RGBA) LF(CRT_PIX_FORMAT_ABGR) LF(CRT_PIX_FORMAT_BGRA)
    LA(true, 2, 0) LA(false, 2, 0)
#undef LF
#undef LA
    return e;
}

#if CRT_B200_BANDLIMITED
template <int FMT, bool COLOR>
static void launch_mod_staged_one(crtx_ctx *ctx, int count, int first, cudaStream_t stream)
{
    k_mod_picture_rgb_staged<FMT, COLOR><<<count, 256, kModSSmem, stream>>>(ctx->d_src + first, ctx->d_cfg, ctx->d_analog, first);
}

// function attributes are per device: set by crtx_create for the context's device
static cudaError_t mod_staged_attr_all()
{
    cudaError_t e = cudaSuccess;
#define MA(F)                                                                                                                        \
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mod_picture_rgb_staged<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kModSSmem);  \
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mod_picture_rgb_staged<F, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kModSSmem);
    MA(0) MA(1) MA(2) MA(3) MA(4) MA(5)
#undef MA
    return e;
}

static void launch_mod_staged(crtx_ctx *ctx, int format, bool color, int count, int first, cudaStream_t stream)
{
#define MS(F)                                                                        \
    case F:                                                                          \
        if (color) launch_mod_staged_one<F, true>(ctx, count, first, stream);        \
        else launch_mod_staged_one<F, false>(ctx, count, first, stream);             \
        break;
    switch (format) { MS(0) MS(1) MS(2) MS(3) MS(4) MS(5) default: break; }
#undef MS
}
#endif

#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
// ---- glibc TYPE_3 rand() replica, host side (glibc 2.39 stdlib/random_r.c: srandom_r, random_r)
typedef std::vector<uint32_t> Mat; // 31 x 31, row major, arithmetic mod 2^32

static Mat mat_mul(const Mat &a, const Mat &b)
{
    Mat c(31 * 31, 0u);
    for (int i = 0; i < 31; i++)
        for (int k = 0; k < 31; k++) {
            const uint32_t aik = a[i * 31 + k];
            if (!aik) continue;
            for (int j = 0; j < 31; j++) c[i * 31 + j] += aik * b[k * 31 + j];
        }
    return c;
}

static Mat mat_pow(Mat base, unsigned e)
{
    Mat r(31 * 31, 0u);
    for (int i = 0; i < 31; i++) r[i * 31 + i] = 1u;
    while (e) {
        if (e & 1u) r = mat_mul(base, r);
        base = mat_mul(base, base);
        e >>= 1;
    }
    return r;
}

static void vhs_build_jump(VhsJump *out)
{
    // one draw on the chronological state (oldest first): new[j] = old[j + 1], new[30] = old[0] + old[28]
    Mat m(31 * 31, 0u);
    for (int j = 0; j < 30; j++) m[j * 31 + j + 1] = 1u;
    m[30 * 31 + 0] = 1u;
    m[30 * 31 + 28] = 1u;
    Mat b = mat_pow(m, 2u * kVhsRun), t = mat_pow(m, (unsigned) kVhsTailRun);
    for (int k = 0; k < kVhsLevels; k++) {
        memcpy(out->bulk[k], b.data(), sizeof(out->bulk[k]));
        memcpy(out->tail[k], t.data(), sizeof(out->tail[k]));
        b = mat_mul(b, b);
        t = mat_mul(t, t);
    }
}

static void vhs_seed_state(unsigned seed, VhsRand *st)
{
    int32_t r[31];
    if (seed == 0) seed = 1;
    int32_t word = (int32_t) seed;
    r[0] = word;
    for (int i = 1; i < 31; i++) {
        const int32_t hi = word / 127773, lo = word % 127773;
        word = 16807 * lo - 2836 * hi;
        if (word < 0) word += 2147483647;
        r[i] = word;
    }
    // fptr = &r[3], rptr = &r[0]: the first draw is r[3] + r[0], so chronologically r[3] is the oldest
    uint32_t h[31];
    for (int j = 0; j < 31; j++) h[j] = (uint32_t) r[(j + 3) % 31];
    for (int k = 0; k < 310; k++) { // srandom_r discards 10 * 31 outputs
        const uint32_t v = h[0] + h[28];
        memmove(h, h + 1, 30 * sizeof(uint32_t));
        h[30] = v;
    }
    memcpy(st->hist, h, sizeof(h));
    st->pad = 0;
}
#endif

// RAII bracket: records start/stop events around one launch when timing is on
struct LaunchTimer {
    crtx_ctx *ctx;
    cudaStream_t stream;
    crtx_ctx::Timed t;
    bool on;
    static cudaEvent_t get(crtx_ctx *ctx)
    {
        cudaEvent_t e = nullptr;
        if (!ctx->event_pool.empty()) {
            e = ctx->event_pool.back();
            ctx->event_pool.pop_back();
        } else {
            cudaEventCreate(&e);
        }
        return e;
    }
    LaunchTimer(crtx_ctx *c, cudaStream_t s, int kernel) : ctx(c), stream(s), on(c->opt_timing != 0)
    {
        if (!on) return;
        t.kernel = kernel;
        t.start = get(ctx);
        t.stop = get(ctx);
        cudaEventRecord(t.start, stream);
    }
    ~LaunchTimer()
    {
        if (!on) return;
        cudaEventRecord(t.stop, stream);
        ctx->timed.push_back(t);
    }
};

int modulate_launch(crtx_ctx *ctx, int first, int count, const SrcCfg *src, cudaStream_t stream)
{
    if (check_range(ctx, first, count)) return 1;
    if (count == 0) return 0;
    if (upload_cfg(ctx, stream)) return 1;
    CUDA_TRY(cudaMemcpyAsync(ctx->d_src + first, src, sizeof(SrcCfg) * count, cudaMemcpyHostToDevice, stream));
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    if (ctx->vhs_draw_aberration) { // batch interface: draw on the device (crt_ntscvhs.c:205-207)
        k_vhs_aberration<<<(count + 63) / 64, 64, 0, stream>>>(ctx->d_src, ctx->d_vhs_wants + first,
                                                               static_cast<VhsRand *>(ctx->d_vhs_rand), first, count);
        ctx->vhs_draw_aberration = 0;
        ctx->launches += 1;
    }
#endif
#if (CRT_SYSTEM == CRT_SYSTEM_NES)
    {
        LaunchTimer lt(ctx, stream, 0);
        k_nes_table<<<count, 256, 0, stream>>>(ctx->d_src + first, ctx->d_cfg, ctx->d_state, ctx->d_nes_tab, first);
        k_mod_nes<<<dim3(kNesParts, count), 256, 0, stream>>>(ctx->d_src + first, ctx->d_nes_tab, ctx->d_analog, first);
    }
    ctx->launches += 2;
#elif (CRT_SYSTEM == CRT_SYSTEM_NESRGB)
    {
        LaunchTimer lt(ctx, stream, 0);
        k_mod_nesrgb<<<dim3(kNesRgbParts, count), 256, 0, stream>>>(ctx->d_src + first, ctx->d_cfg, ctx->d_state,
                                                                  ctx->d_analog, first);
    }
    ctx->launches += 1;
#elif (CRT_SYSTEM == CRT_SYSTEM_SNES)
    {
        LaunchTimer lt(ctx, stream, 0);
        k_mod_snes<<<dim3(kSnesParts, count), 256, 0, stream>>>(ctx->d_src + first, ctx->d_cfg, ctx->d_state, ctx->d_analog,
                                                              first);
    }
    ctx->launches += 1;
#else
    int extra = 0;
    // (the staged kernel steps four samples per carrier period: not for the PV-1000's five, which takes the gather kernel)
    const bool staged = ctx->opt_mod_staged && (kCc == 4 || kCc == 5);
    // The gather kernel only runs for sources the staged one cannot take (their span does not fit a stage row), or for all of
    // them when staging is off: the host can tell (mod_takes is a pure function of the settings), so the usual call saves a launch.
    bool gather = !staged;
    for (int i = 0; i < count; i++) {
        const bool takes = bpp_of(src[i].format) != 0 && staged && mod_takes<true>(src[i]);
        if (bpp_of(src[i].format) != 0 && staged && !takes) gather = true;
        ctx->h_mod_staged[first + i] = takes ? 1 : 0;
    }
    {
        LaunchTimer lt(ctx, stream, 0);
        k_mod_skeleton_rgb<<<count, 256, 0, stream>>>(ctx->d_src + first, ctx->d_state, ctx->d_analog, first);
        extra += 1;
    }
    {
        LaunchTimer lt(ctx, stream, 1);
        if (staged) { // runs of equal (pixel format, colour) share one instantiation
            for (int lo = 0; lo < count;) {
                int hi = lo + 1;
                while (hi < count && src[hi].format == src[lo].format && (src[hi].as_color != 0) == (src[lo].as_color != 0)) hi++;
                if (bpp_of(src[lo].format) != 0) {
                    launch_mod_staged(ctx, src[lo].format, src[lo].as_color != 0, hi - lo, first + lo, stream);
                    extra += 1;
                }
                lo = hi;
            }
        }
        if (gather) {
            k_mod_picture_rgb<<<count, 256, kModSmem, stream>>>(ctx->d_src + first, ctx->d_cfg, ctx->d_analog, first,
                                                                staged ? 1 : 0);
            extra += 1;
        }
    }
    ctx->launches += extra;
#endif
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int demodulate_launch(crtx_ctx *ctx, int first, int count, cudaStream_t stream, const short *d_noise_terms)
{
    if (check_range(ctx, first, count)) return 1;
    if (count == 0) return 0;
    if (upload_cfg(ctx, stream)) return 1;
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    if (d_noise_terms) { // drop-in path: the terms were drawn from the process's libc on the host
        dim3 tgrid((kInputSize + 255) / 256, count);
        LaunchTimer lt(ctx, stream, 2);
        k_noise_terms<<<tgrid, 256, 0, stream>>>(ctx->d_cfg, ctx->d_analog, ctx->d_inp, d_noise_terms, first);
    } else { // batch path: the per-monitor rand() replica (crt_vhs.cuh)
        LaunchTimer lt(ctx, stream, 2);
        // two CTAs per monitor, side by side: (x, 0) the data-dependent tail of the field, (x, 1) its bulk
        k_noise_vhs<<<dim3(count, 2), kVhsThreads, kVhsSmem, stream>>>(ctx->d_cfg, ctx->d_state, static_cast<const VhsRand *>(ctx->d_vhs_rand),
                                                                       static_cast<VhsRand *>(ctx->d_vhs_rand_next),
                                                                       static_cast<const VhsJump *>(ctx->d_vhs_jump),
                                                                       ctx->d_vhs_raw + (size_t) first * kVhsTailRaw, ctx->d_analog,
                                                                       ctx->d_inp, first);
        k_vhs_commit<<<(count * 32 + 255) / 256, 256, 0, stream>>>(static_cast<VhsRand *>(ctx->d_vhs_rand),
                                                                   static_cast<const VhsRand *>(ctx->d_vhs_rand_next), first, count);
    }
    int pre = 2;
#else
    (void) d_noise_terms;
    int pre = 1; // the noise pass runs inside k_sync (crt_sync.cuh)
#endif
    {
        LaunchTimer lt(ctx, stream, 3);
        k_sync<<<count, kSyncThreads, kSyncSmem, stream>>>(ctx->d_cfg, ctx->d_state, ctx->d_lines, ctx->d_analog, ctx->d_inp,
                                                           ctx->d_jump_lo, ctx->d_jump_hi, first, ctx->opt_generic);
    }
    if (kBloom) { // line sums and the beam-energy chain: every line's resampling step and first sample
        LaunchTimer lt(ctx, stream, 3);
        k_bloom<<<count, 256, 0, stream>>>(ctx->d_cfg, ctx->d_lines, ctx->d_inp, static_cast<BloomLine *>(ctx->d_bloom), first);
        pre += 1;
    }
    // The line kernel takes the output geometry as launch-uniform arguments: split the range into
    // runs of monitors that share it (normally one run).
    int launched = 0;
    for (int lo = first; lo < first + count;) {
        const MonCfg &c0 = ctx->h_cfg[lo];
        int hi = lo + 1;
        while (hi < first + count) {
            const MonCfg &c = ctx->h_cfg[hi];
            if (c.outw != c0.outw || c.out_format != c0.out_format || c.blend != c0.blend || c.outh != c0.outh
                || c.v_fac != c0.v_fac)
                break;
            hi++;
        }
        LinesGeom geo;
        geo.outw = c0.outw;
        geo.out_format = c0.out_format;
        geo.bpp = c0.bpp;
        geo.blend = c0.blend ? 1 : 0;
        geo.rnd = 32768;
        geo.dx = c0.outw > 0 ? ((kAvLen - 1) << 12) / c0.outw : 0;
        geo.line_lo = ctx->opt_line_lo;
        geo.line_hi = ctx->opt_line_hi;
        {
            LaunchTimer lt(ctx, stream, 4);
            // the second launch takes the monitors whose signal left the fast equaliser's exact range
            // (flagged by k_sync); it is an empty pass otherwise
            // Fewer output rows than decoded lines: several lines share a row and must be applied in
            // order (crt_core.c:409-664 is a sequential loop).  Without blend only the last line of a run
            // survives; with blend one launch per run position keeps the order.
            const long long rows = (long long) c0.outh + (long long) c0.v_fac;
            if (rows >= kLines) {
                geo.pass = -1;
                launch_lines(ctx, hi - lo, lo, geo, stream);
            } else if (!geo.blend) {
                geo.pass = -2;
                launch_lines(ctx, hi - lo, lo, geo, stream);
            } else {
                const int runs = (int) ((kLines + (rows > 0 ? rows : 1) - 1) / (rows > 0 ? rows : 1)) + 1;
                for (int p = 0; p < runs; p++) {
                    geo.pass = p;
                    launch_lines(ctx, hi - lo, lo, geo, stream);
                    launched += 2;
                }
                launched -= 2;
            }
        }
        launched += 2;
        lo = hi;
    }
    ctx->launches += pre + launched;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// any 16-byte word of a differs from b -> *flag = 1 (crtx_memcmp_device)
__global__ void k_differs(const uint4 *__restrict__ a, const uint4 *__restrict__ b, size_t words, const unsigned char *ta,
                          const unsigned char *tb, int tail, int *flag)
{
    bool diff = false;
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t) gridDim.x * blockDim.x) {
        const uint4 x = a[i], y = b[i];
        diff |= (x.x != y.x) | (x.y != y.y) | (x.z != y.z) | (x.w != y.w);
    }
    if (blockIdx.x == 0 && (int) threadIdx.x < tail) diff |= ta[threadIdx.x] != tb[threadIdx.x];
    if (diff) *flag = 1;
}

// BMP pixel array (bottom-up rows padded to 4 bytes) <-> top-down BGRA (bmp_rw.c:22-146), one thread per pixel
__global__ void k_bmp_unpack(unsigned *__restrict__ bgra, const unsigned char *__restrict__ file, int w, int h, int bytespp,
                             int rowbytes)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const unsigned char *p = file + (size_t) (h - 1 - y) * rowbytes + (size_t) x * bytespp;
    unsigned v;
    if (bytespp == 4) v = *reinterpret_cast<const unsigned *>(p);
    else v = (unsigned) p[0] | (unsigned) p[1] << 8 | (unsigned) p[2] << 16 | 0xff000000u; // bmp_rw.c:90
    bgra[(size_t) y * w + x] = v;
}

__global__ void k_bmp_pack(unsigned *__restrict__ file, const unsigned *__restrict__ bgra, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    file[(size_t) (h - 1 - y) * w + x] = bgra[(size_t) y * w + x];
}

// PPM pixel data (P6: R, G, B bytes, row major) <-> the loaders' int pixels 0x00RRGGBB (ppm_rw.c:79-89, 113-118).
// Four pixels per thread: three 32-bit words of file bytes <-> four int pixels, so both sides move whole words.
__device__ __forceinline__ unsigned ppm_to8(unsigned x, unsigned maxc) { return (x * 255u + maxc / 2u) / maxc; } // ppm_rw.c:80

__global__ void k_ppm_unpack(unsigned *__restrict__ xrgb, const unsigned char *__restrict__ file, size_t npix, unsigned maxc,
                             int aligned)
{
    const size_t q = (size_t) blockIdx.x * blockDim.x + threadIdx.x; // group of 4 pixels
    if (q * 4 >= npix) return;
    unsigned char b[12];
    const size_t left = npix - q * 4;
    if (aligned && left >= 4) {
        const unsigned *w = reinterpret_cast<const unsigned *>(file) + q * 3;
        const unsigned w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            b[k] = (unsigned char) (w0 >> (8 * k));
            b[4 + k] = (unsigned char) (w1 >> (8 * k));
            b[8 + k] = (unsigned char) (w2 >> (8 * k));
        }
    } else {
        for (int k = 0; k < 12; k++) b[k] = ((size_t) k < left * 3) ? file[q * 12 + k] : 0;
    }
    unsigned px[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        unsigned r = b[3 * k], g = b[3 * k + 1], bl = b[3 * k + 2];
        if (maxc != 255u) { r = ppm_to8(r, maxc); g = ppm_to8(g, maxc); bl = ppm_to8(bl, maxc); }
        px[k] = r << 16 | g << 8 | bl;
    }
    if (left >= 4 && (reinterpret_cast<uintptr_t>(xrgb) & 15) == 0) {
        reinterpret_cast<uint4 *>(xrgb)[q] = make_uint4(px[0], px[1], px[2], px[3]);
    } else {
        for (int k = 0; k < 4 && (size_t) k < left; k++) xrgb[q * 4 + k] = px[k];
    }
}

__global__ void k_ppm_pack(unsigned char *__restrict__ file, const unsigned *__restrict__ xrgb, size_t npix, int aligned)
{
    const size_t q = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (q * 4 >= npix) return;
    const size_t left = npix - q * 4;
    unsigned px[4] = { 0u, 0u, 0u, 0u };
    for (int k = 0; k < 4 && (size_t) k < left; k++) px[k] = __ldg(xrgb + q * 4 + k);
    unsigned char b[12];
#pragma unroll
    for (int k = 0; k < 4; k++) { // ppm_rw.c:113-118
        b[3 * k] = (unsigned char) (px[k] >> 16);
        b[3 * k + 1] = (unsigned char) (px[k] >> 8);
        b[3 * k + 2] = (unsigned char) px[k];
    }
    if (aligned && left >= 4) {
        unsigned *w = reinterpret_cast<unsigned *>(file) + q * 3;
        w[0] = (unsigned) b[0] | (unsigned) b[1] << 8 | (unsigned) b[2] << 16 | (unsigned) b[3] << 24;
        w[1] = (unsigned) b[4] | (unsigned) b[5] << 8 | (unsigned) b[6] << 16 | (unsigned) b[7] << 24;
        w[2] = (unsigned) b[8] | (unsigned) b[9] << 8 | (unsigned) b[10] << 16 | (unsigned) b[11] << 24;
    } else {
        for (size_t k = 0; k < left * 3 && k < 12; k++) file[q * 12 + k] = b[k];
    }
}

// the live driver's phosphor decay between frames (crt_main.c:437-452), on int pixels 0x00RRGGBB
__device__ __forceinline__ unsigned fade1(unsigned v)
{
    const unsigned c = v & 0xffffffu;
    return ((c >> 1) & 0x7f7f7fu) + ((c >> 2) & 0x3f3f3fu) + ((c >> 3) & 0x1f1f1fu) + ((c >> 4) & 0x0f0f0fu);
}

__global__ void k_fade_phosphors(unsigned *__restrict__ image, size_t npix)
{
    const size_t stride = (size_t) gridDim.x * blockDim.x;
    const size_t quads = npix / 4;
    if ((reinterpret_cast<uintptr_t>(image) & 15) == 0) {
        uint4 *p = reinterpret_cast<uint4 *>(image);
        for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < quads; i += stride) {
            uint4 v = p[i];
            v.x = fade1(v.x); v.y = fade1(v.y); v.z = fade1(v.z); v.w = fade1(v.w);
            p[i] = v;
        }
        for (size_t i = quads * 4 + (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += stride) image[i] = fade1(image[i]);
    } else {
        for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += stride) image[i] = fade1(image[i]);
    }
}


// ---------------------------------------------------------------------------------------------------------
// crtx_frames_host: only the rows a field touches cross PCIe.
// A field reads 236 of an image's rows (crt_ntsc.c:258-266: row (y * h) / desth + field offset for each picture line
// y) and writes, per decoded line, rows beg .. end - scanlines - 1 (crt_core.c:428-432, 662-664): 384 of 624 with the
// drivers' settings.  The rows are irregularly spaced, so a strided DMA cannot describe them; two copy kernels move
// them through the page-locked host buffers' device mappings instead, 16 bytes per lane, every load of a thread in
// flight before its first store:
//   k_rows_gather   host image -> the monitor's staging slot, picture line y in row y (SrcCfg::compact)
//   k_rows_scatter  device image -> host image, the rows the line table says this field wrote; every other row
//                   of the host image keeps its content, exactly as the reference's own `out` buffer does.
// Pageable, unmapped or unaligned host buffers take the whole-image cudaMemcpyAsync as before.
// ---------------------------------------------------------------------------------------------------------
struct RowGather {
    const unsigned char *src; // device mapping of the page-locked host image, or NULL: not a row job
    unsigned char *dst;       // staging slot
    int row_bytes, h, desth, field;
};

constexpr int kRowWarps = 8;

__device__ __forceinline__ void copy_row16(const uint4 *__restrict__ s, uint4 *__restrict__ d, int n16, int lane)
{
    for (int i = lane; i < n16; i += 32 * 4) {
        uint4 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (i + 32 * k < n16) v[k] = s[i + 32 * k];
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (i + 32 * k < n16) d[i + 32 * k] = v[k];
    }
}

__global__ void __launch_bounds__(kRowWarps * 32) k_rows_gather(const RowGather *__restrict__ jobs, int first)
{
    const RowGather j = jobs[first + blockIdx.y];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int y = blockIdx.x * kRowWarps + warp;
    if (!j.src || y >= j.desth) return;
    int row = (int) (((long long) y * j.h) / j.desth) + (j.field * j.h + j.desth) / j.desth / 2; // crt_ntsc.c:258-266
    if (row >= j.h) row = j.h - 1; // (as the encoder kernels: the reference's one-row over-read is not reproduced)
    copy_row16(reinterpret_cast<const uint4 *>(j.src + (size_t) row * j.row_bytes),
               reinterpret_cast<uint4 *>(j.dst + (size_t) y * j.row_bytes), j.row_bytes / 16, lane);
}

__global__ void __launch_bounds__(kRowWarps * 32)
k_rows_scatter(const MonCfg *__restrict__ cfgs, const LineRec *__restrict__ lines, unsigned char *const *__restrict__ host_out,
               int first, int line_lo, int line_hi)
{
    const int m = first + blockIdx.y;
    unsigned char *host = host_out[m];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k = blockIdx.x * kRowWarps + warp;
    if (!host || k >= kLines || k < line_lo || k >= line_hi) return;
    const LineRec rec = lines[(size_t) m * kLines + k];
    if (rec.beg < 0) return;
    const MonCfg cfg = cfgs[m];
    const int pitch = cfg.outw * cfg.bpp;
    const int nrows = max(1, rec.end - cfg.scanlines - rec.beg); // crt_core.c:662-664
    for (int r = 0; r < nrows; r++) {
        const size_t off = (size_t) (rec.beg + r) * pitch;
        copy_row16(reinterpret_cast<const uint4 *>(cfg.out + off), reinterpret_cast<uint4 *>(host + off), pitch / 16, lane);
    }
}

// device mapping of a page-locked host buffer (NULL if `p` is pageable or not mapped)
static void *host_mapping(const void *p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) return at.devicePointer;
    (void) cudaGetLastError();
    return NULL;
}

void fill_src(SrcCfg *d, const crtx_source *s)
{
    memset(d, 0, sizeof(*d));
    d->data = s->data;
    d->format = s->format;
    d->w = s->w;
    d->h = s->h;
    d->raw = s->raw;
    d->as_color = s->as_color;
    d->field = s->field;
    d->frame = s->frame;
    d->hue = s->hue;
    d->xoffset = s->xoffset;
    d->yoffset = s->yoffset;
    d->aberration = 0;
    d->dot_crawl_offset = s->dot_crawl_offset;
    d->reinit = s->reinit;
#if (CRT_SYSTEM == CRT_SYSTEM_NES)
    d->format = CRT_PIX_FORMAT_RGB; // unused by the NES encoder
#endif
}

} // namespace crt

using namespace crt;

extern "C" {

const char *crtx_last_error(void) { return g_error; }

int crtx_system(void) { return kSystem; }
int crtx_chroma_pattern(void) { return kPattern; }
int crtx_hres(void) { return kHres; }
int crtx_input_size(void) { return kInputSize; }
int crtx_lines(void) { return kLines; }
int crtx_cc_vper(void) { return kVper; }

int crtx_create(crtx_ctx **out, int n)
{
    if (!out || n <= 0) return fail("crtx_create: bad arguments");
    *out = NULL;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
        return fail("crtx_create: device %d is sm_%d%d, this library is built for sm_90a only", dev, prop.major, prop.minor);

    crtx_ctx *ctx = new crtx_ctx();
    ctx->n = n;
    ctx->device = dev;
    ctx->sm_count = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
    ctx->h_cfg.assign(n, MonCfg());
    memset(ctx->h_cfg.data(), 0, sizeof(MonCfg) * n);
    ctx->h_mod_staged.assign(n, 0);
    ctx->cfg_dirty_lo = 0;
    ctx->cfg_dirty_hi = n;
    ctx->tail_dirty_lo = 0;
    ctx->tail_dirty_hi = n;
    ctx->opt_generic = 0;

#define CTX_TRY(expr)                                                                            \
    do {                                                                                         \
        cudaError_t e_ = (expr);                                                                 \
        if (e_ != cudaSuccess) {                                                                 \
            fail("%s: %s", #expr, cudaGetErrorString(e_));                                       \
            crtx_destroy(ctx);                                                                   \
            return 1;                                                                            \
        }                                                                                        \
    } while (0)
    CTX_TRY(cudaMalloc(&ctx->d_cfg, sizeof(MonCfg) * n));
    CTX_TRY(cudaMalloc(&ctx->d_state, sizeof(MonState) * n));
    CTX_TRY(cudaMalloc(&ctx->d_src, sizeof(SrcCfg) * n));
    CTX_TRY(cudaMalloc(&ctx->d_row_jobs, sizeof(RowGather) * n));
    CTX_TRY(cudaMalloc(&ctx->d_host_out, sizeof(unsigned char *) * n));
    CTX_TRY(cudaMalloc(&ctx->d_lines, sizeof(LineRec) * (size_t) n * kLines));
    CTX_TRY(cudaMalloc(&ctx->d_analog, (size_t) n * kSignalBytes));
    CTX_TRY(cudaMalloc(&ctx->d_inp, (size_t) n * kSignalBytes));
    CTX_TRY(cudaMalloc(&ctx->d_jump_lo, sizeof(Affine) * kJumpLo));
    CTX_TRY(cudaMalloc(&ctx->d_jump_hi, sizeof(Affine) * kJumpHi));
    CTX_TRY(cudaMemset(ctx->d_cfg, 0, sizeof(MonCfg) * n));
    CTX_TRY(cudaMemset(ctx->d_lines, 0, sizeof(LineRec) * (size_t) n * kLines));
    CTX_TRY(cudaMemset(ctx->d_analog, 0, (size_t) n * kSignalBytes)); // crt_init memsets the struct
    CTX_TRY(cudaMemset(ctx->d_inp, 0, (size_t) n * kSignalBytes));
    {
        std::vector<MonState> st(n);
        memset(st.data(), 0, sizeof(MonState) * n);
        for (int i = 0; i < n; i++) st[i].rn = 194; // crt_core.c:269
        CTX_TRY(cudaMemcpy(ctx->d_state, st.data(), sizeof(MonState) * n, cudaMemcpyHostToDevice));
        std::vector<Affine> lo(kJumpLo), hi(kJumpHi);
        for (int k = 0; k < kJumpLo; k++) lo[k] = lcg_jump((uint32_t) (kNoiseVec * k));
        for (int k = 0; k < kJumpHi; k++) hi[k] = lcg_jump((uint32_t) (kNoiseVec * kJumpLo * k));
        CTX_TRY(cudaMemcpy(ctx->d_jump_lo, lo.data(), sizeof(Affine) * kJumpLo, cudaMemcpyHostToDevice));
        CTX_TRY(cudaMemcpy(ctx->d_jump_hi, hi.data(), sizeof(Affine) * kJumpHi, cudaMemcpyHostToDevice));
    }
#if (CRT_SYSTEM == CRT_SYSTEM_NES)
    CTX_TRY(cudaMalloc(&ctx->d_nes_tab, (size_t) kNesTabBytes * n));
#endif
    if (kBloom) {
        CTX_TRY(cudaMalloc(&ctx->d_bloom, sizeof(BloomLine) * (size_t) n * kLines));
        CTX_TRY(cudaMemset(ctx->d_bloom, 0, sizeof(BloomLine) * (size_t) n * kLines));
        CTX_TRY(cudaFuncSetAttribute(k_lines_bloom, cudaFuncAttributeMaxDynamicSharedMemorySize, kBloomSmem));
    }
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    {
        CTX_TRY(cudaMalloc(&ctx->d_vhs_rand, sizeof(VhsRand) * n));
        CTX_TRY(cudaMalloc(&ctx->d_vhs_rand_next, sizeof(VhsRand) * n));
        CTX_TRY(cudaMalloc(&ctx->d_vhs_jump, sizeof(VhsJump)));
        CTX_TRY(cudaMalloc(&ctx->d_vhs_raw, sizeof(unsigned) * (size_t) kVhsTailRaw * n));
        CTX_TRY(cudaMalloc(&ctx->d_vhs_wants, sizeof(int) * n));
        std::vector<VhsJump> j(1);
        vhs_build_jump(&j[0]);
        CTX_TRY(cudaMemcpy(ctx->d_vhs_jump, j.data(), sizeof(VhsJump), cudaMemcpyHostToDevice));
        std::vector<VhsRand> r(n);
        for (int i = 0; i < n; i++) vhs_seed_state(1u, &r[i]); // libc's default seed
        CTX_TRY(cudaMemcpy(ctx->d_vhs_rand, r.data(), sizeof(VhsRand) * n, cudaMemcpyHostToDevice));
        CTX_TRY(cudaFuncSetAttribute(k_noise_vhs, cudaFuncAttributeMaxDynamicSharedMemorySize, kVhsSmem));
    }
#endif
    CTX_TRY(lines_attr_all());
    CTX_TRY(lines2_attr_all());
    CTX_TRY(cudaFuncSetAttribute(k_sync, cudaFuncAttributeMaxDynamicSharedMemorySize, kSyncSmem));
#if CRT_B200_BANDLIMITED
    CTX_TRY(cudaFuncSetAttribute(k_mod_picture_rgb, cudaFuncAttributeMaxDynamicSharedMemorySize, kModSmem));
    CTX_TRY(mod_staged_attr_all());
#endif
#undef CTX_TRY
    *out = ctx;
    return 0;
}

void crtx_destroy(crtx_ctx *ctx)
{
    if (!ctx) return;
    cudaFree(ctx->d_cfg);
    cudaFree(ctx->d_state);
    cudaFree(ctx->d_src);
    cudaFree(ctx->d_row_jobs);
    cudaFree(ctx->d_host_out);
    cudaFree(ctx->d_lines);
    cudaFree(ctx->d_analog);
    cudaFree(ctx->d_inp);
    cudaFree(ctx->d_jump_lo);
    cudaFree(ctx->d_jump_hi);
    cudaFree(ctx->d_src_img);
    cudaFree(ctx->d_nes_tab);
    cudaFree(ctx->d_bloom);
    cudaFree(ctx->d_vhs_rand);
    cudaFree(ctx->d_vhs_rand_next);
    cudaFree(ctx->d_vhs_jump);
    cudaFree(ctx->d_vhs_raw);
    cudaFree(ctx->d_vhs_wants);
    for (size_t i = 0; i < ctx->timed.size(); i++) {
        cudaEventDestroy(ctx->timed[i].start);
        cudaEventDestroy(ctx->timed[i].stop);
    }
    for (size_t i = 0; i < ctx->event_pool.size(); i++) cudaEventDestroy(ctx->event_pool[i]);
    if (ctx->cfg_ready) cudaEventDestroy(ctx->cfg_ready);
    delete ctx;
}

int crtx_set_monitors(crtx_ctx *ctx, int first, int count, const crtx_monitor *m)
{
    if (check_range(ctx, first, count)) return 1;
    // validate every entry before any of them is applied: a rejected call leaves the context exactly as it was
    for (int i = 0; i < count; i++) {
        if (m[i].outw < 0 || m[i].outh < 0)
            return fail("monitor %d: negative output size %d x %d", first + i, m[i].outw, m[i].outh);
        if (m[i].outw > kMaxOutw)
            return fail("monitor %d: outw %d above the supported maximum %d", first + i, m[i].outw, kMaxOutw);
        if (bpp_of(m[i].out_format) == 4 && (reinterpret_cast<uintptr_t>(m[i].out) & 3))
            return fail("monitor %d: 4-byte pixel formats need a 4-byte aligned device image", first + i);
    }
    // only what really changed travels to the device (the drop-in calls re-send every knob before every call)
    int lo = ctx->n, hi = 0, tlo = ctx->n, thi = 0;
    for (int i = 0; i < count; i++) {
        MonCfg c;
        memset(&c, 0, sizeof(c));
        c.out = static_cast<unsigned char *>(m[i].out);
        c.outw = m[i].outw;
        c.outh = m[i].outh;
        c.out_format = m[i].out_format;
        c.bpp = bpp_of(m[i].out_format);
        c.hue = m[i].hue;
        c.brightness = m[i].brightness;
        c.contrast = m[i].contrast;
        c.saturation = m[i].saturation;
        c.black_point = m[i].black_point;
        c.white_point = m[i].white_point;
        c.scanlines = m[i].scanlines;
        c.blend = m[i].blend;
        c.v_fac = m[i].v_fac;
        c.noise = m[i].noise;
        MonCfg &old = ctx->h_cfg[first + i];
        if (memcmp(&c, &old, sizeof(MonCfg)) == 0) continue;
        if (c.outw != old.outw || c.outh != old.outh || c.out_format != old.out_format) {
            if (first + i < tlo) tlo = first + i;
            thi = first + i + 1;
        }
        old = c;
        if (first + i < lo) lo = first + i;
        hi = first + i + 1;
    }
    if (lo < ctx->cfg_dirty_lo) ctx->cfg_dirty_lo = lo;
    if (hi > ctx->cfg_dirty_hi) ctx->cfg_dirty_hi = hi;
    if (tlo < ctx->tail_dirty_lo) ctx->tail_dirty_lo = tlo;
    if (thi > ctx->tail_dirty_hi) ctx->tail_dirty_hi = thi;
    return 0;
}

int crtx_set_state(crtx_ctx *ctx, int first, int count, const crtx_state *s, void *stream)
{
    if (check_range(ctx, first, count)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the whole record is rebuilt on the host: its other fields (`field`, `generic`) are outputs of the sync pre-pass that
    // the line kernels of the SAME crtx_demodulate consume, never inputs of a later call -- so no read-back, no
    // synchronisation: one asynchronous copy, ordered on `stream` like everything else
    std::vector<MonState> tmp(count);
    memset(tmp.data(), 0, sizeof(MonState) * count);
    for (int i = 0; i < count; i++) {
        for (int r = 0; r < kVper; r++)
            for (int x = 0; x < kCc; x++) tmp[i].ccf[r][x] = s[i].ccf[r][x];
        tmp[i].hsync = s[i].hsync;
        tmp[i].vsync = s[i].vsync;
        tmp[i].rn = s[i].rn;
    }
    // only the caller's part of each record travels (a strided copy): behind it sit outputs of the sync pre-pass and
    // MonState::track_max, which the device manages across calls.  (pageable source: staged before the call returns, so
    // `tmp` may go out of scope)
    CUDA_TRY(cudaMemcpy2DAsync(ctx->d_state + first, sizeof(MonState), tmp.data(), sizeof(MonState), offsetof(MonState, field),
                               (size_t) count, cudaMemcpyHostToDevice, st));
    return 0;
}

int crtx_get_state(crtx_ctx *ctx, int first, int count, crtx_state *s, void *stream)
{
    if (check_range(ctx, first, count)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::vector<MonState> tmp(count);
    CUDA_TRY(cudaMemcpyAsync(tmp.data(), ctx->d_state + first, sizeof(MonState) * count, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (int i = 0; i < count; i++) {
        memset(s[i].ccf, 0, sizeof(s[i].ccf));
        for (int r = 0; r < kVper; r++)
            for (int x = 0; x < kCc; x++) s[i].ccf[r][x] = tmp[i].ccf[r][x];
        s[i].hsync = tmp[i].hsync;
        s[i].vsync = tmp[i].vsync;
        s[i].rn = tmp[i].rn;
    }
    return 0;
}

int crtx_seed(crtx_ctx *ctx, int first, int count, unsigned seed)
{
    if (check_range(ctx, first, count)) return 1;
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    std::vector<VhsRand> r(count);
    for (int i = 0; i < count; i++) vhs_seed_state(seed, &r[i]); // what srand(seed) leaves in glibc
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(static_cast<VhsRand *>(ctx->d_vhs_rand) + first, r.data(), sizeof(VhsRand) * count,
                        cudaMemcpyHostToDevice));
#else
    (void) seed; // only the VHS variant draws from rand()
#endif
    return 0;
}

signed char *crtx_analog(crtx_ctx *ctx, int i)
{
    if (check_range(ctx, i, 1)) return NULL;
    return ctx->d_analog + (size_t) i * kSignalBytes;
}

signed char *crtx_inp(crtx_ctx *ctx, int i)
{
    if (check_range(ctx, i, 1)) return NULL;
    return ctx->d_inp + (size_t) i * kSignalBytes;
}

int crtx_read_signal(crtx_ctx *ctx, int i, int which, signed char *host, void *stream)
{
    if (check_range(ctx, i, 1)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const signed char *src = (which ? ctx->d_inp : ctx->d_analog) + (size_t) i * kSignalBytes;
    CUDA_TRY(cudaMemcpyAsync(host, src, kInputSize, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

int crtx_write_signal(crtx_ctx *ctx, int i, int which, const signed char *host, void *stream)
{
    if (check_range(ctx, i, 1)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    signed char *dst = (which ? ctx->d_inp : ctx->d_analog) + (size_t) i * kSignalBytes;
    CUDA_TRY(cudaMemcpyAsync(dst, host, kInputSize, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// crtx_modulate; compact[i] != 0: src[i].data is a staging slot that holds only the rows the field reads (crtx_frames_host)
static int modulate_sources(crtx_ctx *ctx, int first, int count, const crtx_source *src, const unsigned char *compact, void *stream)
{
    if (check_range(ctx, first, count)) return 1;
    ctx->scratch_src.resize(count);
    for (int i = 0; i < count; i++) {
        fill_src(&ctx->scratch_src[i], &src[i]);
        ctx->scratch_src[i].compact = (compact && compact[i]) ? 1 : 0;
    }
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    { // the aberration draw happens on the device, from the monitor's rand() replica
        std::vector<int> wants(count);
        for (int i = 0; i < count; i++) wants[i] = src[i].do_aberration ? 1 : 0;
        CUDA_TRY(cudaMemcpyAsync(ctx->d_vhs_wants + first, wants.data(), sizeof(int) * count, cudaMemcpyHostToDevice,
                                 static_cast<cudaStream_t>(stream)));
        ctx->vhs_draw_aberration = 1;
    }
#endif
    return modulate_launch(ctx, first, count, ctx->scratch_src.data(), static_cast<cudaStream_t>(stream));
}

int crtx_modulate(crtx_ctx *ctx, int first, int count, const crtx_source *src, void *stream)
{
    return modulate_sources(ctx, first, count, src, NULL, stream);
}

int crtx_demodulate(crtx_ctx *ctx, int first, int count, void *stream)
{
    return demodulate_launch(ctx, first, count, static_cast<cudaStream_t>(stream), NULL);
}

int crtx_frames_host(crtx_ctx *ctx, int first, int count, const crtx_source *src, void *const *out_host, void *stream)
{
    if (check_range(ctx, first, count)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // device staging for the source images, one slot per monitor
    size_t need = 0;
    for (int i = 0; i < count; i++) {
        size_t b = (size_t) src[i].w * src[i].h * (kIsNes ? 2 : bpp_of(src[i].format));
        b = (b + 255) & ~(size_t) 255;
        if (b > need) need = b;
    }
    if (need > ctx->src_slot) {
        CUDA_TRY(cudaStreamSynchronize(st));
        cudaFree(ctx->d_src_img);
        ctx->d_src_img = NULL;
        ctx->src_slot = 0;
        CUDA_TRY(cudaMalloc(&ctx->d_src_img, need * ctx->n));
        ctx->src_slot = need;
    }
    std::vector<crtx_source> dev(src, src + count);
    std::vector<unsigned char> compact(count, 0);
    std::vector<RowGather> jobs(count);
    int row_jobs = 0, max_desth = 0;
    for (int i = 0; i < count; i++) {
        size_t b = (size_t) src[i].w * src[i].h * (kIsNes ? 2 : bpp_of(src[i].format));
        jobs[i].src = NULL;
        if (ctx->opt_host_src) {
            // "host_src": the encoder reads a page-locked source image in place over PCIe (A/B switch; the encoder's
            // two-deep staging cannot cover the link's latency, the row gather below can).  Pageable images take the copy.
            void *map = host_mapping(src[i].data);
            if (map) {
                dev[i].data = map;
                continue;
            }
        }
        unsigned char *slot = ctx->d_src_img + ctx->src_slot * (size_t) (first + i);
        dev[i].data = slot;
#if CRT_B200_BANDLIMITED
        const int row_bytes = src[i].w * bpp_of(src[i].format);
        void *map = (ctx->opt_host_rows && row_bytes > 0 && (row_bytes & 15) == 0 && src[i].h > 0) ? host_mapping(src[i].data) : NULL;
        if (map && (reinterpret_cast<uintptr_t>(map) & 15) == 0) {
            RowGather &j = jobs[i];
            j.src = static_cast<const unsigned char *>(map);
            j.dst = slot;
            j.row_bytes = row_bytes;
            j.h = src[i].h;
            j.desth = src[i].raw ? (src[i].h < kDestH ? src[i].h : kDestH) : kDestH; // crt_ntsc.c:132-133, 163-172
            j.field = src[i].field & 1;
            compact[i] = 1;
            row_jobs += 1;
            if (j.desth > max_desth) max_desth = j.desth;
            continue;
        }
#endif
        CUDA_TRY(cudaMemcpyAsync(slot, src[i].data, b, cudaMemcpyHostToDevice, st));
    }
    if (row_jobs) {
        CUDA_TRY(cudaMemcpyAsync(static_cast<RowGather *>(ctx->d_row_jobs) + first, jobs.data(), sizeof(RowGather) * count, cudaMemcpyHostToDevice, st));
        k_rows_gather<<<dim3((max_desth + kRowWarps - 1) / kRowWarps, count), kRowWarps * 32, 0, st>>>(
            static_cast<const RowGather *>(ctx->d_row_jobs), first);
        ctx->launches += 1;
    }
    if (modulate_sources(ctx, first, count, dev.data(), compact.data(), stream)) return 1;
    if (crtx_demodulate(ctx, first, count, stream)) return 1;
    std::vector<unsigned char *> maps(count, static_cast<unsigned char *>(NULL));
    int scatter = 0;
    for (int i = 0; i < count; i++) {
        const MonCfg &c = ctx->h_cfg[first + i];
        if (!out_host || !out_host[i]) continue;
        const int pitch = c.outw * c.bpp;
        void *map = (ctx->opt_host_rows && pitch > 0 && (pitch & 15) == 0 && (reinterpret_cast<uintptr_t>(c.out) & 15) == 0
                     && (long long) c.outh + (long long) c.v_fac >= kLines)
                        ? host_mapping(out_host[i]) : NULL;
        if (map && (reinterpret_cast<uintptr_t>(map) & 15) == 0) {
            maps[i] = static_cast<unsigned char *>(map);
            scatter += 1;
            continue;
        }
        CUDA_TRY(cudaMemcpyAsync(out_host[i], c.out, (size_t) c.outw * c.outh * c.bpp, cudaMemcpyDeviceToHost, st));
    }
    if (scatter) {
        CUDA_TRY(cudaMemcpyAsync(ctx->d_host_out + first, maps.data(), sizeof(unsigned char *) * count, cudaMemcpyHostToDevice, st));
        k_rows_scatter<<<dim3((kLines + kRowWarps - 1) / kRowWarps, count), kRowWarps * 32, 0, st>>>(
            ctx->d_cfg, ctx->d_lines, ctx->d_host_out, first, ctx->opt_line_lo, ctx->opt_line_hi);
        ctx->launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_get_lines(crtx_ctx *ctx, int i, crtx_line *table, void *stream)
{
    if (check_range(ctx, i, 1)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaMemcpyAsync(table, ctx->d_lines + (size_t) i * kLines, sizeof(LineRec) * kLines, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

int crtx_get_paths(crtx_ctx *ctx, int first, int count, int *paths, void *stream)
{
    if (check_range(ctx, first, count)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::vector<MonState> tmp(count);
    if (count > 0) {
        CUDA_TRY(cudaMemcpyAsync(tmp.data(), ctx->d_state + first, sizeof(MonState) * count, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    for (int i = 0; i < count; i++)
        paths[i] = (tmp[i].generic ? CRTX_PATH_GENERIC_EQ : 0) | (ctx->h_mod_staged[first + i] ? CRTX_PATH_STAGED_MOD : 0);
    return 0;
}

long crtx_launch_count(crtx_ctx *ctx) { return ctx ? ctx->launches : 0; }
long crtx_lines2_count(crtx_ctx *ctx) { return ctx ? ctx->lines2_launches : 0; }

#if defined(CRTX_PHASE_CLOCKS) && CRTX_PHASE_CLOCKS
// debug builds only (crt_ptx.cuh: phase_mark): the table of phase stamps, 4 x 512 x 16 values
extern "C" int crtx_debug_clocks(unsigned long long *dst)
{
    return (int) cudaMemcpyFromSymbol(dst, crt::g_phase_clk, sizeof(crt::g_phase_clk));
}
#endif

int crtx_get_timing(crtx_ctx *ctx, float *ms, long *launches)
{
    if (!ctx || !ms || !launches) return fail("crtx_get_timing: bad arguments");
    for (int k = 0; k < CRTX_NUM_KERNELS; k++) {
        ms[k] = 0.f;
        launches[k] = 0;
    }
    for (size_t i = 0; i < ctx->timed.size(); i++) {
        crtx_ctx::Timed &t = ctx->timed[i];
        CUDA_TRY(cudaEventSynchronize(t.stop));
        float e = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&e, t.start, t.stop));
        ms[t.kernel] += e;
        launches[t.kernel] += 1;
        ctx->event_pool.push_back(t.start);
        ctx->event_pool.push_back(t.stop);
    }
    ctx->timed.clear();
    return 0;
}

void *crtx_device_alloc(size_t bytes)
{
    void *p = NULL;
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return NULL;
    if (cudaMemset(p, 0, bytes) != cudaSuccess) {
        cudaFree(p);
        return NULL;
    }
    return p;
}

void crtx_device_free(void *p) { if (p) cudaFree(p); }

void *crtx_host_alloc(size_t bytes)
{
    void *p = NULL;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return NULL;
    return p;
}

void crtx_host_free(void *p) { if (p) cudaFreeHost(p); }

int crtx_memcpy(void *dst, const void *src, size_t bytes, int kind, void *stream)
{
    const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (kind < 0 || kind > 2) return fail("crtx_memcpy: kind %d", kind);
    CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, k, (cudaStream_t) stream));
    return 0;
}

int crtx_memcmp_device(const void *a, const void *b, size_t bytes, int *differ, void *stream)
{
    if (!differ) return fail("crtx_memcmp_device: null result");
    if (((uintptr_t) a | (uintptr_t) b) & 15) return fail("crtx_memcmp_device: pointers must be 16-byte aligned");
    int *flag = NULL;
    CUDA_TRY(cudaMalloc(&flag, sizeof(int)));
    cudaMemsetAsync(flag, 0, sizeof(int), (cudaStream_t) stream);
    const size_t words = bytes / 16;
    k_differs<<<264, 256, 0, (cudaStream_t) stream>>>((const uint4 *) a, (const uint4 *) b, words,
                                                     (const unsigned char *) a + words * 16,
                                                     (const unsigned char *) b + words * 16, (int) (bytes - words * 16), flag);
    cudaError_t e = cudaMemcpyAsync(differ, flag, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t) stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t) stream);
    cudaFree(flag);
    CUDA_TRY(e);
    return 0;
}

int crtx_bmp_unpack(void *bgra, const void *file_pixels, int w, int h, int bits, void *stream)
{
    if (!bgra || !file_pixels || w <= 0 || h <= 0 || h > 65535) return fail("crtx_bmp_unpack: bad arguments");
    if (bits != 24 && bits != 32) return fail("crtx_bmp_unpack: %d bits per pixel (24 or 32)", bits);
    const int bytespp = bits / 8, rowbytes = (w * bytespp + 3) & ~3;
    if (bytespp == 4 && (reinterpret_cast<uintptr_t>(file_pixels) & 3)) return fail("crtx_bmp_unpack: unaligned 32-bit pixel array");
    const dim3 grid((w + 255) / 256, h);
    k_bmp_unpack<<<grid, 256, 0, (cudaStream_t) stream>>>((unsigned *) bgra, (const unsigned char *) file_pixels, w, h, bytespp, rowbytes);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_bmp_pack(void *file_pixels, const void *bgra, int w, int h, void *stream)
{
    if (!bgra || !file_pixels || w <= 0 || h <= 0 || h > 65535) return fail("crtx_bmp_pack: bad arguments");
    const dim3 grid((w + 255) / 256, h);
    k_bmp_pack<<<grid, 256, 0, (cudaStream_t) stream>>>((unsigned *) file_pixels, (const unsigned *) bgra, w, h);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_ppm_unpack(void *xrgb, const void *file_pixels, int w, int h, int maxc, void *stream)
{
    if (!xrgb || !file_pixels || w <= 0 || h <= 0) return fail("crtx_ppm_unpack: bad arguments");
    if (maxc < 1 || maxc > 255) return fail("crtx_ppm_unpack: maximum colour value %d (1..255, ppm_rw.c:57-62)", maxc);
    if (reinterpret_cast<uintptr_t>(xrgb) & 3) return fail("crtx_ppm_unpack: unaligned pixel array");
    const size_t npix = (size_t) w * h, groups = (npix + 3) / 4;
    k_ppm_unpack<<<(unsigned) ((groups + 255) / 256), 256, 0, (cudaStream_t) stream>>>(
        (unsigned *) xrgb, (const unsigned char *) file_pixels, npix, (unsigned) maxc,
        (reinterpret_cast<uintptr_t>(file_pixels) & 3) == 0 ? 1 : 0);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_ppm_pack(void *file_pixels, const void *xrgb, int w, int h, void *stream)
{
    if (!xrgb || !file_pixels || w <= 0 || h <= 0) return fail("crtx_ppm_pack: bad arguments");
    if (reinterpret_cast<uintptr_t>(xrgb) & 3) return fail("crtx_ppm_pack: unaligned pixel array");
    const size_t npix = (size_t) w * h, groups = (npix + 3) / 4;
    k_ppm_pack<<<(unsigned) ((groups + 255) / 256), 256, 0, (cudaStream_t) stream>>>(
        (unsigned char *) file_pixels, (const unsigned *) xrgb, npix, (reinterpret_cast<uintptr_t>(file_pixels) & 3) == 0 ? 1 : 0);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_fade_phosphors(void *image, size_t npix, void *stream)
{
    if (!image) return fail("crtx_fade_phosphors: bad arguments");
    if (reinterpret_cast<uintptr_t>(image) & 3) return fail("crtx_fade_phosphors: unaligned pixel array");
    if (npix == 0) return 0;
    size_t blocks = (npix / 4 + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 132 * 8) blocks = 132 * 8; // a few resident CTAs per SM of an H100, grid-stride beyond
    k_fade_phosphors<<<(unsigned) blocks, 256, 0, (cudaStream_t) stream>>>((unsigned *) image, npix);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int crtx_sync(void *stream)
{
    CUDA_TRY(cudaStreamSynchronize((cudaStream_t) stream));
    return 0;
}

int crtx_set_option(crtx_ctx *ctx, const char *name, int value)
{
    if (!ctx || !name) return fail("crtx_set_option: bad arguments");
    if (!strcmp(name, "generic_eq")) ctx->opt_generic = value;
    else if (!strcmp(name, "timing")) ctx->opt_timing = value;
    else if (!strcmp(name, "mod_staged")) ctx->opt_mod_staged = value;
    else if (!strcmp(name, "host_src")) ctx->opt_host_src = value;
    else if (!strcmp(name, "host_rows")) ctx->opt_host_rows = value;
    else if (!strcmp(name, "lines2")) ctx->opt_lines2 = value;
    else if (!strcmp(name, "line_lo")) ctx->opt_line_lo = value;
    else if (!strcmp(name, "line_hi")) ctx->opt_line_hi = value;
    else return fail("crtx_set_option: unknown option '%s'", name);
    return 0;
}

} // extern "C"
