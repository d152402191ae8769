// crt_dropin.cu -- the reference's seven entry points (crt_core.h:100-139) on top of the device
// pipeline, so crt_main.c / extra/video_convert.c link against this library unchanged.
//
// Semantics kept from the reference: all calls are synchronous; on return analog / inp / out /
// ccf / hsync / vsync / rn in the caller's struct are final; every knob is re-read on every call;
// unknown pixel formats make modulate / demodulate silent no-ops (crt_core.c:312-315,
// crt_ntsc.c:190-193).  Because callers may edit struct CRT, its analog[] and the output image
// between calls (crt_main.c:263, 430, 437-452) the host copies are authoritative: in the default
// strict mode they are uploaded before each call and downloaded after it.  CRT_B200_STRICT=0
// trusts that nobody touched analog[] / out between calls and skips those uploads.
//
// There is no CPU implementation here: if CUDA is unusable the library says so and aborts.
#include <cuda_runtime.h>

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>
#include <vector>

#include "crt_b200.h"
#include "crtx_internal.h"

namespace {

using namespace crt;

struct Shadow {
    crtx_ctx *ctx = nullptr;
    cudaStream_t stream = nullptr;
    unsigned char *d_out = nullptr;
    size_t out_bytes = 0;
    unsigned char *d_img = nullptr;
    size_t img_bytes = 0;
    short *d_terms = nullptr; // VHS noise terms
    bool out_valid = false;   // device image mirrors the host image (non-strict mode)
    const unsigned char *out_host = nullptr;
};

std::mutex g_mutex;
std::unordered_map<const void *, Shadow *> g_shadows;

[[noreturn]] void die(const char *what)
{
    fprintf(stderr, "crt_b200: %s: %s\ncrt_b200: this library has no CPU path; aborting.\n", what, crtx_last_error());
    abort();
}

void cuda_or_die(cudaError_t e, const char *what)
{
    if (e != cudaSuccess) {
        fprintf(stderr, "crt_b200: %s: %s\ncrt_b200: this library has no CPU path; aborting.\n", what,
                cudaGetErrorString(e));
        abort();
    }
}

bool strict_mode()
{
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("CRT_B200_STRICT");
        v = (e && *e == '0') ? 0 : 1;
    }
    return v != 0;
}

void drop_shadow(Shadow *sh)
{
    if (!sh) return;
    if (sh->stream) cudaStreamSynchronize(sh->stream);
    cudaFree(sh->d_out);
    cudaFree(sh->d_img);
    cudaFree(sh->d_terms);
    crtx_destroy(sh->ctx);
    if (sh->stream) cudaStreamDestroy(sh->stream);
    delete sh;
}

Shadow *new_shadow()
{
    Shadow *sh = new Shadow();
    if (crtx_create(&sh->ctx, 1)) die("crtx_create");
    cuda_or_die(cudaStreamCreateWithFlags(&sh->stream, cudaStreamNonBlocking), "cudaStreamCreate");
    return sh;
}

// look the shadow of `v` up; `fresh` (crt_init) replaces it by a zeroed one
Shadow *shadow_of(const struct CRT *v, bool fresh)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    auto it = g_shadows.find(v);
    if (it != g_shadows.end()) {
        if (!fresh) return it->second;
        drop_shadow(it->second);
        g_shadows.erase(it);
    }
    Shadow *sh = new_shadow();
    g_shadows[v] = sh;
    return sh;
}

void ensure(unsigned char **buf, size_t *have, size_t need, cudaStream_t st)
{
    if (need <= *have) return;
    cuda_or_die(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    cudaFree(*buf);
    *buf = nullptr;
    *have = 0;
    need = (need + 4095) & ~(size_t) 4095;
    cuda_or_die(cudaMalloc(buf, need), "cudaMalloc");
    cuda_or_die(cudaMemsetAsync(*buf, 0, need, st), "cudaMemset");
    *have = need;
}

void push_state(Shadow *sh, const struct CRT *v)
{
    crtx_state s;
    memset(&s, 0, sizeof(s));
    for (int n = 0; n < CRT_CC_VPER; n++)
        for (int x = 0; x < CRT_CC_SAMPLES; x++) s.ccf[n][x] = v->ccf[n][x];
    s.hsync = v->hsync;
    s.vsync = v->vsync;
    s.rn = v->rn;
    if (crtx_set_state(sh->ctx, 0, 1, &s, sh->stream)) die("crtx_set_state");
}

void pull_state(Shadow *sh, struct CRT *v)
{
    crtx_state s;
    if (crtx_get_state(sh->ctx, 0, 1, &s, sh->stream)) die("crtx_get_state");
    for (int n = 0; n < CRT_CC_VPER; n++)
        for (int x = 0; x < CRT_CC_SAMPLES; x++) v->ccf[n][x] = s.ccf[n][x];
    v->hsync = s.hsync;
    v->vsync = s.vsync;
    v->rn = s.rn;
}

void push_monitor(Shadow *sh, const struct CRT *v, int noise)
{
    crtx_monitor m;
    memset(&m, 0, sizeof(m));
    const int bpp = bpp_of(v->out_format);
    size_t need = (bpp && v->outw > 0 && v->outh > 0) ? (size_t) v->outw * v->outh * bpp : 0;
    if (need > sh->out_bytes || v->out != sh->out_host) sh->out_valid = false;
    ensure(&sh->d_out, &sh->out_bytes, need ? need : 4, sh->stream);
    sh->out_host = v->out;
    m.out = sh->d_out;
    m.outw = v->outw;
    m.outh = v->outh;
    m.out_format = v->out_format;
    m.hue = v->hue;
    m.brightness = v->brightness;
    m.contrast = v->contrast;
    m.saturation = v->saturation;
    m.black_point = v->black_point;
    m.white_point = v->white_point;
    m.scanlines = v->scanlines;
    m.blend = v->blend;
    m.v_fac = v->v_fac;
    m.noise = noise;
    if (crtx_set_monitors(sh->ctx, 0, 1, &m)) die("crtx_set_monitors");
}

} // namespace

extern "C" {

void crt_sincos14(int *s, int *c, int n) { crt::sincos14_host(s, c, n); } /* crt_core.c:42-61 */

int crt_bpp4fmt(int format) { return crt::bpp_of(format); } /* crt_core.c:63-78 */

void crt_resize(struct CRT *v, int w, int h, int f, unsigned char *out) /* crt_core.c:241-248 */
{
    v->outw = w;
    v->outh = h;
    v->out_format = f;
    v->out = out;
}

void crt_reset(struct CRT *v) /* crt_core.c:250-261 */
{
    v->hue = 0;
    v->saturation = 10;
    v->brightness = 0;
    v->contrast = 180;
    v->black_point = 0;
    v->white_point = 100;
    v->hsync = 0;
    v->vsync = 0;
}

void crt_init(struct CRT *v, int w, int h, int f, unsigned char *out) /* crt_core.c:263-289 */
{
    memset(v, 0, sizeof(struct CRT));
    crt_resize(v, w, h, f, out);
    crt_reset(v);
    v->rn = 194;
    (void) shadow_of(v, true); // zeroed device signal buffers, default state
}

void crt_modulate(struct CRT *v, struct NTSC_SETTINGS *s)
{
    Shadow *sh = shadow_of(v, false);
    SrcCfg src;
    memset(&src, 0, sizeof(src));
#if (CRT_SYSTEM == CRT_SYSTEM_NES)
    src.reinit = !s->field_initialized; /* crt_nes.c:118-121 */
    s->field_initialized = 1;
    src.format = CRT_PIX_FORMAT_RGB;
    src.w = s->w;
    src.h = s->h;
    src.hue = s->hue;
    src.xoffset = s->xoffset;
    src.yoffset = s->yoffset;
    src.dot_crawl_offset = s->dot_crawl_offset;
#if NES_BORDER
    src.border_color = s->border_color; /* crt_nes.c:138-161 */
#endif
    const size_t img_bytes = (size_t) s->w * s->h * sizeof(unsigned short);
#elif (CRT_SYSTEM == CRT_SYSTEM_NESRGB)
    src.reinit = !s->field_initialized; /* crt_nesrgb.c:63-66: setup_field runs before the format check */
    s->field_initialized = 1;
    const int bpp = bpp_of(s->format);
    if (bpp == 0 && !src.reinit) return; /* crt_nesrgb.c:81-84 */
    src.format = s->format;
    src.w = s->w;
    src.h = s->h;
    src.hue = s->hue;
    src.xoffset = s->xoffset;
    src.yoffset = s->yoffset;
    src.dot_crawl_offset = s->dot_crawl_offset;
    const size_t img_bytes = (size_t) s->w * s->h * bpp;
#else
    s->iirs_initialized = 1; /* crt_ntsc.c:142-147 */
    const int bpp = bpp_of(s->format);
    if (bpp == 0) return; /* crt_ntsc.c:190-193 */
    s->field &= 1;        /* crt_ntsc.c:197-198 */
    s->frame &= 1;
    src.format = s->format;
    src.w = s->w;
    src.h = s->h;
    src.raw = s->raw;
    src.as_color = s->as_color;
    src.field = s->field;
    src.frame = s->frame;
    src.hue = s->hue;
    src.xoffset = s->xoffset;
    src.yoffset = s->yoffset;
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    if (s->do_aberration) src.aberration = ((rand() % 12) - 8) + 14; /* crt_ntscvhs.c:205-207 */
#endif
#if (CRT_SYSTEM == CRT_SYSTEM_SNES) || (CRT_SYSTEM == CRT_SYSTEM_TEMP) || (CRT_SYSTEM == CRT_SYSTEM_PV1K)
    src.dot_crawl_offset = s->dot_crawl_offset; /* crt_snes.c:172, crt_template.c:168, crt_pv1k.c:168 */
#endif
    const size_t img_bytes = (size_t) s->w * s->h * bpp;
#endif
    src.pitch = (int) src_row_bytes(src.format, src.w); // the reference's images are dense
    ensure(&sh->d_img, &sh->img_bytes, img_bytes ? img_bytes : 4, sh->stream);
    cuda_or_die(cudaMemcpyAsync(sh->d_img, s->data, img_bytes, cudaMemcpyHostToDevice, sh->stream), "image upload");
    src.data = sh->d_img;

    push_monitor(sh, v, 0); // black_point / white_point feed the encoder
    push_state(sh, v);
    signed char *d_analog = crtx_analog(sh->ctx, 0);
    if (strict_mode())
        cuda_or_die(cudaMemcpyAsync(d_analog, v->analog, CRT_INPUT_SIZE, cudaMemcpyHostToDevice, sh->stream),
                    "analog upload");
    if (modulate_launch(sh->ctx, 0, 1, &src, sh->stream)) die("crt_modulate");
    cuda_or_die(cudaMemcpyAsync(v->analog, d_analog, CRT_INPUT_SIZE, cudaMemcpyDeviceToHost, sh->stream),
                "analog download");
    pull_state(sh, v); // synchronises the stream
}

void crt_demodulate(struct CRT *v, int noise)
{
    const int bpp = bpp_of(v->out_format);
    if (bpp == 0) return; /* crt_core.c:312-315 */
    Shadow *sh = shadow_of(v, false);
    push_monitor(sh, v, noise);
    push_state(sh, v);
    const size_t out_bytes = (size_t) v->outw * v->outh * bpp;
    signed char *d_analog = crtx_analog(sh->ctx, 0);
    if (strict_mode() || !sh->out_valid) {
        cuda_or_die(cudaMemcpyAsync(sh->d_out, v->out, out_bytes, cudaMemcpyHostToDevice, sh->stream), "image upload");
        cuda_or_die(cudaMemcpyAsync(d_analog, v->analog, CRT_INPUT_SIZE, cudaMemcpyHostToDevice, sh->stream),
                    "analog upload");
    }
    const short *d_terms = nullptr;
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    /* The VHS noise pass draws from the process's libc rand() (crt_core.c:343-357); to stay a
     * drop-in (same stream, same global PRNG state afterwards) the draws happen here on the host
     * in the reference's order, and only the add-and-clamp runs on the device. */
    int last_rn = v->rn;
    {
        static std::vector<short> terms;
        terms.resize(CRT_INPUT_SIZE);
        const int wobble = ((rand() % 8) - 4) + 14;
        for (int i = 0; i < CRT_INPUT_SIZE; i++) {
            int nn = noise;
            int rn = rand();
            if (i > (CRT_INPUT_SIZE - CRT_HRES * (16 + ((rand() % 20) - 10)))
                && i < (CRT_INPUT_SIZE - CRT_HRES * (5 + ((rand() % 8) - 4)))) {
                int sn, cs;
                int ln = (i * wobble) / CRT_HRES;
                crt::sincos14_host(&sn, &cs, ln * 8192 / 180);
                nn = cs >> 8;
            }
            int t = (int) ((unsigned) ((((rn >> 16) & 0xff) - 0x7f)) * (unsigned) nn) >> 8;
            /* analog is within [-128, 127]: beyond +-255 the sum saturates regardless */
            terms[i] = (short) (t > 255 ? 255 : (t < -255 ? -255 : t));
            last_rn = rn;
        }
        if (!sh->d_terms) cuda_or_die(cudaMalloc(&sh->d_terms, sizeof(short) * CRT_INPUT_SIZE), "cudaMalloc");
        cuda_or_die(cudaMemcpyAsync(sh->d_terms, terms.data(), sizeof(short) * CRT_INPUT_SIZE, cudaMemcpyHostToDevice,
                                    sh->stream), "noise upload");
        cuda_or_die(cudaStreamSynchronize(sh->stream), "sync"); /* terms is reused by the next call */
        d_terms = sh->d_terms;
    }
#endif
    if (demodulate_launch(sh->ctx, 0, 1, sh->stream, d_terms)) die("crt_demodulate");
    cuda_or_die(cudaMemcpyAsync(v->inp, crtx_inp(sh->ctx, 0), CRT_INPUT_SIZE, cudaMemcpyDeviceToHost, sh->stream),
                "inp download");
    cuda_or_die(cudaMemcpyAsync(v->out, sh->d_out, out_bytes, cudaMemcpyDeviceToHost, sh->stream), "image download");
    pull_state(sh, v); // synchronises the stream
    sh->out_valid = true;
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    v->rn = last_rn; /* crt_core.c:367 */
#endif
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) cuda_or_die(e, "kernel");
}

} // extern "C"
