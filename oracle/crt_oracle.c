/* oracle/crt_oracle.c -- TEST INFRASTRUCTURE ONLY (the parity checker).
 *
 * CPU restatement of the reference hot path; see crt_oracle.h for the rules about
 * who may use it.  Every routine cites the reference lines it restates.  All
 * arithmetic is 32-bit two's complement with arithmetic right shift and C's
 * truncating '/' and '%' (build with -fwrapv; SURVEY.md section 5).
 *
 * Pinned by tests/test_oracle_vs_ref.py against oracle/_ref/libref_*.so (the
 * unmodified reference compiled here) -- the reference has no tests of its own.
 */
#include "crt_oracle.h"

#include <stdlib.h>
#include <string.h>

typedef int i32;
typedef unsigned u32;

static i32 wmul(i32 a, i32 b) { return (i32) ((u32) a * (u32) b); }
static i32 wadd(i32 a, i32 b) { return (i32) ((u32) a + (u32) b); }
static i32 wsub(i32 a, i32 b) { return (i32) ((u32) a - (u32) b); }
static i32 posmod(i32 x, i32 n) { return ((x % n) + n) % n; } /* crt_core.c:17 */

/* WHITE_LEVEL * white_point / 100, the white scale of the RGB encoders (crt_ntsc.c:318 and the same line of every
 * other RGB encoder).  Signed overflow being undefined, gcc -O3 folds it to white_point where WHITE_LEVEL is 100 --
 * every system that computes it -- so the compiled reference does not wrap 100 * white_point there. */
static i32
white_scale(const ocrt_sys *sys, i32 white_point)
{
    return sys->white_level == 100 ? white_point : wmul(sys->white_level, white_point) / 100;
}

/* ------------------------------------------------------------------------- */
/* fixed-point trigonometry (crt_core.c:19-61)                               */
/* ------------------------------------------------------------------------- */

/* 16 steps of a quarter sine at 15 bits, plus the mirrored 17th for the lerp */
static const i32 quarter15[18] = {
    0x0000, 0x0c88, 0x18f8, 0x2528, 0x30f8, 0x3c50, 0x4718, 0x5130, 0x5a80,
    0x62f0, 0x6a68, 0x70e0, 0x7640, 0x7a78, 0x7d88, 0x7f60, 0x8000, 0x7f60
};

static i32
quarter_lerp(i32 a) /* crt_core.c:26-39 */
{
    i32 k = (a >> 8) & 0xff, fr = a & 0xff;
    i32 lo = quarter15[k], hi = quarter15[k + 1];
    return lo + (((hi - lo) * fr) >> 8);
}

void
ocrt_sincos14(int *s, int *c, int n) /* crt_core.c:42-61 */
{
    i32 half;
    n &= 16383;
    half = n & 8191;
    if (half >= 4096) {
        *c = -quarter_lerp(half - 4096);
        *s = quarter_lerp(8192 - half);
    } else {
        *c = quarter_lerp(4096 - half);
        *s = quarter_lerp(half);
    }
    if (n >= 8192) {
        *c = -*c;
        *s = -*s;
    }
}

static i32 sin14(i32 n) { int s, c; ocrt_sincos14(&s, &c, n); return s; }
static i32 cos14(i32 n) { int s, c; ocrt_sincos14(&s, &c, n); return c; }

int
ocrt_bpp(int format) /* crt_core.c:63-78 */
{
    if (format == 0 || format == 1) return 3;
    if (format >= 2 && format <= 5) return 4;
    return 0;
}

/* byte offsets of R, G, B inside a pixel of each CRT_PIX_FORMAT (crt_core.h:62-67),
 * and of the alpha byte (-1 = none) */
static const int fmt_r[6] = { 0, 2, 1, 0, 3, 2 };
static const int fmt_g[6] = { 1, 1, 2, 1, 2, 1 };
static const int fmt_b[6] = { 2, 0, 3, 2, 1, 0 };
static const int fmt_a[6] = { -1, -1, 0, 3, 0, 3 };

/* ------------------------------------------------------------------------- */
/* glibc TYPE_3 rand() (glibc 2.39 stdlib/random_r.c: srandom_r, random_r)    */
/* ------------------------------------------------------------------------- */

int
ocrt_rand_next(ocrt_rand *g)
{
    u32 v = (g->r[g->f] += g->r[g->b]);
    if (++g->f == 31) g->f = 0;
    if (++g->b == 31) g->b = 0;
    return (int) (v >> 1);
}

void
ocrt_rand_seed(ocrt_rand *g, unsigned seed)
{
    i32 word, k;
    if (seed == 0) seed = 1;
    word = (i32) seed;
    g->r[0] = (u32) word;
    for (k = 1; k < 31; k++) {
        i32 hi = word / 127773, lo = word % 127773;
        word = 16807 * lo - 2836 * hi;
        if (word < 0) word += 2147483647;
        g->r[k] = (u32) word;
    }
    g->f = 3;
    g->b = 0;
    for (k = 0; k < 310; k++) (void) ocrt_rand_next(g);
}

/* ------------------------------------------------------------------------- */
/* system descriptors                                                         */
/* ------------------------------------------------------------------------- */

/* Q11 e^x (crt_ntsc.c:25-83) */
static i32
exp_q11(i32 n)
{
    static const i32 epow[5] = { 2048, 5567, 15133, 41135, 111817 };
    i32 neg = n < 0, whole, res = 2048, term = 2048, sum = 0, fact = 1, k;
    if (n == 0) return 2048;
    if (neg) n = -n;
    whole = n >> 11;
    for (k = 0; k < whole / 4; k++) res = wmul(res, epow[4]) >> 11;
    if (whole & 3) res = wmul(res, epow[whole & 3]) >> 11;
    n &= 2047;
    for (k = 1; k < 17; k++) {
        sum += term / fact;
        term = wmul(term, n) >> 11;
        fact = wmul(fact, k);
        if (fact > term || term <= 0 || fact <= 0) break;
    }
    res = wmul(res, sum) >> 11;
    if (neg) res = (2048 << 11) / res;
    return res;
}

static i32
bandlimit_coeff(i32 limit) /* init_iir, crt_ntsc.c:98-106 */
{
    i32 rate = (1431818 << 9) / limit;
    return 2048 - exp_q11(-((6434 << 9) / rate));
}

static void
eq_coeffs(int *dst, i32 hres, i32 khz_lo, i32 khz_hi, i32 g0, i32 g1, i32 g2)
{
    /* kHz2L (crt_core.c:272) then init_eq (crt_core.c:171-196), EQ_P = 16 */
    i32 lo = hres * (khz_lo * 100) / 1431818;
    i32 hi = hres * (khz_hi * 100) / 1431818;
    dst[0] = 2 * (sin14(8192 * lo / hres) << 1);
    dst[1] = 2 * (sin14(8192 * hi / hres) << 1);
    dst[2] = g0;
    dst[3] = g1;
    dst[4] = g2;
}

static void
finish_sys(ocrt_sys *s)
{
    s->input_size = s->hres * s->vres;
    s->lines = s->bot - s->top;
    if (!s->cc_samples) s->cc_samples = 4;
    s->burst_len = 10 * s->cc_samples; /* CB_CYCLES * CRT_CB_FREQ (CB_FREQ == CC_SAMPLES in every system) */
    if (s->cc_samples == 5) eq_coeffs(s->eq[0], s->hres, 1500, 3000, 65536, 12192, 7775); /* crt_core.c:282 */
    else eq_coeffs(s->eq[0], s->hres, 1500, 3000, 65536, 8192, 9175);                    /* crt_core.c:278 */
    eq_coeffs(s->eq[1], s->hres, 80, 1150, 65536, 65536, 1311);   /* crt_core.c:279 */
    eq_coeffs(s->eq[2], s->hres, 80, 1000, 65536, 65536, 0);      /* crt_core.c:280 */
}

static void
make_rgb_sys(ocrt_sys *s, int system)
{
    /* crt_ntsc.h:25-109 (CRT_CHROMA_PATTERN 1) / crt_ntscvhs.h:25-131 */
    const i32 line_ns = 1500 + 4700 + 600 + 2500 + 1600 + 52600;
    memset(s, 0, sizeof(*s));
    s->system = system;
    s->chroma_pattern = 1;
    s->hres = 2275 * 4 / 10;
    s->vres = 262;
    s->top = 21;
    s->bot = 261;
    s->cc_vper = 1;
    s->hsync_window = 8;
    s->vsync_window = 8;
    s->hsync_thresh = 4;
    s->vsync_thresh = 94;
    s->sync_beg = 1500 * s->hres / line_ns;
    s->bw_beg = (1500 + 4700) * s->hres / line_ns;
    s->cb_beg = (1500 + 4700 + 600) * s->hres / line_ns;
    s->av_beg = (1500 + 4700 + 600 + 2500 + 1600) * s->hres / line_ns;
    s->av_len = 52600 * s->hres / line_ns;
    s->white_level = 100;
    s->burst_level = 20;
    s->black_level = 7;
    s->blank_level = 0;
    s->sync_level = -40;
    if (system == OCRT_SYS_VHS) {
        s->vhs_noise = 1;
        s->iir_c[0] = bandlimit_coeff(300000); /* crt_ntscvhs.h:110-113, VHS_SP */
        s->iir_c[1] = bandlimit_coeff(62700);
        s->iir_c[2] = bandlimit_coeff(62700);
    } else {
        s->iir_c[0] = bandlimit_coeff(420000); /* crt_ntsc.h:99-101 */
        s->iir_c[1] = bandlimit_coeff(150000);
        s->iir_c[2] = bandlimit_coeff(55000);
    }
    finish_sys(s);
}

static void
make_nes_sys(ocrt_sys *s, int pattern)
{
    /* crt_nes.h:30-130 */
    static const i32 cc_line[3] = { 2280, 2275, 2273 };
    const i32 line_px = 9 + 25 + 4 + 15 + 5 + 1 + 15 + 256 + 11;
    memset(s, 0, sizeof(*s));
    s->system = OCRT_SYS_NES;
    s->chroma_pattern = pattern;
    s->hres = cc_line[pattern] * 4 / 10;
    s->vres = 262;
    s->top = 15;
    s->bot = 255;
    s->cc_vper = 3;
    s->hsync_window = 6;
    s->vsync_window = 6;
    s->hsync_thresh = 4;
    s->vsync_thresh = 94;
    s->sync_beg = 9 * s->hres / line_px;
    s->bw_beg = (9 + 25) * s->hres / line_px;
    s->cb_beg = (9 + 25 + 4) * s->hres / line_px;
    s->av_beg = (9 + 25 + 4 + 15 + 5 + 1 + 15) * s->hres / line_px;
    s->av_len = 256 * s->hres / line_px;
    s->nes_vsync_end = 327 * s->hres / line_px;
    s->white_level = 110;
    s->burst_level = 30;
    s->black_level = 0;
    s->blank_level = 0;
    s->sync_level = -37;
    finish_sys(s);
}

static void
make_snes_sys(ocrt_sys *s)
{
    /* crt_snes.h:20-109: the NES line layout at 227.3 cycles per line, composite NTSC levels */
    make_nes_sys(s, 2);
    s->system = OCRT_SYS_SNES;
    s->nes_vsync_end = 0;
    s->white_level = 100;
    s->burst_level = 20;
    s->black_level = 7;
    s->blank_level = 0;
    s->sync_level = -40;
}

static void
make_template_sys(ocrt_sys *s)
{
    /* crt_template.h: the composite NTSC timing and band-limit of crt_ntsc.h with CRT_CC_VPER 2 */
    make_rgb_sys(s, OCRT_SYS_NTSC);
    s->system = OCRT_SYS_TEMP;
    s->chroma_pattern = 1;
    s->cc_vper = 2;
}

static void
make_pv1k_sys(ocrt_sys *s)
{
    /* crt_pv1k.h: 5 samples per chroma period, 1920 samples per line, a 5-line chroma cycle */
    const i32 u = 892, line_ns = (3 + 3 + 2 + 4 + 4 + 55) * 892;
    memset(s, 0, sizeof(*s));
    s->system = OCRT_SYS_PV1K;
    s->chroma_pattern = 0;
    s->cc_samples = 5;
    s->hres = 2304 * 5 / 6;
    s->vres = 262;
    s->top = 21;
    s->bot = 261;
    s->cc_vper = 5;
    s->hsync_window = 8;
    s->vsync_window = 8;
    s->hsync_thresh = 4;
    s->vsync_thresh = 94;
    s->sync_beg = (3 * u) * s->hres / line_ns;
    s->bw_beg = (6 * u) * s->hres / line_ns;
    s->cb_beg = (8 * u) * s->hres / line_ns;
    s->av_beg = (16 * u) * s->hres / line_ns;
    s->av_len = (55 * u) * s->hres / line_ns;
    s->white_level = 100;
    s->burst_level = 20;
    s->black_level = 7;
    s->blank_level = 0;
    s->sync_level = -40;
    s->iir_c[0] = bandlimit_coeff(420000); /* crt_pv1k.h: the NTSC bandwidths */
    s->iir_c[1] = bandlimit_coeff(150000);
    s->iir_c[2] = bandlimit_coeff(55000);
    finish_sys(s);
}

static void
make_nesrgb_sys(ocrt_sys *s, int pattern)
{
    /* crt_nesrgb.h: the NES layout (all three chroma patterns, crt_nesrgb.h:27-40) and sync / burst levels, white at 100 */
    make_nes_sys(s, pattern);
    s->system = OCRT_SYS_NESRGB;
    s->white_level = 100;
}

const ocrt_sys *
ocrt_system(int system, int chroma_pattern)
{
    static ocrt_sys table[11];
    static int ready = 0;
    if (!ready) {
        make_snes_sys(&table[5]);
        make_nesrgb_sys(&table[6], 2);
        make_nesrgb_sys(&table[9], 0);
        make_nesrgb_sys(&table[10], 1);
        make_template_sys(&table[7]);
        make_pv1k_sys(&table[8]);
        make_rgb_sys(&table[0], OCRT_SYS_NTSC);
        make_rgb_sys(&table[1], OCRT_SYS_VHS);
        make_nes_sys(&table[2], 0);
        make_nes_sys(&table[3], 1);
        make_nes_sys(&table[4], 2);
        ready = 1;
    }
    if (system == OCRT_SYS_NTSC) return &table[0];
    if (system == OCRT_SYS_VHS) return &table[1];
    if (system == OCRT_SYS_SNES) return &table[5];
    if (system == OCRT_SYS_NESRGB) return chroma_pattern == 0 ? &table[9] : chroma_pattern == 1 ? &table[10] : &table[6];
    if (system == OCRT_SYS_TEMP) return &table[7];
    if (system == OCRT_SYS_PV1K) return &table[8];
    if (system == OCRT_SYS_NES && chroma_pattern >= 0 && chroma_pattern <= 2)
        return &table[2 + chroma_pattern];
    return NULL;
}

const ocrt_sys *
ocrt_system_conv_taps(int system, int chroma_pattern, int taps)
{
    static ocrt_sys table[4][9];
    static int ready[4][9];
    const ocrt_sys *base = ocrt_system(system, chroma_pattern);
    int slot;
    if (!base || taps < 4 || taps > 7) return NULL;
    slot = (system == OCRT_SYS_NTSC) ? 0 : (system == OCRT_SYS_VHS) ? 1 : (system == OCRT_SYS_SNES) ? 5 : (system == OCRT_SYS_NESRGB) ? 6 : (system == OCRT_SYS_TEMP) ? 7 : (system == OCRT_SYS_PV1K) ? 8 : 2 + chroma_pattern;
    if (!ready[taps - 4][slot]) {
        table[taps - 4][slot] = *base;
        table[taps - 4][slot].conv = taps;
        ready[taps - 4][slot] = 1;
    }
    return &table[taps - 4][slot];
}

const ocrt_sys *
ocrt_system_bloom(int system, int chroma_pattern)
{
    static ocrt_sys table[9];
    static int ready[9];
    const ocrt_sys *base = ocrt_system(system, chroma_pattern);
    int slot;
    if (!base || system == OCRT_SYS_NES || system == OCRT_SYS_NESRGB) return NULL; /* "does not work for NES" */
    slot = (system == OCRT_SYS_NTSC) ? 0 : (system == OCRT_SYS_VHS) ? 1 : (system == OCRT_SYS_SNES) ? 5
         : (system == OCRT_SYS_TEMP) ? 7 : 8;
    if (!ready[slot]) {
        table[slot] = *base;
        table[slot].bloom = 1;
        ready[slot] = 1;
    }
    return &table[slot];
}

const ocrt_sys *
ocrt_system_conv(int system, int chroma_pattern)
{
    return ocrt_system_conv_taps(system, chroma_pattern, 7); /* USE_7_SAMPLE_KERNEL 1 is the stock setting */
}

/* ------------------------------------------------------------------------- */
/* monitor state (crt_core.c:241-289)                                         */
/* ------------------------------------------------------------------------- */

void
ocrt_monitor_reset(ocrt_monitor *m) /* crt_core.c:250-261 */
{
    m->hue = 0;
    m->saturation = 10;
    m->brightness = 0;
    m->contrast = 180;
    m->black_point = 0;
    m->white_point = 100;
    m->hsync = 0;
    m->vsync = 0;
}

int
ocrt_monitor_create(const ocrt_sys *sys, ocrt_monitor *m, int w, int h, int f, unsigned char *out)
{
    memset(m, 0, sizeof(*m));
    m->analog = (signed char *) calloc((size_t) sys->input_size + OCRT_PAD, 1);
    m->inp = (signed char *) calloc((size_t) sys->input_size + OCRT_PAD, 1);
    if (!m->analog || !m->inp) return 0;
    m->outw = w;
    m->outh = h;
    m->out_format = f;
    m->out = out;
    ocrt_monitor_reset(m);
    m->rn = 194; /* crt_core.c:269 */
    return 1;
}

void
ocrt_monitor_destroy(ocrt_monitor *m)
{
    free(m->analog);
    free(m->inp);
    m->analog = m->inp = NULL;
}

/* ------------------------------------------------------------------------- */
/* encoder, RGB systems (crt_ntsc.c:128-330, crt_ntscvhs.c:128-337)           */
/* ------------------------------------------------------------------------- */

static void
fill(signed char *line, i32 from, i32 to, i32 level)
{
    i32 t;
    for (t = from; t < to; t++) line[t] = (signed char) level;
}

/* size of the encoded picture (crt_ntsc.c:148-172, same block in crt_snes.c / crt_template.c / crt_pv1k.c):
 * with CRT_DO_BLOOM the picture leaves room for the line to widen */
static void
picture_size(const ocrt_sys *sys, const ocrt_rgb_source *src, i32 *destw, i32 *desth)
{
    const i32 maxw = sys->bloom ? (sys->av_len * 55500) >> 16 : sys->av_len;
    const i32 maxh = sys->bloom ? (sys->lines * 63500) >> 16 : (sys->lines * 64500) >> 16;
    if (src->raw) {
        *destw = src->w < maxw ? src->w : maxw;
        *desth = src->h < maxh ? src->h : maxh;
    } else {
        *destw = maxw;
        *desth = maxh;
    }
}

void
ocrt_encode_rgb(const ocrt_sys *sys, ocrt_monitor *m, ocrt_rgb_source *src, ocrt_rand *g)
{
    const i32 H = sys->hres;
    i32 destw, desth;
    i32 burst[4], modI[4], modQ[4], primed[4] = { 0, 0, 0, 0 };
    i32 k, n, x, y, xo, yo, flip, ph, bpp, aberration = 0, white;

    picture_size(sys, src, &destw, &desth);
    for (k = 0; k < 4; k++) { /* crt_ntsc.c:174-188 */
        if (src->as_color) {
            i32 deg = src->hue + k * 90;
            burst[k] = sin14((deg + 33) * 8192 / 180) >> 10;
            modI[k] = sin14(deg * 8192 / 180) >> 10;
            modQ[k] = sin14((deg - 90) * 8192 / 180) >> 10;
        } else {
            burst[k] = modI[k] = modQ[k] = 0;
        }
    }
    bpp = ocrt_bpp(src->format);
    if (bpp == 0) return; /* crt_ntsc.c:190-193 */

    xo = sys->av_beg + src->xoffset + (sys->av_len - destw) / 2;
    yo = sys->top + src->yoffset + (sys->lines - desth) / 2;
    src->field &= 1;
    src->frame &= 1;
    flip = (src->field == src->frame);
    ph = flip ? -1 : 1; /* CC_PHASE, crt_ntsc.c:18-23, pattern 1 */
    xo &= ~3;

    if (sys->system == OCRT_SYS_VHS && src->do_aberration) /* crt_ntscvhs.c:205-207 */
        aberration = ((ocrt_rand_next(g) % 12) - 8) + 14;

    /* sync / blanking / burst skeleton of every line (crt_ntsc.c:205-252) */
    for (n = 0; n < sys->vres; n++) {
        signed char *line = m->analog + n * H;
        if (n <= 3 || (n >= 7 && n <= 9)) {
            fill(line, 0, 4 * H / 100, sys->sync_level);
            fill(line, 4 * H / 100, 50 * H / 100, sys->blank_level);
            fill(line, 50 * H / 100, 54 * H / 100, sys->sync_level);
            fill(line, 54 * H / 100, H, sys->blank_level);
        } else if (n >= 4 && n <= 6) {
            i32 first = (src->field == 1) ? 4 : 46;
            fill(line, 0, first * H / 100, sys->sync_level);
            fill(line, first * H / 100, 50 * H / 100, sys->blank_level);
            fill(line, 50 * H / 100, 96 * H / 100, sys->sync_level);
            fill(line, 96 * H / 100, H, sys->blank_level);
        } else {
            i32 t;
            if (n < sys->vres - aberration) { /* crt_ntscvhs.c:234-238 */
                fill(line, 0, sys->sync_beg, sys->blank_level);
                fill(line, sys->sync_beg, sys->bw_beg, sys->sync_level);
                fill(line, sys->bw_beg, sys->av_beg, sys->blank_level);
            } else {
                fill(line, 0, sys->av_beg, sys->blank_level);
            }
            if (n < sys->top) fill(line, sys->av_beg, H, sys->blank_level);
            for (t = sys->cb_beg; t < sys->cb_beg + sys->burst_len; t++) {
                i32 cb = burst[(t + flip * 2) & 3];
                line[t] = (signed char) ((sys->blank_level + cb * sys->burst_level) >> 5);
                primed[t & 3] = line[t];
            }
        }
    }
    if (sys->system == OCRT_SYS_VHS) m->hsync = 0; /* crt_ntscvhs.c:258-259 */

    /* picture (crt_ntsc.c:254-324) */
    white = white_scale(sys, m->white_point);
    for (y = 0; y < desth; y++) {
        i32 hy = 0, hi = 0, hq = 0;
        i32 row = (y * src->h) / desth + (src->field * src->h + desth) / desth / 2;
        if (row >= src->h) row = src->h;
        for (x = 0; x < destw; x++) {
            const unsigned char *px = src->data + (size_t) (((x * src->w) / destw) + row * src->w) * bpp;
            i32 r = px[fmt_r[src->format]], gg = px[fmt_g[src->format]], b = px[fmt_b[src->format]];
            i32 fy = (19595 * r + 38470 * gg + 7471 * b) >> 14;
            i32 fi = (39059 * r - 18022 * gg - 21103 * b) >> 14;
            i32 fq = (13894 * r - 34275 * gg + 20382 * b) >> 14;
            i32 ph4 = (x + xo) % 4, ire;
            hy += wmul(fy - hy, sys->iir_c[0]) >> 11; /* iirf, crt_ntsc.c:117-126 */
            hi += wmul(fi - hi, sys->iir_c[1]) >> 11;
            hq += wmul(fq - hq, sys->iir_c[2]) >> 11;
            fi = wmul(wmul(hi, ph), modI[ph4]) >> 4;
            fq = wmul(wmul(hq, ph), modQ[ph4]) >> 4;
            ire = sys->black_level + m->black_point;
            ire += wmul(hy + fi + fq, white) >> 10;
            if (ire < 0) ire = 0;
            if (ire > 110) ire = 110;
            m->analog[(x + xo) + (y + yo) * H] = (signed char) ire;
        }
    }
    for (n = 0; n < sys->cc_vper; n++) /* crt_ntsc.c:325-329 / crt_ntscvhs.c:332-336 */
        for (x = 0; x < 4; x++)
            m->ccf[n][x] = (sys->system == OCRT_SYS_VHS) ? 0 : primed[x] * 128;
}

/* ------------------------------------------------------------------------- */
/* encoder, SNES (crt_snes.c:125-327)                                          */
/* ------------------------------------------------------------------------- */

/* crt_snes.c, crt_template.c and crt_pv1k.c are one encoder with a handful of switches */
typedef struct enc_family {
    i32 vert_step;  /* degrees per line of the vertical chroma cycle: 360 / VPER, PV-1000 720 / VPER */
    i32 burst_off;  /* HUE_OFFSET added to the burst angle (crt_snes.h:99, crt_template.h:68; 0 for the PV-1000) */
    i32 q_off;      /* Q_OFFSET: -90, PV-1000 +90 (crt_pv1k.c:176) */
    int bandlimit;  /* CRT_DO_BANDLIMITING */
    int fielded;    /* the field parity shapes the vertical sync and the source row (crt_template.c:217-225, 252-258) */
    i32 equ_a_lo, equ_a_hi, equ_b_lo, equ_b_hi, sync_lo, sync_hi; /* template line ranges */
} enc_family;

static void
encode_template_family(const ocrt_sys *sys, ocrt_monitor *m, ocrt_rgb_source *src, const enc_family *fam)
{
    const i32 H = sys->hres, V = sys->cc_vper, CC = sys->cc_samples;
    i32 bpp = ocrt_bpp(src->format);
    i32 destw, desth;
    i32 modI[OCRT_MAX_VPER][OCRT_MAX_CC], modQ[OCRT_MAX_VPER][OCRT_MAX_CC], burst[OCRT_MAX_VPER][OCRT_MAX_CC];
    i32 primed[OCRT_MAX_VPER][OCRT_MAX_CC];
    i32 n, x, y, xo, yo, white;

    picture_size(sys, src, &destw, &desth); /* crt_snes.c:148-168 */
    for (y = 0; y < V; y++) /* crt_snes.c:170-187 */
        for (x = 0; x < CC; x++) {
            i32 step = 360 / CC, deg = (y + src->dot_crawl_offset) * fam->vert_step + src->hue + x * step;
            burst[y][x] = modI[y][x] = modQ[y][x] = 0;
            if (src->as_color) {
                burst[y][x] = sin14((deg - step + fam->burst_off) * 8192 / 180) >> 10;
                modI[y][x] = sin14(deg * 8192 / 180) >> 10;
                modQ[y][x] = sin14((deg + fam->q_off) * 8192 / 180) >> 10;
            }
        }
    if (bpp == 0) return; /* crt_snes.c:189-192 */
    xo = sys->av_beg + src->xoffset + (sys->av_len - destw) / 2;
    yo = sys->top + src->yoffset + (sys->lines - desth) / 2;
    src->field &= 1;
    src->frame &= 1;
    xo = xo - (xo % CC);
    memset(primed, 0, sizeof(primed));

    for (n = 0; n < sys->vres; n++) { /* crt_snes.c:203-250 */
        signed char *line = m->analog + n * H;
        if ((n >= fam->equ_a_lo && n <= fam->equ_a_hi) || (n >= fam->equ_b_lo && n <= fam->equ_b_hi)) {
            fill(line, 0, 4 * H / 100, sys->sync_level);
            fill(line, 4 * H / 100, 50 * H / 100, sys->blank_level);
            fill(line, 50 * H / 100, 54 * H / 100, sys->sync_level);
            fill(line, 54 * H / 100, H, sys->blank_level);
        } else if (n >= fam->sync_lo && n <= fam->sync_hi) {
            i32 first = (fam->fielded && src->field == 1) ? 4 : 46; /* crt_template.c:220-225 */
            fill(line, 0, first * H / 100, sys->sync_level);
            fill(line, first * H / 100, 50 * H / 100, sys->blank_level);
            fill(line, 50 * H / 100, 96 * H / 100, sys->sync_level);
            fill(line, 96 * H / 100, H, sys->blank_level);
        } else {
            i32 t;
            fill(line, 0, sys->sync_beg, sys->blank_level);
            fill(line, sys->sync_beg, sys->bw_beg, sys->sync_level);
            fill(line, sys->bw_beg, sys->av_beg, sys->blank_level);
            if (n < sys->top) fill(line, sys->av_beg, H, sys->blank_level);
            for (t = sys->cb_beg; t < sys->cb_beg + sys->burst_len; t++) {
                line[t] = (signed char) ((sys->blank_level + burst[n % V][t % CC] * sys->burst_level) >> 5);
                primed[(n + 3) % V][t % CC] = line[t];
            }
        }
    }

    white = white_scale(sys, m->white_point);
    for (y = 0; y < desth; y++) { /* crt_snes.c:252-320 */
        i32 hy = 0, hi = 0, hq = 0; /* reset_iir per line */
        i32 row = (y * src->h) / desth, ph = (y + yo) % V;
        if (fam->fielded) row += (src->field * src->h + desth) / desth / 2; /* crt_template.c:255-258 */
        if (row >= src->h) row = src->h;
        for (x = 0; x < destw; x++) {
            const unsigned char *px = src->data + (size_t) (((x * src->w) / destw) + row * src->w) * bpp;
            i32 r = px[fmt_r[src->format]], gg = px[fmt_g[src->format]], b = px[fmt_b[src->format]];
            i32 fy = (19595 * r + 38470 * gg + 7471 * b) >> 14;
            i32 fi = (39059 * r - 18022 * gg - 21103 * b) >> 14;
            i32 fq = (13894 * r - 34275 * gg + 20382 * b) >> 14;
            i32 xoff = (x + xo) % CC, ire;
            if (fam->bandlimit) { /* iirf, crt_template.c:117-126 (CRT_DO_BANDLIMITING 1) */
                hy += wmul(fy - hy, sys->iir_c[0]) >> 11;
                hi += wmul(fi - hi, sys->iir_c[1]) >> 11;
                hq += wmul(fq - hq, sys->iir_c[2]) >> 11;
                fy = hy;
                fi = hi;
                fq = hq;
            }
            fi = wmul(fi, modI[ph][xoff]) >> 4;
            fq = wmul(fq, modQ[ph][xoff]) >> 4;
            ire = sys->black_level + m->black_point + (wmul(fy + fi + fq, white) >> 10);
            if (ire < 0) ire = 0;
            if (ire > 110) ire = 110;
            m->analog[(x + xo) + (y + yo) * H] = (signed char) ire;
        }
    }
    for (n = 0; n < V; n++) /* crt_snes.c:322-326 */
        for (x = 0; x < CC; x++) m->ccf[n][x] = primed[n][x] * 128;
}

void
ocrt_encode_snes(const ocrt_sys *sys, ocrt_monitor *m, ocrt_rgb_source *src)
{
    static const enc_family fam = { 360 / 3, 210, -90, 0, 0, 0, 2, 7, 9, 3, 6 }; /* crt_snes.h:84-109 */
    encode_template_family(sys, m, src, &fam);
}

/* crt_template.c:125-337: the reference's worked example for new systems -- NTSC timing with a 2-line
 * chroma cycle, band-limited (crt_template.h:52, 68) */
void
ocrt_encode_template(const ocrt_sys *sys, ocrt_monitor *m, ocrt_rgb_source *src)
{
    static const enc_family fam = { 360 / 2, -60, -90, 1, 1, 0, 2, 7, 9, 3, 6 };
    encode_template_family(sys, m, src, &fam);
}

/* crt_pv1k.c:125-321: Casio PV-1000 -- 5 samples per chroma period, 5-line cycle stepping 144 degrees, no
 * first equalising region, vertical sync on lines 258-260 */
void
ocrt_encode_pv1k(const ocrt_sys *sys, ocrt_monitor *m, ocrt_rgb_source *src)
{
    static const enc_family fam = { 360 * 2 / 5, 0, 90, 1, 1, 1, 0, 7, 9, 258, 260 };
    encode_template_family(sys, m, src, &fam);
}

/* ------------------------------------------------------------------------- */
/* encoder, NES-RGB (crt_nesrgb.c:19-172)                                      */
/* ------------------------------------------------------------------------- */

void
ocrt_encode_nesrgb(const ocrt_sys *sys, ocrt_monitor *m, ocrt_nesrgb_source *src)
{
    const i32 H = sys->hres;
    i32 modI[3][4], modQ[3][4], burst[3][4], primed[3][4];
    i32 n, x, y, xo, yo, white, bpp;

    memset(primed, 0, sizeof(primed));
    if (!src->field_initialized) { /* setup_field, crt_nesrgb.c:19-47 */
        for (n = 0; n < sys->vres; n++) {
            signed char *line = m->analog + n * H;
            fill(line, 0, sys->sync_beg, sys->blank_level);
            fill(line, sys->sync_beg, n >= 259 ? sys->nes_vsync_end : sys->bw_beg, sys->sync_level);
            fill(line, n >= 259 ? sys->nes_vsync_end : sys->bw_beg, H, sys->blank_level);
        }
        src->field_initialized = 1;
    }
    for (y = 0; y < 3; y++) /* crt_nesrgb.c:68-79 */
        for (x = 0; x < 4; x++) {
            i32 deg = (y + src->dot_crawl_offset) * 120 + x * 90;
            burst[y][x] = sin14((src->hue + 90 + deg + 33) * 8192 / 180) >> 10;
            modI[y][x] = sin14(deg * 8192 / 180) >> 10;
            modQ[y][x] = sin14((deg - 90) * 8192 / 180) >> 10;
        }
    bpp = ocrt_bpp(src->format);
    if (bpp == 0) return; /* crt_nesrgb.c:81-84 */
    xo = (sys->av_beg + src->xoffset) & ~3;
    yo = sys->top + src->yoffset;
    white = white_scale(sys, m->white_point);

    for (y = 0; y < sys->lines; y++) { /* crt_nesrgb.c:92-164 */
        signed char *line = m->analog + (y + yo) * H;
        i32 row = (y * src->h) / sys->lines, t, ph = (y + yo) % 3;
        if (row >= src->h) row = src->h;
        if (row < 0) row = 0;
        for (t = sys->cb_beg; t < sys->cb_beg + sys->burst_len; t++) {
            line[t] = (signed char) ((sys->blank_level + burst[ph][t % 4] * sys->burst_level) >> 5);
            primed[ph][t % 4] = line[t];
        }
        for (x = 0; x < sys->av_len; x++) {
            const unsigned char *px = src->data + (size_t) (((x * src->w) / sys->av_len) + row * src->w) * bpp;
            i32 r = px[fmt_r[src->format]], gg = px[fmt_g[src->format]], b = px[fmt_b[src->format]];
            i32 fy = (19595 * r + 38470 * gg + 7471 * b) >> 14;
            i32 fi = (39059 * r - 18022 * gg - 21103 * b) >> 14;
            i32 fq = (13894 * r - 34275 * gg + 20382 * b) >> 14;
            i32 xoff = (x + xo) % 4, ire;
            fi = wmul(fi, modI[ph][xoff]) >> 4;
            fq = wmul(fq, modQ[ph][xoff]) >> 4;
            ire = sys->black_level + m->black_point + (wmul(fy + fi + fq, white) >> 10);
            if (ire < 0) ire = 0;
            if (ire > 110) ire = 110;
            line[x + xo] = (signed char) ire;
        }
    }
    for (n = 0; n < 3; n++) /* crt_nesrgb.c:166-170 */
        for (x = 0; x < 4; x++) m->ccf[n][x] = primed[n][x] * 128;
}

/* ------------------------------------------------------------------------- */
/* encoder, NES (crt_nes.c:21-61, 81-201)                                      */
/* ------------------------------------------------------------------------- */

static i32
nes_square(i32 p, i32 phase) /* crt_nes.c:21-61 */
{
    static const i32 level[16] = {
        -12042, 0, 34406, 81427, -17203, -8028, 19497, 57342,
        43581, 75693, 112965, 112965, 26951, 52181, 83721, 83721
    };
    static const i32 emph_mask[6] = { 0300, 0100, 0500, 0400, 0600, 0200 };
    i32 hue = p & 15, high, emph;
    if (hue >= 14) return 0;
    emph = ((p & 0700) & emph_mask[(phase >> 1) % 6]) > 0;
    if (hue == 0) high = 1;
    else if (hue == 13) high = 0;
    else high = ((hue + phase) % 12) < 6;
    return level[high * 8 + emph * 4 + ((p >> 4) & 3)];
}

void
ocrt_encode_nes(const ocrt_sys *sys, ocrt_monitor *m, ocrt_nes_source *src)
{
    const i32 H = sys->hres;
    i32 burst[3][4], primed[3][4];
    i32 n, x, y, xo, yo;

    memset(primed, 0, sizeof(primed));
    if (!src->field_initialized) { /* setup_field, crt_nes.c:81-104 */
        for (n = 0; n < sys->vres; n++) {
            signed char *line = m->analog + n * H;
            fill(line, 0, sys->sync_beg, sys->blank_level);
            fill(line, sys->sync_beg, n >= 259 ? sys->nes_vsync_end : sys->bw_beg, sys->sync_level);
            fill(line, n >= 259 ? sys->nes_vsync_end : sys->bw_beg, H, sys->blank_level);
        }
        src->field_initialized = 1;
    }
    for (y = 0; y < 3; y++) /* crt_nes.c:123-130 */
        for (x = 0; x < 4; x++) {
            i32 deg = (src->hue + x * 90 + (y + src->dot_crawl_offset) * 120 + 33) % 360;
            burst[y][x] = sin14(deg * 8192 / 180) >> 10;
        }
    xo = (sys->av_beg + src->xoffset) & ~3;
    yo = sys->top + src->yoffset;

    for (y = 0; y < sys->lines; y++) { /* crt_nes.c:160-194 */
        signed char *line = m->analog + (y + yo) * H;
        i32 row = (y * src->h) / sys->lines, t, phase;
        if (row >= src->h) row = src->h;
        if (row < 0) row = 0;
        n = y + yo;
        for (t = sys->cb_beg; t < sys->cb_beg + sys->burst_len; t++) {
            line[t] = (signed char) ((sys->blank_level + burst[n % 3][t & 3] * sys->burst_level) >> 5);
            primed[n % 3][t & 3] = line[t];
        }
        phase = ((y + yo + src->dot_crawl_offset) % 3) * 4; /* phasetab, crt_nes.c:116 */
        for (x = 0; x < sys->av_len; x++) {
            i32 p = src->data[((x * src->w) / sys->av_len) + row * src->w];
            i32 ire = sys->black_level + m->black_point;
            ire += nes_square(p, phase) + nes_square(p, phase + 1)
                 + nes_square(p, phase + 2) + nes_square(p, phase + 3);
            ire = (wmul(ire, m->white_point) / 100) >> 12;
            line[x + xo] = (signed char) ire;
            phase += 3;
        }
    }
    for (n = 0; n < 3; n++)
        for (x = 0; x < 4; x++)
            m->ccf[n][x] = primed[n][x] * 128;
}

/* ------------------------------------------------------------------------- */
/* decoder (crt_core.c:291-666)                                               */
/* ------------------------------------------------------------------------- */

void
ocrt_lcg_jump(unsigned n, unsigned *mul, unsigned *add)
{
    u32 am = 214019u, ac = 140327895u, rm = 1u, rc = 0u;
    while (n) {
        if (n & 1) { rc = rc * am + ac; rm = rm * am; }
        ac = ac * am + ac;
        am = am * am;
        n >>= 1;
    }
    *mul = rm;
    *add = rc;
}

/* In the reference inp[] is followed, inside struct CRT, by outw, outh, out_format and four bytes of padding
 * (crt_core.h:74-92; crt_init zeroes the struct): a decode window or sync search that runs a few samples past the
 * end of inp[] reads those bytes.  They are deterministic, so they are reproduced here (16 bytes); what follows
 * them is the `out` pointer, which is not (windows that reach it are outside the parity domain). */
static void
inp_struct_tail(const ocrt_sys *sys, ocrt_monitor *m)
{
    i32 v[4];
    v[0] = m->outw;
    v[1] = m->outh;
    v[2] = m->out_format;
    v[3] = 0;
    memcpy(m->inp + sys->input_size, v, sizeof(v));
}

/* signal + noise -> inp (crt_core.c:343-367) */
void
ocrt_noise_pass(const ocrt_sys *sys, ocrt_monitor *m, int noise, ocrt_rand *g)
{
    i32 i, rn = m->rn, wobble = 0;
    m->last_noise = noise;
    inp_struct_tail(sys, m);
    if (sys->vhs_noise) wobble = ((ocrt_rand_next(g) % 8) - 4) + 14; /* crt_core.c:344 */
    for (i = 0; i < sys->input_size; i++) {
        i32 gain = noise, s;
        if (sys->vhs_noise) { /* crt_core.c:348-357 */
            rn = ocrt_rand_next(g);
            if (i > sys->input_size - sys->hres * (16 + ((ocrt_rand_next(g) % 20) - 10))
                && i < sys->input_size - sys->hres * (5 + ((ocrt_rand_next(g) % 8) - 4))) {
                i32 ln = (i * wobble) / sys->hres;
                gain = cos14(ln * 8192 / 180) >> 8;
            }
        } else {
            rn = wadd(wmul(214019, rn), 140327895); /* crt_core.c:359 */
        }
        s = m->analog[i] + (wmul(((rn >> 16) & 0xff) - 0x7f, gain) >> 8);
        if (s > 127) s = 127;
        if (s < -127) s = -127;
        m->inp[i] = (signed char) s;
    }
    m->rn = rn;
}

/* vsync search, then the line-to-line chain of hsync search and colour-burst lock
 * (crt_core.c:369-479).  Returns the detected field (0/1) and fills one record per
 * decoded scanline; updates m->vsync, m->hsync and m->ccf exactly as the reference. */
int
ocrt_sync_pass(const ocrt_sys *sys, ocrt_monitor *m, ocrt_line *table)
{
    const i32 H = sys->hres;
    i32 i, j = 0, line = 0, acc, field, ratio, huesn, huecs, k;

    {
        int sn, cs;
        ocrt_sincos14(&sn, &cs, ((m->hue % 360) + 33) * 8192 / 180); /* crt_core.c:318-320 */
        huesn = sn >> 11;
        huecs = cs >> 11;
    }
    for (i = -sys->vsync_window; i < sys->vsync_window; i++) { /* crt_core.c:379-396 */
        const signed char *sig;
        line = posmod(m->vsync + i, sys->vres);
        sig = m->inp + line * H;
        acc = 0;
        for (j = 0; j < H; j++) {
            acc += sig[j];
            if (acc <= sys->vsync_thresh * sys->sync_level) goto locked;
        }
    }
locked:
    m->vsync = line;
    field = (j > H / 2);
    ratio = (((m->outh << 16) / sys->lines) + 32768) >> 16; /* crt_core.c:404-405 */
    field *= ratio / 2;

    for (k = 0; k < sys->lines; k++) {
        ocrt_line *rec = &table[k];
        const signed char *sig;
        i32 ln, xpos, ypos, pa, dci, dcq, w0, w1;
        i32 *ccr;
        line = sys->top + k;
        memset(rec, 0, sizeof(*rec));
        rec->beg = (i32) ((u32) k * ((u32) m->outh + m->v_fac) / (u32) sys->lines + (u32) field);
        rec->end = (i32) ((u32) (k + 1) * ((u32) m->outh + m->v_fac) / (u32) sys->lines + (u32) field);
        if (rec->beg >= m->outh) { rec->skip = 1; rec->hsync = m->hsync; continue; }
        if (rec->end > m->outh) rec->end = m->outh;

        ln = posmod(line + m->vsync, sys->vres) * H; /* crt_core.c:437-450 */
        sig = m->inp + ln + m->hsync;
        acc = 0;
        for (i = -sys->hsync_window; i < sys->hsync_window; i++) {
            acc += sig[sys->sync_beg + i];
            if (acc <= sys->hsync_thresh * sys->sync_level) break;
        }
        m->hsync = posmod(i + m->hsync, H);
        rec->hsync = m->hsync;

        xpos = posmod(sys->av_beg + m->hsync - 3, H); /* xnudge -3, ynudge +3 */
        ypos = posmod(line + m->vsync + 3, sys->vres);
        rec->pos = xpos + ypos * H;

        ccr = m->ccf[ypos % sys->cc_vper]; /* crt_core.c:456-467 */
        if (sys->cc_samples == 4) {
            sig = m->inp + ln + (m->hsync & ~3);
            for (i = sys->cb_beg; i < sys->cb_beg + sys->burst_len; i++)
                ccr[i & 3] = wadd(wmul(ccr[i & 3], 127) / 128, sig[i]);

            pa = m->hsync & 3; /* crt_core.c:469-479 */
            dci = wsub(ccr[(pa + 1) & 3], ccr[(pa + 3) & 3]);
            dcq = wsub(ccr[(pa + 2) & 3], ccr[pa & 3]);
            w0 = wmul(wsub(wmul(dci, huecs), wmul(dcq, huesn)) >> 4, m->saturation);
            w1 = wmul(wadd(wmul(dcq, huecs), wmul(dci, huesn)) >> 4, m->saturation);
            rec->wave[0] = w0;
            rec->wave[1] = w1;
            rec->wave[2] = wsub(0, w0);
            rec->wave[3] = wsub(0, w1);
        } else { /* CRT_CC_SAMPLES 5, crt_core.c:459-467, 480-509 */
            const i32 CC = sys->cc_samples;
            i32 ang = m->hue % 360, peak_a, peak_b;
            sig = m->inp + ln + (m->hsync - (m->hsync % CC));
            for (i = sys->cb_beg; i < sys->cb_beg + sys->burst_len; i++)
                ccr[i % CC] = wadd(wmul(ccr[i % CC], 127) / 128, sig[i]);
            pa = posmod(m->hsync, CC);
            peak_a = pa + CC / 4;
            peak_b = pa;
            dci = wsub(ccr[peak_a % CC], wadd(ccr[(peak_a + CC / 2) % CC], ccr[(peak_a + CC / 2 + 1) % CC]) / 2);
            dcq = wsub(ccr[(peak_b + CC / 2) % CC], ccr[peak_b % CC]);
            for (i = 0; i < CC; i++) {
                int sn, cs;
                ocrt_sincos14(&sn, &cs, ang * 8192 / 180);
                rec->wave_i[i] = wmul(wadd(wmul(dci, cs), wmul(dcq, sn)) >> 15, m->saturation);
                ocrt_sincos14(&sn, &cs, (ang + 90) * 8192 / 180);
                rec->wave_q[i] = wmul(wadd(wmul(dci, cs), wmul(dcq, sn)) >> 15, m->saturation);
                ang += 360 / CC;
            }
            (void) w0;
            (void) w1;
        }
    }
    return field;
}

/* one channel of the three-band equaliser (crt_core.c:151-233) */
typedef struct eq_state {
    i32 lo[4], hi[4], hist[3];
} eq_state;

static i32
eq_step(eq_state *f, const int *c, i32 s)
{
    i32 k, r0, r1, r2, in_lo = s, in_hi = s;
    for (k = 0; k < 4; k++) {
        f->lo[k] = wadd(f->lo[k], wadd(wmul(c[0], wsub(in_lo, f->lo[k])), 32768) >> 16);
        f->hi[k] = wadd(f->hi[k], wadd(wmul(c[1], wsub(in_hi, f->hi[k])), 32768) >> 16);
        in_lo = f->lo[k];
        in_hi = f->hi[k];
    }
    r0 = wmul(f->lo[3], c[2]) >> 16;
    r1 = wmul(wsub(f->hi[3], f->lo[3]), c[3]) >> 16;
    r2 = wmul(wsub(f->hist[2], f->hi[3]), c[4]) >> 16;
    f->hist[2] = f->hist[1];
    f->hist[1] = f->hist[0];
    f->hist[0] = s;
    return wadd(wadd(r0, r1), r2);
}

/* eqf() of the USE_CONVOLUTION build (crt_core.c:96-147): a 7-deep history, zero at the start of every
 * line (reset_eq, crt_core.c:117-121), newest sample in h[0]; the kernel is chosen at compile time among
 * USE_7_SAMPLE_KERNEL (default), USE_6_, USE_5_ and the 4-tap fall-back (crt_core.c:86-88, 130-146) */
typedef struct fir_state {
    i32 h[7];
} fir_state;

static i32
fir_step(fir_state *f, i32 s, int taps)
{
    i32 k;
    i32 *h = f->h;
    for (k = 6; k > 0; k--) h[k] = h[k - 1];
    h[0] = s;
    if (taps == 7) /* weights 1 4 7 8 7 4 1 */
        return wadd(wadd(wadd(wadd(s, h[6]), wmul(wadd(h[1], h[5]), 4)), wmul(wadd(h[2], h[4]), 7)), wmul(h[3], 8)) >> 5;
    if (taps == 6) /* weights 1 3 4 4 3 1 */
        return wadd(wadd(wadd(s, h[5]), wmul(3, wadd(h[1], h[4]))), wmul(4, wadd(h[2], h[3]))) >> 4;
    if (taps == 5) /* weights 1 2 2 2 1 */
        return wadd(wadd(s, h[4]), wmul(wadd(wadd(h[1], h[2]), h[3]), 2)) >> 3;
    return wadd(wadd(wadd(s, h[3]), h[1]), h[2]) >> 2; /* weights 1 1 1 1 */
}

/* carrier sample of I / Q at signal sample i: crt_core.c:538-543 (4 samples per period: one table, Q three
 * samples behind) or 545-549 (5 samples: two tables) */
#define WAVE_I(i) (sys->cc_samples == 4 ? rec->wave[(i) & 3] : rec->wave_i[(i) % sys->cc_samples])
#define WAVE_Q(i) (sys->cc_samples == 4 ? rec->wave[((i) + 3) & 3] : rec->wave_q[(i) % sys->cc_samples])

/* filter + resample + YIQ->RGB for decoded lines [first, first+count)
 * (crt_core.c:511-664) */
void
ocrt_line_pass(const ocrt_sys *sys, ocrt_monitor *m, const ocrt_line *table, int first, int count)
{
    const i32 L = sys->av_len;
    i32 bpp = ocrt_bpp(m->out_format), pitch, bright, k, dx;
    i32 *yy, *ii, *qq;
    /* CRT_DO_BLOOM (crt_core.c:399-402, 512-526): filtered beam energy, carried from line to line of the call */
    const i32 max_e = (128 + (m->last_noise / 2)) * sys->av_len;
    i32 prev_e = 16384 / 8, k0 = sys->bloom ? 0 : first;

    if (bpp == 0) return;
    pitch = m->outw * bpp;
    bright = m->brightness - (sys->black_level + m->black_point);
    yy = (i32 *) calloc((size_t) (L + 1) * 3, sizeof(i32));
    ii = yy + (L + 1);
    qq = ii + (L + 1);
    dx = ((L - 1) << 12) / m->outw;

    for (k = k0; k < first + count; k++) { /* (with bloom the energy chain is walked from the first line) */
        const ocrt_line *rec = &table[k];
        const signed char *sig = m->inp + rec->pos;
        eq_state ey, ei, eq;
        fir_state fy, fi, fq;
        unsigned char *px, *row_end;
        u32 pos, scan_l = 0, scan_r = (u32) ((L - 1) << 12);
        i32 i, row, f_lo = 0, f_hi = L;
        if (rec->skip) continue;
        if (sys->bloom) {
            i32 e = 0, line_w;
            for (i = 0; i < L; i++) e += sig[i];
            prev_e = (prev_e * 123 / 128) + ((((max_e >> 1) - e) << 10) / max_e);
            line_w = (L * 112 / 128) + (prev_e >> 9);
            dx = (line_w << 12) / m->outw;
            scan_l = (u32) (((L / 2) - (line_w >> 1) + 8) << 12);
            f_lo = (i32) (scan_l >> 12);
            f_hi = (i32) (scan_r >> 12);
            if (k < first) continue;
        }
        memset(&ey, 0, sizeof(ey));
        memset(&ei, 0, sizeof(ei));
        memset(&eq, 0, sizeof(eq));
        memset(&fy, 0, sizeof(fy));
        memset(&fi, 0, sizeof(fi));
        memset(&fq, 0, sizeof(fq));
        for (i = f_lo; sys->conv && i < f_hi; i++) { /* crt_core.c:538-543 with the FIR eqf */
            yy[i] = wmul(fir_step(&fy, sig[i] + bright, sys->conv), 16);
            ii[i] = fir_step(&fi, wmul(sig[i], WAVE_I(i)) >> 9, sys->conv) >> 3;
            qq[i] = fir_step(&fq, wmul(sig[i], WAVE_Q(i)) >> 9, sys->conv) >> 3;
        }
        for (i = f_lo; !sys->conv && i < f_hi; i++) { /* crt_core.c:538-543 */
            yy[i] = eq_step(&ey, sys->eq[0], sig[i] + bright) * 16;
            ii[i] = eq_step(&ei, sys->eq[1], wmul(sig[i], WAVE_I(i)) >> 9) >> 3;
            qq[i] = eq_step(&eq, sys->eq[2], wmul(sig[i], WAVE_Q(i)) >> 9) >> 3;
        }
        px = m->out + (size_t) rec->beg * pitch;
        row_end = px + pitch;
        for (pos = scan_l; pos < scan_r && px < row_end; pos += (u32) dx, px += bpp) {
            i32 R = pos & 0xfff, Lw = 0xfff - R, s = (i32) (pos >> 12);
            i32 y = (wmul(yy[s], Lw) >> 2) + (wmul(yy[s + 1], R) >> 2); /* crt_core.c:568-570 */
            i32 ci = (wmul(ii[s], Lw) >> 14) + (wmul(ii[s + 1], R) >> 14);
            i32 cq = (wmul(qq[s], Lw) >> 14) + (wmul(qq[s + 1], R) >> 14);
            i32 r = wmul(wadd(wadd(y, wmul(3879, ci)), wmul(2556, cq)) >> 12, m->contrast) >> 8;
            i32 g = wmul(wsub(wsub(y, wmul(1126, ci)), wmul(2605, cq)) >> 12, m->contrast) >> 8;
            i32 b = wmul(wadd(wsub(y, wmul(4530, ci)), wmul(7021, cq)) >> 12, m->contrast) >> 8;
            i32 rgb;
            r = r < 0 ? 0 : (r > 255 ? 255 : r);
            g = g < 0 ? 0 : (g > 255 ? 255 : g);
            b = b < 0 ? 0 : (b > 255 ? 255 : b);
            rgb = r << 16 | g << 8 | b;
            if (m->blend) { /* crt_core.c:584-609 */
                i32 old = px[fmt_r[m->out_format]] << 16 | px[fmt_g[m->out_format]] << 8
                        | px[fmt_b[m->out_format]];
                rgb = ((rgb & 0xfefeff) >> 1) + ((old & 0xfefeff) >> 1);
            }
            px[fmt_r[m->out_format]] = (unsigned char) (rgb >> 16);
            px[fmt_g[m->out_format]] = (unsigned char) (rgb >> 8);
            px[fmt_b[m->out_format]] = (unsigned char) rgb;
            if (fmt_a[m->out_format] >= 0) px[fmt_a[m->out_format]] = 0xff;
        }
        for (row = rec->beg + 1; row < rec->end - m->scanlines; row++) /* crt_core.c:662-664 */
            memcpy(m->out + (size_t) row * pitch, m->out + (size_t) (row - 1) * pitch, (size_t) pitch);
    }
    free(yy);
}

void
ocrt_decode(const ocrt_sys *sys, ocrt_monitor *m, int noise, ocrt_rand *g)
{
    ocrt_line *table;
    if (ocrt_bpp(m->out_format) == 0) return; /* crt_core.c:312-315 */
    table = (ocrt_line *) calloc((size_t) sys->lines, sizeof(*table));
    ocrt_noise_pass(sys, m, noise, g);
    (void) ocrt_sync_pass(sys, m, table);
    ocrt_line_pass(sys, m, table, 0, sys->lines);
    free(table);
}
