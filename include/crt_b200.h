/* include/crt_b200.h -- the drop-in boundary (C89).
 *
 * Byte-identical replacement for the reference's public interface of the hot path:
 *   struct CRT            crt_core.h:74-92
 *   struct NTSC_SETTINGS  crt_ntsc.h:111-124 / crt_ntscvhs.h:133-147 / crt_nes.h:132-143
 *   crt_init, crt_resize, crt_reset, crt_modulate, crt_demodulate,
 *   crt_bpp4fmt, crt_sincos14          crt_core.h:100-139
 * so the reference's unmodified C89 drivers (crt_main.c, extra/video_convert.c) compile
 * against it and link with lib/libcrt_b200_<variant>.so instead of crt_core.c + crt_<sys>.c
 * (see INTEGRATION.md).  Behind these entry points the work is done by sm_90a CUDA
 * kernels; there is no CPU implementation in the library.
 *
 * Like the reference, the interface is compile-time polymorphic: define CRT_SYSTEM
 * (and, for the NES, CRT_CHROMA_PATTERN) exactly as you would for the reference, and
 * link the matching library variant:
 *      CRT_SYSTEM 0                          libcrt_b200_ntsc.so
 *      CRT_SYSTEM 5                          libcrt_b200_vhs.so
 *      CRT_SYSTEM 1 (CRT_CHROMA_PATTERN 2)   libcrt_b200_nes.so
 *      CRT_SYSTEM 1, CRT_CHROMA_PATTERN 0    libcrt_b200_nes_p0.so
 *      CRT_SYSTEM 1, CRT_CHROMA_PATTERN 1    libcrt_b200_nes_p1.so
 *      CRT_SYSTEM 3                          libcrt_b200_snes.so
 *      CRT_SYSTEM 6 (CRT_CHROMA_PATTERN 2)   libcrt_b200_nesrgb.so
 *      CRT_SYSTEM 6, CRT_CHROMA_PATTERN 0 / 1  libcrt_b200_nesrgb_p0.so / libcrt_b200_nesrgb_p1.so
 *      CRT_SYSTEM 4                          libcrt_b200_template.so
 *      CRT_SYSTEM 2                          libcrt_b200_pv1k.so
 *      CRT_SYSTEM 0, CRT_DO_BLOOM 1          libcrt_b200_ntsc_bloom.so
 * (and libcrt_b200_ntsc_conv{,6,5,4}.so for the USE_CONVOLUTION builds of crt_core.c:85-88)
 */
#ifndef CRT_B200_H
#define CRT_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define CRT_MAJOR 2 /* interface level of the reference we mirror (crt_core.h:25-27) */
#define CRT_MINOR 3
#define CRT_PATCH 2

/* crt_core.h:30-36 */
#define CRT_SYSTEM_NTSC    0
#define CRT_SYSTEM_NES     1
#define CRT_SYSTEM_PV1K    2
#define CRT_SYSTEM_SNES    3
#define CRT_SYSTEM_TEMP    4
#define CRT_SYSTEM_NTSCVHS 5
#define CRT_SYSTEM_NESRGB  6

#ifndef CRT_SYSTEM
#define CRT_SYSTEM CRT_SYSTEM_NTSC
#endif

/* crt_core.h:62-67 */
#define CRT_PIX_FORMAT_RGB  0
#define CRT_PIX_FORMAT_BGR  1
#define CRT_PIX_FORMAT_ARGB 2
#define CRT_PIX_FORMAT_RGBA 3
#define CRT_PIX_FORMAT_ABGR 4
#define CRT_PIX_FORMAT_BGRA 5

#if (CRT_SYSTEM == CRT_SYSTEM_PV1K)
#define CRT_CB_FREQ    5 /* crt_pv1k.h:41,49: five samples per chroma period */
#define CRT_CC_SAMPLES 5
#else
#define CRT_CB_FREQ    4
#define CRT_CC_SAMPLES 4
#endif
#define CRT_VRES       262
#define CB_CYCLES      10
#define L_FREQ         1431818
#define LINE_BEG       0
#define CRT_HSYNC_THRESH 4
#define CRT_VSYNC_THRESH 94
#define BLANK_LEVEL    0

#if (CRT_SYSTEM == CRT_SYSTEM_NTSC) || (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
/* ---- composite NTSC timing, crt_ntsc.h:25-109 / crt_ntscvhs.h:25-131 ---- */
#define CRT_CHROMA_PATTERN 1
#define CRT_CC_LINE  2275
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 10)
#define CRT_TOP      21
#define CRT_BOT      261
#define CRT_CC_VPER  1
#define CRT_HSYNC_WINDOW 8
#define CRT_VSYNC_WINDOW 8
#define CRT_B200_LINE_UNITS (1500 + 4700 + 600 + 2500 + 1600 + 52600) /* ns */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define SYNC_BEG     CRT_B200_POS(1500)
#define BW_BEG       CRT_B200_POS(1500 + 4700)
#define CB_BEG       CRT_B200_POS(1500 + 4700 + 600)
#define BP_BEG       CRT_B200_POS(1500 + 4700 + 600 + 2500)
#define AV_BEG       CRT_B200_POS(1500 + 4700 + 600 + 2500 + 1600)
#define AV_LEN       CRT_B200_POS(52600)
#define WHITE_LEVEL  100
#define BURST_LEVEL  20
#define BLACK_LEVEL  7
#define SYNC_LEVEL   (-40)
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
#define CRT_VHS_NOISE 1
#endif

struct NTSC_SETTINGS {
    const unsigned char *data; /* image, one of the CRT_PIX_FORMATs */
    int format;
    int w, h;
    int raw;      /* 1 = do not scale to the active picture area */
    int as_color; /* 0 = monochrome */
    int field;    /* 0 even / 1 odd */
    int frame;    /* 0 even / 1 odd */
    int hue;      /* 0..359 */
    int xoffset;  /* samples */
    int yoffset;  /* lines */
#if (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
    int do_aberration; /* bottom-of-frame head-switching loss of sync */
#endif
    int iirs_initialized; /* zero the struct before first use */
};

#elif (CRT_SYSTEM == CRT_SYSTEM_NES)
/* ---- NES PPU timing, crt_nes.h:30-130 ---- */
#ifndef CRT_CHROMA_PATTERN
#define CRT_CHROMA_PATTERN 2
#endif
#if (CRT_CHROMA_PATTERN == 1)
#define CRT_CC_LINE 2275
#elif (CRT_CHROMA_PATTERN == 2)
#define CRT_CC_LINE 2273
#else
#define CRT_CC_LINE 2280
#endif
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 10)
#define CRT_TOP      15
#define CRT_BOT      255
#define CRT_CC_VPER  3
#define CRT_HSYNC_WINDOW 6
#define CRT_VSYNC_WINDOW 6
#define CRT_B200_LINE_UNITS 341 /* PPU pixels */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define PPUpx2pos(u) CRT_B200_POS(u)
#define SYNC_BEG     CRT_B200_POS(9)
#define BW_BEG       CRT_B200_POS(9 + 25)
#define CB_BEG       CRT_B200_POS(9 + 25 + 4)
#define BP_BEG       CRT_B200_POS(9 + 25 + 4 + 15)
#define LAV_BEG      CRT_B200_POS(9 + 25 + 4 + 15 + 5)
#define AV_BEG       CRT_B200_POS(9 + 25 + 4 + 15 + 5 + 1 + 15)
#define AV_LEN       CRT_B200_POS(256)
#define WHITE_LEVEL  110
#define BURST_LEVEL  30
#define BLACK_LEVEL  0
#define SYNC_LEVEL   (-37)

struct NTSC_SETTINGS {
    const unsigned short *data; /* 6- or 9-bit PPU pixels */
    int w, h;
    unsigned int border_color;
    int dot_crawl_offset; /* 0, 1, 2 */
    int hue;
    int xoffset;
    int yoffset;
    int field_initialized; /* zero the struct before first use */
};

#elif (CRT_SYSTEM == CRT_SYSTEM_SNES)
/* ---- SNES timing, crt_snes.h:20-139: NES line layout, RGB source, no encoder band-limit ---- */
#define CRT_CC_LINE  2273
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 10)
#define CRT_TOP      15
#define CRT_BOT      255
#define CRT_CC_VPER  3
#define CRT_HSYNC_WINDOW 6
#define CRT_VSYNC_WINDOW 6
#define CRT_B200_LINE_UNITS 341 /* PPU pixels */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define PPUpx2pos(u) CRT_B200_POS(u)
#define SYNC_BEG     CRT_B200_POS(9)
#define BW_BEG       CRT_B200_POS(9 + 25)
#define CB_BEG       CRT_B200_POS(9 + 25 + 4)
#define BP_BEG       CRT_B200_POS(9 + 25 + 4 + 15)
#define LAV_BEG      CRT_B200_POS(9 + 25 + 4 + 15 + 5)
#define AV_BEG       CRT_B200_POS(9 + 25 + 4 + 15 + 5 + 1 + 15)
#define AV_LEN       CRT_B200_POS(256)
#define WHITE_LEVEL  100
#define BURST_LEVEL  20
#define BLACK_LEVEL  7
#define SYNC_LEVEL   (-40)
#define CRT_DO_BANDLIMITING 0

struct NTSC_SETTINGS {
    const unsigned char *data; /* image, one of the CRT_PIX_FORMATs */
    int format;
    int w, h;
    int raw;      /* 1 = do not scale to the active picture area */
    int as_color; /* 0 = monochrome */
    int field;    /* unused */
    int frame;    /* unused */
    int hue;      /* 0..359 */
    int xoffset;  /* samples */
    int yoffset;  /* lines */
    int dot_crawl_offset; /* 0..3 */
    int iirs_initialized; /* zero the struct before first use */
};

#elif (CRT_SYSTEM == CRT_SYSTEM_NESRGB)
/* ---- RGB image with NES timing and artifacts, crt_nesrgb.h (chroma patterns as for the NES, crt_nesrgb.h:27-40) ---- */
#ifndef CRT_CHROMA_PATTERN
#define CRT_CHROMA_PATTERN 2
#endif
#if (CRT_CHROMA_PATTERN == 1)
#define CRT_CC_LINE 2275
#elif (CRT_CHROMA_PATTERN == 2)
#define CRT_CC_LINE 2273
#else
#define CRT_CC_LINE 2280
#endif
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 10)
#define CRT_TOP      15
#define CRT_BOT      255
#define CRT_CC_VPER  3
#define CRT_HSYNC_WINDOW 6
#define CRT_VSYNC_WINDOW 6
#define CRT_B200_LINE_UNITS 341 /* PPU pixels */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define PPUpx2pos(u) CRT_B200_POS(u)
#define SYNC_BEG     CRT_B200_POS(9)
#define BW_BEG       CRT_B200_POS(9 + 25)
#define CB_BEG       CRT_B200_POS(9 + 25 + 4)
#define BP_BEG       CRT_B200_POS(9 + 25 + 4 + 15)
#define LAV_BEG      CRT_B200_POS(9 + 25 + 4 + 15 + 5)
#define AV_BEG       CRT_B200_POS(9 + 25 + 4 + 15 + 5 + 1 + 15)
#define AV_LEN       CRT_B200_POS(256)
#define WHITE_LEVEL  100
#define BURST_LEVEL  30
#define BLACK_LEVEL  0
#define SYNC_LEVEL   (-37)

struct NTSC_SETTINGS {
    const unsigned char *data; /* image, one of the CRT_PIX_FORMATs */
    int format;
    int w, h;
    int dot_crawl_offset; /* 0, 1, 2 */
    int hue;
    int xoffset;
    int yoffset;
    int field_initialized; /* zero the struct before first use */
};

#elif (CRT_SYSTEM == CRT_SYSTEM_TEMP)
/* ---- the reference's worked example for new systems, crt_template.h:22-175: composite NTSC timing, a 2-line
 * chroma cycle walked by dot_crawl_offset, band-limited RGB encoder ---- */
#define CRT_CC_LINE  2275
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 10)
#define CRT_TOP      21
#define CRT_BOT      261
#define CRT_CC_VPER  2
#define CRT_HSYNC_WINDOW 8
#define CRT_VSYNC_WINDOW 8
#define CRT_B200_LINE_UNITS (1500 + 4700 + 600 + 2500 + 1600 + 52600) /* ns */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define ns2pos(u)    CRT_B200_POS(u)
#define SYNC_BEG     CRT_B200_POS(1500)
#define BW_BEG       CRT_B200_POS(1500 + 4700)
#define CB_BEG       CRT_B200_POS(1500 + 4700 + 600)
#define BP_BEG       CRT_B200_POS(1500 + 4700 + 600 + 2500)
#define AV_BEG       CRT_B200_POS(1500 + 4700 + 600 + 2500 + 1600)
#define AV_LEN       CRT_B200_POS(52600)
#define WHITE_LEVEL  100
#define BURST_LEVEL  20
#define BLACK_LEVEL  7
#define SYNC_LEVEL   (-40)
#define CRT_DO_BANDLIMITING 1
#define Q_OFFSET     (-90) /* crt_template.h:139 */
#define HUE_OFFSET   (-60) /* crt_template.h:142 */

struct NTSC_SETTINGS {
    const unsigned char *data; /* image, one of the CRT_PIX_FORMATs */
    int format;
    int w, h;
    int raw;      /* 1 = do not scale to the active picture area */
    int as_color; /* 0 = monochrome */
    int field;    /* 0 even / 1 odd */
    int frame;    /* 0 even / 1 odd (unused by this encoder) */
    int hue;      /* 0..359 */
    int xoffset;  /* samples */
    int yoffset;  /* lines */
    int dot_crawl_offset; /* 0..5 */
    int iirs_initialized; /* zero the struct before first use */
};

#elif (CRT_SYSTEM == CRT_SYSTEM_PV1K)
/* ---- Casio PV-1000, crt_pv1k.h:36-151: 1920 samples per line, FIVE samples per chroma period, a 5-line chroma
 * cycle walked by dot_crawl_offset, band-limited RGB encoder ---- */
#define CRT_CC_LINE  2304
#define CRT_HRES     (CRT_CC_LINE * CRT_CB_FREQ / 6)
#define CRT_TOP      21
#define CRT_BOT      261
#define CRT_CC_VPER  5
#define CRT_HSYNC_WINDOW 8
#define CRT_VSYNC_WINDOW 8
#define DOT_ns       223
#define DOTx4_ns     892
#define CRT_B200_LINE_UNITS ((3 + 3 + 2 + 4 + 4 + 55) * DOTx4_ns) /* ns */
#define CRT_B200_POS(u) ((u) * CRT_HRES / CRT_B200_LINE_UNITS)
#define ns2pos(u)    CRT_B200_POS(u)
#define SYNC_BEG     CRT_B200_POS(3 * DOTx4_ns)
#define BW_BEG       CRT_B200_POS((3 + 3) * DOTx4_ns)
#define CB_BEG       CRT_B200_POS((3 + 3 + 2) * DOTx4_ns)
#define BP_BEG       CRT_B200_POS((3 + 3 + 2 + 4) * DOTx4_ns)
#define AV_BEG       CRT_B200_POS((3 + 3 + 2 + 4 + 4) * DOTx4_ns)
#define AV_LEN       CRT_B200_POS(55 * DOTx4_ns)
#define WHITE_LEVEL  100
#define BURST_LEVEL  20
#define BLACK_LEVEL  7
#define SYNC_LEVEL   (-40)

struct NTSC_SETTINGS {
    const unsigned char *data; /* image, one of the CRT_PIX_FORMATs */
    int format;
    int w, h;
    int raw;      /* 1 = do not scale to the active picture area */
    int as_color; /* 0 = monochrome */
    int field;    /* 0 even / 1 odd */
    int frame;    /* 0 even / 1 odd (unused by this encoder) */
    int hue;      /* 0..359 */
    int xoffset;  /* samples */
    int yoffset;  /* lines */
    int dot_crawl_offset; /* 0..5 */
    int iirs_initialized; /* zero the struct before first use */
};

#else
#error "crt_b200: unknown CRT_SYSTEM (0 NTSC, 1 NES, 2 PV1K, 3 SNES, 4 TEMP, 5 NTSCVHS, 6 NESRGB)"
#endif

#define CRT_INPUT_SIZE (CRT_HRES * CRT_VRES)
#define CRT_LINES      (CRT_BOT - CRT_TOP)

/* crt_core.h:70 (an unguarded #define there): beam-energy dependent line width.  Compile the caller with
 * -DCRT_DO_BLOOM=1 and link libcrt_b200_ntsc_bloom.so, the build of the library with the option on. */
#ifndef CRT_DO_BLOOM
#define CRT_DO_BLOOM 0
#endif
#define CRT_DO_VSYNC 1
#define CRT_DO_HSYNC 1

struct CRT {
    signed char analog[CRT_INPUT_SIZE]; /* encoder output (host mirror, kept coherent) */
    signed char inp[CRT_INPUT_SIZE];    /* decoder input after noise (host mirror)     */

    int outw, outh;
    int out_format;
    unsigned char *out; /* caller-owned host image */

    int hue, brightness, contrast, saturation;
    int black_point, white_point;
    int scanlines;
    int blend;
    unsigned v_fac;

    int ccf[CRT_CC_VPER][CRT_CC_SAMPLES];
    int hsync, vsync;
    int rn;
};

extern void crt_init(struct CRT *v, int w, int h, int f, unsigned char *out);
extern void crt_resize(struct CRT *v, int w, int h, int f, unsigned char *out);
extern void crt_reset(struct CRT *v);
extern void crt_modulate(struct CRT *v, struct NTSC_SETTINGS *s);
extern void crt_demodulate(struct CRT *v, int noise);
extern int  crt_bpp4fmt(int format);

#define T14_2PI  16384
#define T14_MASK (T14_2PI - 1)
#define T14_PI   (T14_2PI / 2)
extern void crt_sincos14(int *s, int *c, int n);

#ifdef __cplusplus
}
#endif
#endif
