/* include/crtx_batch.h -- device-resident batch interface (C89, plain pointers and sizes).
 *
 * An additive extension beside the drop-in calls of crt_b200.h: a context owns N
 * "monitors" -- N independent `struct CRT` instances (crt_core.h:74-92) whose signal
 * buffers (analog / inp), persistent decoder state (ccf / hsync / vsync / rn) and
 * per-line tables live in HBM.  One crtx_modulate + crtx_demodulate pair advances every
 * monitor by one field, exactly as one crt_modulate + crt_demodulate call pair on each of
 * N reference instances would (crt_ntsc.c:128, crt_nes.c:106, crt_ntscvhs.c:128,
 * crt_core.c:291), but as a handful of kernel launches for the whole batch, asynchronously
 * on the caller's CUDA stream.  Images are DEVICE pointers here; crtx_frames_host is the
 * host-buffer entry point (pinned staging + async copies inside the call).
 *
 * The library variant fixes the emulated system, as in the reference (compile-time
 * CRT_SYSTEM): query it with crtx_system().
 *
 * All functions return 0 on success, non-zero on failure (crtx_last_error() explains);
 * they never fall back to a CPU path.
 */
#ifndef CRTX_BATCH_H
#define CRTX_BATCH_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct crtx_ctx crtx_ctx;

/* the caller-settable part of struct CRT, plus crt_demodulate's `noise` argument */
typedef struct crtx_monitor {
    void *out; /* DEVICE image: outh rows of outw * bpp bytes, out_pitch bytes apart */
    int outw, outh, out_format;
    int hue, brightness, contrast, saturation;
    int black_point, white_point;
    int scanlines, blend;
    unsigned v_fac;
    int noise;
    int out_pitch; /* bytes between the starts of two output rows; 0 = dense (outw * bpp) */
} crtx_monitor;

/* struct NTSC_SETTINGS with the image on the DEVICE; fields a system lacks are ignored */
typedef struct crtx_source {
    const void *data; /* h rows, pitch bytes apart; RGB systems: w*bpp bytes per row; NES: w unsigned short */
    int format, w, h;
    int raw, as_color, field, frame;
    int hue, xoffset, yoffset;
    int do_aberration;    /* CRT_SYSTEM_NTSCVHS */
    int dot_crawl_offset; /* CRT_SYSTEM_NES, _NESRGB, _SNES, _TEMP, _PV1K */
    int reinit;           /* CRT_SYSTEM_NES: settings.field_initialized was 0 */
    int pitch;            /* bytes between the starts of two source rows; 0 = dense (w * bpp, NES w * 2) */
} crtx_source;

/* Row pitches.  A pitch of 0 means dense rows, which is what a zeroed struct gives.  Otherwise the pitch must be at
 * least the row's bytes (outw * bpp, w * bpp, NES w * 2) and positive; 4-byte pixel formats need a pitch that is a
 * multiple of 4 (as they need a 4-byte aligned image), NES sources an even one.  crtx_set_monitors, crtx_modulate and
 * crtx_frames_host reject anything else, name the monitor and the rule in crtx_last_error(), and leave the context as it
 * was.  No kernel writes a byte between the end of one row and the start of the next, so an image can be a window of a
 * larger buffer (a cudaMallocPitch allocation, a decoder surface, one tile of a mosaic).  The fast paths need rows that
 * start on 16-byte boundaries -- the image's address AND its pitch multiples of 16; other pitches take the general
 * paths, with the same results.  Only the crtx_modulate / crtx_demodulate / crtx_frames_host images have pitches:
 * the BMP / PPM wire kernels and crtx_fade_phosphors below work on dense arrays, whose layout the file formats and a
 * pixel count fix. */

/* the persistent decoder state of struct CRT */
typedef struct crtx_state {
    int ccf[5][5]; /* ccf[CRT_CC_VPER][CRT_CC_SAMPLES] of the variant in the top-left corner (5 x 5: the PV-1000) */
    int hsync, vsync;
    int rn;
} crtx_state;

/* what the sync pre-pass decided for one decoded scanline (diagnostics / tests) */
typedef struct crtx_line {
    int pos;        /* start of the 1-line decode window in inp[] (crt_core.c:452-454) */
    int wave0, wave1; /* hue-rotated carrier (crt_core.c:476-477); PV-1000: dci and dcq (crt_core.c:494-495) */
    int beg;        /* first output row, or -1 when the line is skipped (crt_core.c:431) */
    int end;        /* one past the last output row (crt_core.c:429,432) */
    int hsync;      /* after this line's search (crt_core.c:446) */
    int pad0, pad1;
} crtx_line;

/* geometry of this library variant */
int crtx_system(void);          /* CRT_SYSTEM */
int crtx_chroma_pattern(void);  /* CRT_CHROMA_PATTERN */
int crtx_hres(void);            /* CRT_HRES */
int crtx_input_size(void);      /* CRT_INPUT_SIZE */
int crtx_lines(void);           /* CRT_LINES */
int crtx_cc_vper(void);         /* CRT_CC_VPER */

int  crtx_create(crtx_ctx **ctx, int n_monitors); /* on the current CUDA device */
void crtx_destroy(crtx_ctx *ctx);

/* configuration and state; `m` / `s` are HOST arrays of `count` entries */
int crtx_set_monitors(crtx_ctx *ctx, int first, int count, const crtx_monitor *m);
int crtx_set_state(crtx_ctx *ctx, int first, int count, const crtx_state *s, void *stream);
int crtx_get_state(crtx_ctx *ctx, int first, int count, crtx_state *s, void *stream);
int crtx_seed(crtx_ctx *ctx, int first, int count, unsigned seed); /* VHS libc-rand() replica */

/* DEVICE pointers to monitor i's signal buffers (CRT_INPUT_SIZE + slack bytes each) */
signed char *crtx_analog(crtx_ctx *ctx, int i);
signed char *crtx_inp(crtx_ctx *ctx, int i);

/* copy monitor i's analog[] (which = 0) or inp[] (which = 1), CRT_INPUT_SIZE bytes, to / from a HOST
 * buffer; synchronises `stream` */
int crtx_read_signal(crtx_ctx *ctx, int i, int which, signed char *host, void *stream);
int crtx_write_signal(crtx_ctx *ctx, int i, int which, const signed char *host, void *stream);

/* one field for monitors [first, first+count); asynchronous on `stream` (a cudaStream_t) */
int crtx_modulate(crtx_ctx *ctx, int first, int count, const crtx_source *src, void *stream);
int crtx_demodulate(crtx_ctx *ctx, int first, int count, void *stream);

/* host-buffer entry point: src[i].data and out_host[i] are HOST pointers; moves the images in, runs modulate +
 * demodulate, moves the decoded images out, all on `stream`; the monitors' `out` must have been set to device images
 * of the right size.  The host images have the same pitches as the device ones: src[i].pitch for src[i].data, the
 * monitor's out_pitch for out_host[i] (and for its `out`).  out_host[i] is the monitor's PERSISTENT host image, like
 * the `out` buffer of the reference's struct CRT: with page-locked (crtx_host_alloc / cudaHostAlloc) images whose rows
 * start on 16-byte boundaries (address and pitch multiples of 16; a dense image whose rows are not a multiple of 16
 * bytes can get there by padding its rows), only the source rows the field reads (crt_ntsc.c:258-266) and only the
 * output rows it writes (crt_core.c:428-432, 662-664) cross PCIe, and every other row of out_host[i], and the padding
 * behind every row, keeps its bytes.  Pageable or unaligned images, and option "host_rows" 0, take whole-image copies
 * (of the rows' bytes only). */
int crtx_frames_host(crtx_ctx *ctx, int first, int count, const crtx_source *src,
                     void *const *out_host, void *stream);

/* Memory and stream helpers, so that a plain C89 caller (tools/crtx_video.c) needs no CUDA header:
 * device images, pinned host buffers, copies ordered on `stream` (0 = the default stream), and a
 * stream / device synchronise.  crtx_memcpy's kind: 0 host -> device, 1 device -> host, 2 device -> device. */
void *crtx_device_alloc(size_t bytes);   /* zero-filled; NULL on failure */
void  crtx_device_free(void *p);
void *crtx_host_alloc(size_t bytes);     /* page-locked; NULL on failure */
void  crtx_host_free(void *p);
int   crtx_memcpy(void *dst, const void *src, size_t bytes, int kind, void *stream);
int   crtx_memcmp_device(const void *a, const void *b, size_t bytes, int *differ, void *stream); /* synchronises */
int   crtx_sync(void *stream);

/* BMP wire format on the device (the subset bmp_rw.c reads and writes): `file_pixels` is the pixel array
 * exactly as it sits in the file after the 54-byte header -- rows bottom-up, each padded to 4 bytes.
 * unpack: 24 or 32 bits per pixel -> top-down BGRA with alpha 255 for 24-bit input (bmp_rw.c:22-94);
 * pack: top-down BGRA -> 32-bit bottom-up rows, what bmp_write24 stores (bmp_rw.c:96-146).  All pointers
 * are DEVICE pointers; asynchronous on `stream`. */
int crtx_bmp_unpack(void *bgra, const void *file_pixels, int w, int h, int bits, void *stream);
int crtx_bmp_pack(void *file_pixels, const void *bgra, int w, int h, void *stream);

/* PPM wire format on the device (what ppm_rw.c reads and writes): `file_pixels` is the P6 pixel data exactly as it
 * sits in the file after the header -- R, G, B bytes, rows top-down, no padding; `xrgb` are the loaders' int pixels
 * 0x00RRGGBB (= CRT_PIX_FORMAT_BGRA in memory).  unpack rescales a maximum colour value below 255 like ppm_rw.c:80;
 * pack drops the top byte (ppm_rw.c:113-118).  DEVICE pointers; asynchronous on `stream`. */
int crtx_ppm_unpack(void *xrgb, const void *file_pixels, int w, int h, int maxc, void *stream);
int crtx_ppm_pack(void *file_pixels, const void *xrgb, int w, int h, void *stream);

/* the live driver's phosphor decay (crt_main.c:437-452, run between frames when `fadephos` is on): every int pixel
 * c becomes (c>>1 & 0x7f7f7f) + (c>>2 & 0x3f3f3f) + (c>>3 & 0x1f1f1f) + (c>>4 & 0x0f0f0f), top byte cleared.
 * `image` is a DEVICE array of `npix` int pixels; asynchronous on `stream`. */
int crtx_fade_phosphors(void *image, size_t npix, void *stream);

/* per-kernel device timing.  After crtx_set_option(ctx, "timing", 1) every launch is bracketed by
 * CUDA events on its stream; crtx_get_timing synchronises, then reports the summed milliseconds and
 * the launch count of each kernel since the last call.  Index: 0 modulate skeleton (or the single
 * NES encoder kernel), 1 modulate picture, 2 noise pass, 3 sync pre-pass, 4 line kernel. */
#define CRTX_NUM_KERNELS 5
int crtx_get_timing(crtx_ctx *ctx, float *ms /* [CRTX_NUM_KERNELS] */, long *launches /* [CRTX_NUM_KERNELS] */);

/* diagnostics */
int crtx_get_lines(crtx_ctx *ctx, int i, crtx_line *table /* crtx_lines() entries */, void *stream);
long crtx_launch_count(crtx_ctx *ctx); /* kernels launched through this context so far */
long crtx_lines2_count(crtx_ctx *ctx); /* of those, line passes taken by k_lines2 (two monitors per CTA, tabulated resampler: the
                                         * stock IIR decoder on 4-byte pixels, 16-byte aligned rows, outw a multiple of 4 in about
                                         * [528, 1312]); every other geometry runs k_lines.  For tests and A/B runs (option "lines2"). */
/* which code paths monitors [first, first + count) took: paths[i] has CRTX_PATH_GENERIC_EQ set when the last demodulate's sync
 * pass put monitor first + i on the wrap-exact equaliser (its carrier or brightness is outside the fast equaliser's exact range,
 * or option "generic_eq" is on), and CRTX_PATH_STAGED_MOD when the last modulate encoded its picture with the staged encoder
 * (the source span of a 32-sample chunk fits a stage row) rather than the gather encoder, and CRTX_PATH_ROW16 when the line
 * pass writes its output rows with 16-byte stores (k_lines2, or the row path of k_lines / k_lines_fir: 4-byte pixels, outw a
 * multiple of 4, the image's address and out_pitch multiples of 16; never in the bloom build) rather than pixel by pixel.
 * Synchronises `stream`. */
#define CRTX_PATH_GENERIC_EQ 1
#define CRTX_PATH_STAGED_MOD 2
#define CRTX_PATH_ROW16 4
int crtx_get_paths(crtx_ctx *ctx, int first, int count, int *paths, void *stream);
/* options: "generic_eq", "timing", "mod_staged", "lines2", "host_rows" (0/1 switches), "host_src" (1:
 * crtx_frames_host lets the encoder read page-locked source images in place instead of copying them), and
 * "line_lo" / "line_hi": crtx_demodulate's line pass only decodes scanlines [line_lo, line_hi) of every
 * field (sync search and noise still cover the whole field).  This is the scanline-block partition of
 * ONE image across GPUs (fields of one image depend on each other through the blend, crt_core.c:584-608,
 * so they cannot be spread over ranks): every rank runs the same calls with its own block and owns the
 * output rows those lines write; see ntsc-crt_b200/sharding.py. */
int crtx_set_option(crtx_ctx *ctx, const char *name, int value);
const char *crtx_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
