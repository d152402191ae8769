/* tools/crtx_video.c -- batch video driver over the crtx_* interface (C89).
 *
 * Same job, arguments and files as the reference's extra/video_convert.c (frames/%06d.bmp in,
 * output/%06d.bmp out, one crt_modulate + crt_demodulate pair per image, blend 0, the field
 * toggling every image and the frame parity every other one, video_convert.c:226-277), and the
 * same pixels -- but the sequence is cut into SEGMENTS that advance side by side, one monitor of
 * a crtx context each, so every step decodes `segments` images in a handful of kernel launches.
 *
 * What the sequential loop carries from image to image, and how each piece is handled:
 *   rn (noise LCG)       closed form: image f starts from rn0 advanced CRT_INPUT_SIZE * f steps
 *                        (crt_core.c:359, 367)
 *   hsync, vsync         speculated from a 4-image probe, then VERIFIED against what the preceding
 *                        segment really ended with
 *   ccf (burst lock)     re-primed by every crt_modulate (crt_ntsc.c:325-329)
 *   the output buffer    never cleared, a field rewrites only its own rows: every segment first
 *                        decodes the two images before its own ("halo"); the buffer it then holds
 *                        must equal the preceding segment's last image, which is verified too
 * File bytes travel as they are stored: the pixel array of each BMP goes to the device unchanged and is
 * unpacked there (crtx_bmp_unpack), decoded images are packed into the writer's layout on the device too.
 * File I/O overlaps the device: while step t runs, one thread reads the files of step t + 1 into the other set of
 * page-locked buffers and another writes the images of step t - 1 (only the main thread talks to the library).
 * A segment that fails verification is decoded again, sequentially, from the true state; its
 * files are rewritten.  The result is what the sequential loop writes (tests/test_gpu_video_driver.py).
 *
 * Linked against the VHS library (crtx_system() says so at run time) it is video_convert.c's VHS build.  There the
 * noise comes from rand(): the sequence is srand(seed) followed by the loop, and every segment's generator is made
 * exact from the seed (crtx_seed, then crtx_skip_fields to its first image), saved after the halo and restored when
 * the segment is redone.  hsync is reset by every crt_modulate of that build (crt_ntscvhs.c:259), so only vsync and
 * the image are verified.
 *
 *   cc -std=c89 -O2 -pthread -I../include crtx_video.c -L../ntsc-crt_b200/lib -lcrt_b200_ntsc -o crtx_video
 *   ./crtx_video [-m] [-p] [-a] [-s] [-S segments] [-R seed] num_frames outwidth outheight noise
 * (-m monochrome, -p progressive, -s no scanlines: the letters of video_convert.c's option word; -a is no scanlines
 * too, except on the VHS build, where it draws the aberration as video_convert.c's -a does.  -R: the rand() seed of
 * the VHS build, time(0) by default as in video_convert.c:218; the seed used is printed.)
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "crtx_batch.h"

#define PIX_BGRA 5 /* CRT_PIX_FORMAT_BGRA, crt_core.h:67 */
#define SYSTEM_NTSCVHS 5 /* CRT_SYSTEM_NTSCVHS, crt_core.h:35 */

/* 1 for crtx_video_vhs (tools/Makefile): the generator calls of crtx_batch.h are linked in, and used when the library
 * says at run time that it is the VHS build.  The NTSC binary references none of them. */
#ifndef CRTX_VIDEO_VHS
#define CRTX_VIDEO_VHS 0
#endif

static void
die(const char *what)
{
    fprintf(stderr, "crtx_video: %s (%s)\n", what, crtx_last_error());
    exit(EXIT_FAILURE);
}

#define TRY(call) do { if ((call) != 0) die(#call); } while (0)

/* ---- BMP, the subset bmp_rw.c reads and writes: 54-byte header, 24 or 32 bits per pixel in,
 * 32 out, rows bottom-up, rows padded to 4 bytes (bmp_rw.c:22-146) ---- */
static unsigned
le32(const unsigned char *p)
{
    return (unsigned) p[0] | ((unsigned) p[1] << 8) | ((unsigned) p[2] << 16) | ((unsigned) p[3] << 24);
}

/* reads the pixel array of `file` (as stored: bottom-up, padded rows) into dst; returns 0 on failure */
static int
bmp_load(const char *file, unsigned char *dst, size_t cap, int *w, int *h, int *bits)
{
    FILE *f = fopen(file, "rb");
    unsigned char header[54];
    unsigned width, height, bytespp, rowbytes;
    size_t need;
    if (f == NULL) return 0;
    if (fread(header, 1, 54, f) != 54) {
        fclose(f);
        return 0;
    }
    width = le32(header + 18);
    height = le32(header + 22);
    bytespp = (le32(header + 28) & 0xff) / 8;
    rowbytes = width * bytespp + ((4 - (width * bytespp) % 4) % 4);
    need = (size_t) rowbytes * height;
    if ((bytespp != 3 && bytespp != 4) || width == 0 || height == 0 || need > cap || fread(dst, 1, need, f) != need) {
        fclose(f);
        return 0;
    }
    fclose(f);
    *w = (int) width;
    *h = (int) height;
    *bits = (int) bytespp * 8;
    return 1;
}

/* writes the 54-byte header bmp_rw.c:96-146 writes, then the (already bottom-up, 32-bit) pixel array */
static int
bmp_save(const char *file, const unsigned char *file_pixels, int w, int h)
{
    FILE *f;
    unsigned char head[54];
    unsigned filesize = 14 + 40 + (unsigned) w * (unsigned) h * 4;
    memset(head, 0, sizeof(head));
    head[0] = 'B';
    head[1] = 'M';
    head[2] = (unsigned char) filesize;
    head[3] = (unsigned char) (filesize >> 8);
    head[4] = (unsigned char) (filesize >> 16);
    head[5] = (unsigned char) (filesize >> 24);
    head[10] = 14 + 40;
    head[14] = 40;
    head[18] = (unsigned char) w;
    head[19] = (unsigned char) (w >> 8);
    head[20] = (unsigned char) (w >> 16);
    head[21] = (unsigned char) (w >> 24);
    head[22] = (unsigned char) h;
    head[23] = (unsigned char) (h >> 8);
    head[24] = (unsigned char) (h >> 16);
    head[25] = (unsigned char) (h >> 24);
    head[26] = 1;
    head[28] = 32;
    f = fopen(file, "wb");
    if (f == NULL) return 0;
    fwrite(head, 1, 54, f);
    fwrite(file_pixels, 4, (size_t) w * (size_t) h, f);
    fclose(f);
    return 1;
}

/* ---- the VHS build's rand() replica: seed, skip to each segment's first image, save and restore ---- */
#if CRTX_VIDEO_VHS
static int build_is_vhs(void) { return crtx_system() == SYSTEM_NTSCVHS; }
static void rand_seed(crtx_ctx *c, int n, unsigned seed) { TRY(crtx_seed(c, 0, n, seed)); }
static void rand_skip(crtx_ctx *c, int n, const int *fields, int ab) { TRY(crtx_skip_fields(c, 0, n, fields, ab, NULL)); }
static void rand_get(crtx_ctx *c, int n, unsigned *words) { TRY(crtx_get_rand(c, 0, n, words, NULL)); }
static void rand_set(crtx_ctx *c, int i, const unsigned *words) { TRY(crtx_set_rand(c, i, 1, words, NULL)); }
#else
static int build_is_vhs(void) { return 0; }
static void rand_seed(crtx_ctx *c, int n, unsigned seed) { (void) c; (void) n; (void) seed; }
static void rand_skip(crtx_ctx *c, int n, const int *fields, int ab) { (void) c; (void) n; (void) fields; (void) ab; }
static void rand_get(crtx_ctx *c, int n, unsigned *words) { (void) c; (void) n; (void) words; }
static void rand_set(crtx_ctx *c, int i, const unsigned *words) { (void) c; (void) i; (void) words; }
#endif

/* ---- n steps of rn = 214019 * rn + 140327895 (crt_core.c:359) as one multiply-add ---- */
static unsigned
lcg_advance(unsigned rn, unsigned long n)
{
    unsigned am = 214019u, ac = 140327895u, rm = 1u, rc = 0u;
    while (n) {
        if (n & 1) {
            rc = (rc * am + ac) & 0xffffffffu;
            rm = (rm * am) & 0xffffffffu;
        }
        ac = (ac * am + ac) & 0xffffffffu;
        am = (am * am) & 0xffffffffu;
        n >>= 1;
    }
    return (rn * rm + rc) & 0xffffffffu;
}

static int
as_int32(unsigned v)
{
    return (v & 0x80000000u) ? -(int) ((~v + 1u) & 0xffffffffu) : (int) v;
}

/* contiguous split of n items over `parts`: item range of part p, earlier parts one longer */
static void
span_of(int n, int p, int parts, int *lo, int *hi)
{
    int base = n / parts, extra = n % parts;
    *lo = p * base + (p < extra ? p : extra);
    *hi = *lo + base + (p < extra ? 1 : 0);
}

struct job {
    int n;              /* images: files 1 .. n, image index f = file number - 1 */
    int outw, outh, noise;
    int color, progressive, scanlines;
    int vhs, aberration; /* VHS build; its -a */
    int w, h;           /* source size (all images alike) */
    int bits;           /* of the source files: 24 or 32 */
    size_t src_bytes, out_bytes, file_bytes; /* device image, device output, source pixel array as stored */
};

static void
parity_of(const struct job *j, int f, int *field, int *frame)
{
    if (j->progressive) {
        *field = 0;
        *frame = 0;
    } else { /* video_convert.c:261-267 */
        *field = f & 1;
        *frame = (f >> 1) & 1;
    }
}

static void
load_image(struct job *j, int f, unsigned char *host)
{
    char name[64];
    int w, h, bits;
    sprintf(name, "frames/%06d.bmp", f + 1);
    if (!bmp_load(name, host, j->file_bytes, &w, &h, &bits) || w != j->w || h != j->h || bits != j->bits) {
        fprintf(stderr, "crtx_video: unable to read image %s (all images must be %dx%d, %d bits)\n", name, j->w, j->h, j->bits);
        exit(EXIT_FAILURE);
    }
}

static void
save_image(const struct job *j, int f, const unsigned char *host)
{
    char name[64];
    sprintf(name, "output/%06d.bmp", f + 1);
    if (!bmp_save(name, host, j->outw, j->outh)) {
        fprintf(stderr, "crtx_video: unable to write image %s\n", name);
        exit(EXIT_FAILURE);
    }
}

/* file -> pinned host (pixel array as stored) -> device -> top-down BGRA on the device; asynchronous */
static void
stage_image(struct job *j, int f, unsigned char *host, void *dev_file, void *dev_bgra)
{
    load_image(j, f, host);
    TRY(crtx_memcpy(dev_file, host, j->file_bytes, 0, NULL));
    TRY(crtx_bmp_unpack(dev_bgra, dev_file, j->w, j->h, j->bits, NULL));
}

/* decoded device image -> bottom-up 32-bit rows on the device -> pinned host; asynchronous */
static void
fetch_image(const struct job *j, const void *dev_bgra, void *dev_file, unsigned char *host)
{
    TRY(crtx_bmp_pack(dev_file, dev_bgra, j->outw, j->outh, NULL));
    TRY(crtx_memcpy(host, dev_file, j->out_bytes, 1, NULL));
}

/* ---- file I/O of one step on its own thread: `count` images read into / written from page-locked buffers ---- */
struct io_batch {
    struct job *j;
    int count, write, running;
    int *frame;
    unsigned char **buf;
    pthread_t th;
};

static void *
io_main(void *arg)
{
    struct io_batch *b = (struct io_batch *) arg;
    int i;
    for (i = 0; i < b->count; i++) {
        if (b->write) save_image(b->j, b->frame[i], b->buf[i]);
        else load_image(b->j, b->frame[i], b->buf[i]);
    }
    return NULL;
}

static void
io_start(struct io_batch *b)
{
    if (b->count == 0) return;
    if (pthread_create(&b->th, NULL, io_main, b) != 0) { /* no thread: do it here */
        io_main(b);
        return;
    }
    b->running = 1;
}

static void
io_join(struct io_batch *b)
{
    if (b->running) pthread_join(b->th, NULL);
    b->running = 0;
}

static void
fill_source(const struct job *j, crtx_source *s, const void *dev, int f)
{
    memset(s, 0, sizeof(*s)); /* raw, hue, offsets 0 as video_convert.c:231-236 intends */
    s->data = dev;
    s->format = PIX_BGRA;
    s->w = j->w;
    s->h = j->h;
    s->as_color = j->color;
    s->do_aberration = j->aberration;
    parity_of(j, f, &s->field, &s->frame);
}

int
main(int argc, char **argv)
{
    struct job j;
    int segments = 64, a = 1, S, s, t, longest, recomputed = 0;
    int *lo, *hi;
    crtx_ctx *ctx, *probe;
    crtx_monitor *mons;
    crtx_source *srcs;
    crtx_state *st, *st_halo, *fin;
    unsigned char **hsrc, **hout, **hsrc2, **hout2; /* two sets of staging buffers: [s] and [S + s] */
    struct io_batch rd[2], wr[2];
    void **dsrc, **draw, **dfile, **work, **halo;
    int after_hs[2], after_vs[2], have_after[2];
    unsigned rn0 = 194u; /* crt_init, crt_core.c:269 */
    unsigned seed = (unsigned) time(0);
    unsigned *rand_halo = NULL; /* VHS: every segment's generator after its halo, CRTX_RAND_WORDS words each */
    int *skip = NULL;
    char name[64];

    memset(&j, 0, sizeof(j));
    j.color = 1;
    j.scanlines = 1;
    j.vhs = build_is_vhs();
    while (a < argc && argv[a][0] == '-') {
        const char *o = argv[a] + 1;
        if (*o == 'S' && a + 1 < argc) {
            segments = atoi(argv[a + 1]);
            a += 2;
            continue;
        }
        if (*o == 'R' && a + 1 < argc) {
            seed = (unsigned) strtoul(argv[a + 1], NULL, 0);
            a += 2;
            continue;
        }
        for (; *o; o++) {
            if (*o == 'm') j.color = 0;
            else if (*o == 'p') j.progressive = 1;
            else if (*o == 's') j.scanlines = 0;
            else if (*o == 'a' && j.vhs) j.aberration = 1;
            else if (*o == 'a') j.scanlines = 0;
            else if (*o != 'o') {
                fprintf(stderr, "crtx_video: unknown option -%c\n", *o);
                return EXIT_FAILURE;
            }
        }
        a++;
    }
    if (argc - a < 4) {
        fprintf(stderr, "usage: %s [-m] [-p] [-a] [-s] [-S segments] [-R seed] num_frames outwidth outheight noise\n", argv[0]);
        return EXIT_FAILURE;
    }
    j.n = atoi(argv[a]) - 1; /* the reference converts files 1 .. num_frames - 1 (video_convert.c:246) */
    j.outw = atoi(argv[a + 1]);
    j.outh = atoi(argv[a + 2]);
    j.noise = atoi(argv[a + 3]);
    if (j.noise < 0) j.noise = 0;
    if (j.n <= 0 || j.outw <= 0 || j.outh <= 0 || segments <= 0) {
        fprintf(stderr, "crtx_video: num_frames must be > 1, sizes and segments > 0\n");
        return EXIT_FAILURE;
    }

    { /* the first image fixes the source size */
        FILE *f;
        unsigned char header[54];
        sprintf(name, "frames/%06d.bmp", 1);
        f = fopen(name, "rb");
        if (f == NULL || fread(header, 1, 54, f) != 54) {
            fprintf(stderr, "crtx_video: unable to read image %s\n", name);
            return EXIT_FAILURE;
        }
        fclose(f);
        j.w = (int) le32(header + 18);
        j.h = (int) le32(header + 22);
        j.bits = (int) (le32(header + 28) & 0xff);
        if (j.w <= 0 || j.h <= 0 || (j.bits != 24 && j.bits != 32)) {
            fprintf(stderr, "crtx_video: %s is not a 24- or 32-bit BMP\n", name);
            return EXIT_FAILURE;
        }
    }
    j.src_bytes = (size_t) j.w * j.h * 4;
    j.file_bytes = (size_t) ((j.w * (j.bits / 8) + 3) & ~3) * j.h;
    j.out_bytes = (size_t) j.outw * j.outh * 4;

    S = segments < j.n ? segments : j.n;
    lo = (int *) malloc(sizeof(int) * S);
    hi = (int *) malloc(sizeof(int) * S);
    skip = (int *) malloc(sizeof(int) * S);
    rand_halo = (unsigned *) malloc(sizeof(unsigned) * CRTX_RAND_WORDS * S);
    mons = (crtx_monitor *) calloc(S, sizeof(*mons));
    srcs = (crtx_source *) calloc(S, sizeof(*srcs));
    st = (crtx_state *) calloc(S, sizeof(*st));
    st_halo = (crtx_state *) calloc(S, sizeof(*st));
    fin = (crtx_state *) calloc(S, sizeof(*st));
    hsrc = (unsigned char **) calloc(S, sizeof(*hsrc));
    hout = (unsigned char **) calloc(S, sizeof(*hout));
    hsrc2 = (unsigned char **) calloc(S, sizeof(*hsrc2));
    hout2 = (unsigned char **) calloc(S, sizeof(*hout2));
    dsrc = (void **) calloc(S, sizeof(*dsrc));
    draw = (void **) calloc(S, sizeof(*draw));
    dfile = (void **) calloc(S, sizeof(*dfile));
    work = (void **) calloc(S, sizeof(*work));
    halo = (void **) calloc(S, sizeof(*halo));
    if (!lo || !hi || !skip || !rand_halo || !mons || !srcs || !st || !st_halo || !fin || !hsrc || !hout || !hsrc2 || !hout2 || !dsrc || !draw || !dfile || !work || !halo) die("out of memory");

    TRY(crtx_create(&ctx, S));
    longest = 0;
    for (s = 0; s < S; s++) {
        span_of(j.n, s, S, &lo[s], &hi[s]);
        if (hi[s] - lo[s] > longest) longest = hi[s] - lo[s];
        hsrc[s] = (unsigned char *) crtx_host_alloc(j.file_bytes);
        hout[s] = (unsigned char *) crtx_host_alloc(j.out_bytes);
        hsrc2[s] = (unsigned char *) crtx_host_alloc(j.file_bytes);
        hout2[s] = (unsigned char *) crtx_host_alloc(j.out_bytes);
        dsrc[s] = crtx_device_alloc(j.src_bytes);
        draw[s] = crtx_device_alloc(j.file_bytes);
        dfile[s] = crtx_device_alloc(j.out_bytes);
        work[s] = crtx_device_alloc(j.out_bytes);
        halo[s] = crtx_device_alloc(j.out_bytes);
        if (!hsrc[s] || !hout[s] || !hsrc2[s] || !hout2[s] || !dsrc[s] || !draw[s] || !dfile[s] || !work[s] || !halo[s]) die("out of memory (device or pinned host)");
        mons[s].out = work[s];
        mons[s].outw = j.outw;
        mons[s].outh = j.outh;
        mons[s].out_format = PIX_BGRA;
        mons[s].contrast = 180;   /* crt_reset, crt_core.c:250-261 */
        mons[s].saturation = 10;  /* video_convert.c:241 */
        mons[s].white_point = 100;
        mons[s].scanlines = j.scanlines;
        mons[s].blend = 0;
        mons[s].noise = j.noise;
    }
    TRY(crtx_set_monitors(ctx, 0, S, mons));
    printf("converting %d images %dx%d -> %dx%d in %d segments...\n", j.n, j.w, j.h, j.outw, j.outh, S);
    if (j.vhs) printf("rand() seed %u\n", seed);

    /* ---- what a steady decode holds after an image of each parity: a 4-image probe, noise 0 ---- */
    have_after[0] = have_after[1] = 0;
    {
        crtx_monitor pm = mons[0];
        crtx_source ps;
        crtx_state pst;
        void *pout = crtx_device_alloc(j.out_bytes);
        int f;
        if (!pout) die("out of memory");
        pm.out = pout;
        pm.noise = 0;
        TRY(crtx_create(&probe, 1));
        TRY(crtx_set_monitors(probe, 0, 1, &pm));
        if (j.vhs) rand_seed(probe, 1, seed);
        for (f = 0; f < 4 && f < j.n; f++) {
            stage_image(&j, f, hsrc[0], draw[0], dsrc[0]);
            fill_source(&j, &ps, dsrc[0], f);
            TRY(crtx_modulate(probe, 0, 1, &ps, NULL));
            TRY(crtx_demodulate(probe, 0, 1, NULL));
            TRY(crtx_get_state(probe, 0, 1, &pst, NULL));
            after_hs[f & 1] = pst.hsync;
            after_vs[f & 1] = pst.vsync;
            have_after[f & 1] = 1;
        }
        crtx_destroy(probe);
        crtx_device_free(pout);
    }

    /* ---- start states: every segment but the first begins two images early ---- */
    for (s = 0; s < S; s++) {
        int h0 = lo[s] - 2 > 0 ? lo[s] - 2 : 0;
        memset(&st[s], 0, sizeof(st[s]));
        if (h0 > 0 && have_after[(h0 - 1) & 1]) {
            st[s].hsync = after_hs[(h0 - 1) & 1];
            st[s].vsync = after_vs[(h0 - 1) & 1];
        }
        st[s].rn = as_int32(lcg_advance(rn0, (unsigned long) crtx_input_size() * (unsigned long) h0));
        skip[s] = h0;
    }
    TRY(crtx_set_state(ctx, 0, S, st, NULL));
    if (j.vhs) { /* every segment's generator where the sequential loop has it before image h0 */
        rand_seed(ctx, S, seed);
        rand_skip(ctx, S, skip, j.aberration);
    }

    /* ---- halo: images lo - 2 and lo - 1 (segments that have them are a suffix of the list) ---- */
    for (t = 2; t >= 1; t--) {
        int first = S;
        for (s = 0; s < S; s++) {
            if (lo[s] >= t) {
                if (s < first) first = s;
                stage_image(&j, lo[s] - t, hsrc[s], draw[s], dsrc[s]);
                fill_source(&j, &srcs[s], dsrc[s], lo[s] - t);
            }
        }
        if (first < S) {
            TRY(crtx_modulate(ctx, first, S - first, srcs + first, NULL));
            TRY(crtx_demodulate(ctx, first, S - first, NULL));
        }
        TRY(crtx_sync(NULL)); /* the pinned staging buffers are reused by the next step */
    }
    TRY(crtx_get_state(ctx, 0, S, st_halo, NULL));
    if (j.vhs) rand_get(ctx, S, rand_halo); /* exact: the halo's draws do not depend on its sync state */
    for (s = 1; s < S; s++) TRY(crtx_memcpy(halo[s], work[s], j.out_bytes, 2, NULL));

    /* ---- main steps: step t decodes image lo[s] + t of every segment still inside its span; longer
     * segments come first, so the active ones are 0 .. count - 1.  Two sets of page-locked buffers alternate:
     * the files of step t + 1 are read, and the images of step t - 1 written, by two helper threads while the
     * device works on step t.  A set is handed to a thread only after the crtx_sync that ends the step which
     * copied from / into it, and taken back (join) before the next step that uses it issues its copies. ---- */
    for (t = 0; t < 2; t++) {
        rd[t].j = wr[t].j = &j;
        rd[t].write = 0;
        wr[t].write = 1;
        rd[t].running = wr[t].running = 0;
        rd[t].count = wr[t].count = 0;
        rd[t].frame = (int *) malloc(sizeof(int) * S);
        wr[t].frame = (int *) malloc(sizeof(int) * S);
        rd[t].buf = (unsigned char **) malloc(sizeof(unsigned char *) * S);
        wr[t].buf = (unsigned char **) malloc(sizeof(unsigned char *) * S);
        if (!rd[t].frame || !wr[t].frame || !rd[t].buf || !wr[t].buf) die("out of memory");
    }
#define ACTIVE_AT(step, n) do { (n) = 0; for (s = 0; s < S; s++) if (lo[s] + (step) < hi[s]) (n) = s + 1; } while (0)
#define SET_OF(step, a, b) (((step) & 1) ? (b) : (a))
    ACTIVE_AT(0, rd[0].count);
    for (s = 0; s < rd[0].count; s++) {
        rd[0].frame[s] = lo[s];
        rd[0].buf[s] = hsrc[s];
    }
    io_start(&rd[0]);
    for (t = 0; t < longest; t++) {
        const int cur = t & 1;
        unsigned char **in = SET_OF(t, hsrc, hsrc2), **outb = SET_OF(t, hout, hout2);
        int count;
        ACTIVE_AT(t, count);
        io_join(&rd[cur]); /* the files of this step are in `in` */
        if (t + 1 < longest) { /* the other input set was last copied from in step t - 1, which has been synced */
            unsigned char **nin = SET_OF(t + 1, hsrc, hsrc2);
            ACTIVE_AT(t + 1, rd[cur ^ 1].count);
            for (s = 0; s < rd[cur ^ 1].count; s++) {
                rd[cur ^ 1].frame[s] = lo[s] + t + 1;
                rd[cur ^ 1].buf[s] = nin[s];
            }
            io_start(&rd[cur ^ 1]);
        }
        io_join(&wr[cur]); /* the writer of step t - 2 is done with `outb` */
        for (s = 0; s < count; s++) {
            TRY(crtx_memcpy(draw[s], in[s], j.file_bytes, 0, NULL));
            TRY(crtx_bmp_unpack(dsrc[s], draw[s], j.w, j.h, j.bits, NULL));
            fill_source(&j, &srcs[s], dsrc[s], lo[s] + t);
        }
        TRY(crtx_modulate(ctx, 0, count, srcs, NULL));
        TRY(crtx_demodulate(ctx, 0, count, NULL));
        for (s = 0; s < count; s++) fetch_image(&j, work[s], dfile[s], outb[s]);
        TRY(crtx_sync(NULL));
        wr[cur].count = count;
        for (s = 0; s < count; s++) {
            wr[cur].frame[s] = lo[s] + t;
            wr[cur].buf[s] = outb[s];
        }
        io_start(&wr[cur]);
        printf("step %d / %d\n", t + 1, longest);
    }
    io_join(&wr[0]);
    io_join(&wr[1]);
    io_join(&rd[0]);
    io_join(&rd[1]);
#undef ACTIVE_AT
#undef SET_OF
    for (t = 0; t < 2; t++) {
        free(rd[t].frame);
        free(wr[t].frame);
        free(rd[t].buf);
        free(wr[t].buf);
    }
    TRY(crtx_get_state(ctx, 0, S, fin, NULL));

    /* ---- verification in sequence order; a failed segment is redone from the true state ---- */
    for (s = 1; s < S; s++) {
        int differ = 0, f;
        if ((j.vhs || st_halo[s].hsync == fin[s - 1].hsync) && st_halo[s].vsync == fin[s - 1].vsync) {
            TRY(crtx_memcmp_device(halo[s], work[s - 1], j.out_bytes, &differ, NULL));
            if (!differ) continue;
        }
        recomputed++;
        memset(&st[s], 0, sizeof(st[s]));
        st[s].hsync = fin[s - 1].hsync;
        st[s].vsync = fin[s - 1].vsync;
        st[s].rn = as_int32(lcg_advance(rn0, (unsigned long) crtx_input_size() * (unsigned long) lo[s]));
        TRY(crtx_set_state(ctx, s, 1, &st[s], NULL));
        if (j.vhs) rand_set(ctx, s, rand_halo + (size_t) s * CRTX_RAND_WORDS);
        TRY(crtx_memcpy(work[s], work[s - 1], j.out_bytes, 2, NULL));
        for (f = lo[s]; f < hi[s]; f++) {
            stage_image(&j, f, hsrc[s], draw[s], dsrc[s]);
            fill_source(&j, &srcs[s], dsrc[s], f);
            TRY(crtx_modulate(ctx, s, 1, &srcs[s], NULL));
            TRY(crtx_demodulate(ctx, s, 1, NULL));
            fetch_image(&j, work[s], dfile[s], hout[s]);
            TRY(crtx_sync(NULL));
            save_image(&j, f, hout[s]);
        }
        TRY(crtx_get_state(ctx, s, 1, &fin[s], NULL));
    }
    printf("done: %d images, %d segments, %d redone, %ld kernel launches\n", j.n, S, recomputed, crtx_launch_count(ctx));

    for (s = 0; s < S; s++) {
        crtx_host_free(hsrc[s]);
        crtx_host_free(hout[s]);
        crtx_host_free(hsrc2[s]);
        crtx_host_free(hout2[s]);
        crtx_device_free(dsrc[s]);
        crtx_device_free(draw[s]);
        crtx_device_free(dfile[s]);
        crtx_device_free(work[s]);
        crtx_device_free(halo[s]);
    }
    crtx_destroy(ctx);
    free(skip);
    free(rand_halo);
    return EXIT_SUCCESS;
}
