// crt_records.h -- the small records host code and kernels exchange.
#pragma once

#include "crt_b200.h"
#include "crtx_batch.h"

namespace crt {

// ---------------------------------------------------------------------------------------
// device-side records
// ---------------------------------------------------------------------------------------
struct MonCfg { // host -> device, the caller-settable part of struct CRT
    unsigned char *out;
    int outw, outh, out_format, bpp;
    int hue, brightness, contrast, saturation;
    int black_point, white_point;
    int scanlines, blend;
    unsigned v_fac;
    int noise;
    int out_pitch; // bytes between output rows (never 0: the host resolves crtx_monitor's 0 to outw * bpp)
};

struct MonState { // device resident, the persistent decoder state of struct CRT
    int ccf[CRT_CC_VPER > 3 ? CRT_CC_VPER : 3][CRT_CC_SAMPLES]; // [3][4] everywhere but the PV-1000 ([5][5])
    int hsync, vsync, rn;
    int field;   // detected field * (ratio / 2) of the last demodulate (crt_core.c:398-407)
    int generic; // last sync pass: some line needs the wrap-exact (generic) equaliser path
    int track_max; // last sync pass: some line's carrier was large enough for the fast path to hinge on the line's largest sample:
                   // the next pass measures every signal line's while it copies it (crt_sync.cuh); device-managed
    int pad;
};

struct SrcCfg { // host -> device, struct NTSC_SETTINGS
    const void *data;
    int format, w, h;
    int raw, as_color, field, frame;
    int hue, xoffset, yoffset;
    int aberration; // VHS: already drawn number of sync-less lines (crt_ntscvhs.c:205-207)
    int dot_crawl_offset;
    int reinit;
    int compact; // internal (crtx_frames_host): `data` holds only the rows this field reads, picture line y in row y
    int pitch;   // bytes between source rows (resolved by the host: crtx_source's 0 becomes w * bpp, NES w * 2)
};

typedef crtx_line LineRec; // 32 bytes

} // namespace crt
