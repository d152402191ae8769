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
    int lines2;    // host-managed: this demodulate's line plan decodes the monitor with k_lines2, so at noise 0 k_sync may
                   // leave inp[] unwritten (crtx.cu: plan_lines)
};

struct MonState { // device resident, the persistent decoder state of struct CRT
    int ccf[CRT_CC_VPER > 3 ? CRT_CC_VPER : 3][CRT_CC_SAMPLES]; // [3][4] everywhere but the PV-1000 ([5][5])
    int hsync, vsync, rn;
    int field;   // detected field * (ratio / 2) of the last demodulate (crt_core.c:398-407)
    int generic; // last sync pass: some line needs the wrap-exact (generic) equaliser path
    int track_max; // last sync pass: some line's carrier was large enough for the fast path to hinge on the line's largest sample:
                   // the next pass measures every signal line's while it copies it (crt_sync.cuh); device-managed
    int inp_late;  // last sync pass left inp[] unwritten: k_lines2 decodes from analog[], clamping each sample as it reads it
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
    int staged;  // internal (modulate_launch): k_mod_picture_rgb_staged encodes the picture, k_mod_picture_rgb leaves it
#if NES_BORDER
    unsigned border_color; // (only in the border build: every other build keeps the record, and its kernels, as they were)
#endif
};

struct LinesGeom { // uniform over a launch: host groups monitors by these (crtx.cu)
    int outw, out_format, bpp, blend;
    int pitch; // bytes between output rows (MonCfg::out_pitch, shared by every monitor of the launch)
    int pass; // -1: every line; -2: only the last line of each shared-row run; >= 0: lines at this run position (level)
    int rnd; // 32768, passed as an argument so that it lives in a register (see pole())
    int dx;  // ((AV_LEN - 1) << 12) / outw (crt_core.c:527), computed by the host: no division in the kernels
    int line_lo, line_hi; // decoded lines [lo, hi) this launch may touch (scanline-block sharding across ranks)
};

typedef crtx_line LineRec; // 32 bytes

} // namespace crt
