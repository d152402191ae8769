// crtx_internal.h -- what crtx.cu and crt_dropin.cu share (not part of the C-ABI).
#pragma once

#include <cuda_runtime.h>

#include <vector>

#include "crt_sys.cuh"
#include "crtx_batch.h"

#include "crt_records.h"

namespace crt {
// A monitor's inp[] after the calls so far.  At noise 0 a demodulate may leave it unwritten (crt_sync.cuh: inp_late): it is
// late, made from analog[] when it is handed out, and gone once a modulate has rewritten that analog[].  Once crtx_inp has
// handed out a raw pointer to it, it is pinned: k_sync writes it on every demodulate, so it is never late again.  A gone
// inp[] that gets pinned stays unreadable until the next demodulate or write of it (kInpPinnedGone).
enum InpState : unsigned char { kInpWritten, kInpLate, kInpGone, kInpPinned, kInpPinnedGone };
inline bool inp_pinned(InpState s) { return s == kInpPinned || s == kInpPinnedGone; }
inline bool inp_gone(InpState s) { return s == kInpGone || s == kInpPinnedGone; }

// The line passes of a run of monitors: LinesGeom::pass takes first, first + 1, .. first + count - 1 (crtx.cu: line_passes)
struct LinePasses {
    int first, count;
};

// One run of a demodulate's line plan (crtx.cu: plan_lines): monitors [lo, hi) share the output geometry `geo` (its pass
// is set per launch) and are decoded by `passes` launches of k_lines2 (`lines2`) or of the build's line kernel
struct LineRun {
    int lo, hi;
    LinesGeom geo;
    LinePasses passes;
    bool lines2;
};
} // namespace crt

struct crtx_ctx {
    int n = 0;
    int device = 0;
    int sm_count = 132;
    crt::MonCfg *d_cfg = nullptr;
    crt::MonState *d_state = nullptr;
    crt::SrcCfg *d_src = nullptr;
    void *d_row_jobs = nullptr;            // crtx_frames_host: RowGather[n]
    unsigned char **d_host_out = nullptr;  // crtx_frames_host: device mappings of the callers' host images, [n]
    crtx_line *d_lines = nullptr;
    signed char *d_analog = nullptr;
    signed char *d_inp = nullptr;
    crt::Affine *d_jump_lo = nullptr;
    crt::Affine *d_jump_hi = nullptr;
    signed char *d_nes_tab = nullptr; // NES: per-monitor 512 x 12 sample table + burst rows
    void *d_bloom = nullptr;      // CRT_DO_BLOOM build: BloomLine[n][CRT_LINES], each line's resampling step and start
    void *d_vhs_rand = nullptr;   // VHS: VhsRand[n], glibc rand() replica per monitor
    void *d_vhs_rand_next = nullptr; // VHS: the state after the running call (k_vhs_commit copies it back)
    void *d_vhs_jump = nullptr;   // VHS: jump-ahead matrices
    unsigned *d_vhs_raw = nullptr; // VHS: tail raw-stream scratch
    int *d_vhs_wants = nullptr;   // VHS: do_aberration flags of the current modulate
    int *d_vhs_fields = nullptr;  // VHS: field counts of the current crtx_skip_fields
    bool vhs_seeded = false;
    int vhs_draw_aberration = 0;
    unsigned char *d_src_img = nullptr; // crtx_frames_host staging, src_slot bytes per monitor
    size_t src_slot = 0;
    std::vector<crt::MonCfg> h_cfg;
    std::vector<unsigned char> h_mod_staged; // per monitor: the last modulate encoded its picture with k_mod_picture_rgb_staged (crtx_get_paths)
    std::vector<crt::SrcCfg> scratch_src;
    std::vector<crt::LineRun> scratch_runs; // demodulate_launch's line plan
    std::vector<crt::InpState> h_inp; // per monitor
    int cfg_dirty_lo = 0, cfg_dirty_hi = 0;
    int tail_dirty_lo = 0, tail_dirty_hi = 0; // monitors whose output geometry changed: k_struct_tail rewrites the bytes behind their signals
    cudaEvent_t cfg_ready = nullptr;   // recorded behind the last configuration upload; launches on other streams wait on it
    cudaStream_t cfg_stream = nullptr; // the stream that upload went to
    long launches = 0;
    long lines2_launches = 0; // line passes that took k_lines2 (crtx_lines2_count)
    int opt_generic = 0;
    int opt_timing = 0;
    int opt_mod_staged = 1;
    int opt_lines2 = 1;   // line pass: 1 = k_lines2 where the geometry qualifies (crt_lines2.cuh), 0 = always k_lines (A/B switch)
    int opt_host_rows = 1; // crtx_frames_host: move only the rows a field reads / writes (page-locked, 16-byte granular images)
    int opt_host_src = 0; // crtx_frames_host: read page-locked source images in place
    int opt_line_lo = 0, opt_line_hi = 1 << 30; // decoded-line window of the line pass (crtx_set_option)
    struct Timed {
        int kernel;
        cudaEvent_t start, stop;
    };
    std::vector<Timed> timed;            // recorded, not yet read
    std::vector<cudaEvent_t> event_pool; // recycled events
};

namespace crt {
// bytes of one source row: w pixels of the format's size, 2-byte pixels on the NES (the dense pitch)
inline long long src_row_bytes(int format, int w) { return (long long) w * (kIsNes ? 2 : bpp_of(format)); }
int fail(const char *fmt, ...);
void fill_src(SrcCfg *d, const crtx_source *s);
// sets SrcCfg::staged of every src[i] before it uploads them
int modulate_launch(crtx_ctx *ctx, int first, int count, SrcCfg *src, cudaStream_t stream);
// d_noise_terms: VHS only -- per-sample noise term already drawn on the host from libc rand()
int demodulate_launch(crtx_ctx *ctx, int first, int count, cudaStream_t stream, const short *d_noise_terms);
// inp[] of monitors [first, first + count) made from analog[] where the last demodulate left it (ordered on `stream`)
int inp_from_analog(crtx_ctx *ctx, int first, int count, cudaStream_t stream);
} // namespace crt
