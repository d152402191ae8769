// crt_sys.cuh -- compile-time description of the emulated system and the integer
// helpers shared by host and device code.
//
// The reference selects the system with -DCRT_SYSTEM=n (crt_core.h:39-59); so do we: one
// shared library per variant, every timing constant a compile-time constant so ptxas can fold
// them into immediates.  The filter coefficients the reference computes at run time in
// crt_init (crt_core.c:263-289) and init_iir (crt_ntsc.c:98-106) are evaluated here by
// constexpr restatements of the same integer formulas and pinned with static_asserts against
// the values probed from the compiled reference (SURVEY.md 8a).
#pragma once

#include <stdint.h>
#include "crt_b200.h"

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace crt {

constexpr int kSystem = CRT_SYSTEM;
#ifndef CRT_CHROMA_PATTERN /* crt_snes.h has no such switch: 227.3 cycles per line, as NES pattern 2; */
#if (CRT_SYSTEM == CRT_SYSTEM_TEMP) /* nor has crt_template.h: 227.5 cycles per line, as NTSC's pattern 1 */
#define CRT_CHROMA_PATTERN 1
#elif (CRT_SYSTEM == CRT_SYSTEM_PV1K) /* crt_pv1k.h: 230.4 cycles per line, none of the NES patterns */
#define CRT_CHROMA_PATTERN 0
#else
#define CRT_CHROMA_PATTERN 2
#endif
#endif
constexpr int kPattern = CRT_CHROMA_PATTERN;
constexpr bool kIsNes = (CRT_SYSTEM == CRT_SYSTEM_NES);
constexpr bool kIsVhs = (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS);
constexpr bool kIsSnes = (CRT_SYSTEM == CRT_SYSTEM_SNES);
constexpr bool kIsNesRgb = (CRT_SYSTEM == CRT_SYSTEM_NESRGB);
constexpr bool kIsTemp = (CRT_SYSTEM == CRT_SYSTEM_TEMP);
constexpr bool kIsPv1k = (CRT_SYSTEM == CRT_SYSTEM_PV1K);
constexpr int kCc = CRT_CC_SAMPLES; // samples per chroma period: 4, or 5 for the PV-1000 (crt_pv1k.h:49)
static_assert(kCc == 4 || kCc == 5, "crt_core.c:286-288");
// the systems whose encoder is crt_ntsc.c / crt_ntscvhs.c / crt_template.c (band-limited RGB on the NTSC line
// layout, 227.5 cycles per line); the template system walks a 2-line chroma cycle instead of flipping the phase
#define CRT_B200_NTSC_FAMILY \
    ((CRT_SYSTEM == CRT_SYSTEM_NTSC) || (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS) || (CRT_SYSTEM == CRT_SYSTEM_TEMP))
// ... plus the PV-1000 (crt_pv1k.c): the same encoder structure on its own line layout, five carrier phases, a 5-line cycle
#define CRT_B200_BANDLIMITED (CRT_B200_NTSC_FAMILY || (CRT_SYSTEM == CRT_SYSTEM_PV1K))
constexpr bool kRowCarrier = kIsTemp || kIsPv1k; // carrier tables per colour row (line % CRT_CC_VPER), no phase flip
// -DCRTX_CONV=1 builds the decoder of the reference's USE_CONVOLUTION 1 configuration (an unguarded
// #define at crt_core.c:85, so a separate library like every other compile-time choice there)
#ifndef CRTX_CONV
#define CRTX_CONV 0
#endif
constexpr bool kConv = (CRTX_CONV != 0);
// taps of the convolution kernel: -DCRTX_CONV=1 (or 7) is the stock USE_7_SAMPLE_KERNEL, 6 / 5 / 4 the other
// compile-time choices of crt_core.c:86-88
constexpr int kConvTaps = (CRTX_CONV == 0) ? 0 : (CRTX_CONV == 1) ? 7 : CRTX_CONV;
static_assert(kConvTaps == 0 || (kConvTaps >= 4 && kConvTaps <= 7), "CRTX_CONV: 0, 1 or the tap count 4..7");
// crt_core.c:89-93: "the current convolutions do not filter properly at > 4 samples" -- the reference forces
// USE_CONVOLUTION back to 0 for the PV-1000, so there is no such configuration to reproduce
static_assert(!kConv || CRT_CC_SAMPLES == 4, "CRTX_CONV: the reference disables USE_CONVOLUTION when CRT_CC_SAMPLES != 4 (crt_core.c:89-93)");

// CRT_DO_BLOOM 1 (crt_core.h:70): the decoder derives each line's width from a filtered beam energy
// (crt_core.c:399-402, 512-526) and the encoders shrink the picture (crt_ntsc.c:148-160)
constexpr bool kBloom = (CRT_DO_BLOOM != 0);
// CRT_DO_VSYNC 0 (crt_core.h:71): k_sync takes the field from analog[] before the noise and decodes from vsync -3
// (crt_core.c:323-342).  CRT_DO_HSYNC 0 (crt_core.h:72): hsync is 0 after every decoded line (crt_core.c:446-450).
constexpr bool kDoVsync = (CRT_DO_VSYNC != 0);
constexpr bool kDoHsync = (CRT_DO_HSYNC != 0);

constexpr int kHres = CRT_HRES;
constexpr int kVres = CRT_VRES;
constexpr int kInputSize = CRT_INPUT_SIZE;
constexpr int kTop = CRT_TOP;
constexpr int kBot = CRT_BOT;
constexpr int kLines = CRT_LINES;
constexpr int kVper = CRT_CC_VPER;
constexpr int kHsyncWindow = CRT_HSYNC_WINDOW;
constexpr int kVsyncWindow = CRT_VSYNC_WINDOW;
constexpr int kHsyncLevel = CRT_HSYNC_THRESH * SYNC_LEVEL;
constexpr int kVsyncLevel = CRT_VSYNC_THRESH * SYNC_LEVEL;
constexpr int kSyncBeg = SYNC_BEG;
constexpr int kBwBeg = BW_BEG;
constexpr int kCbBeg = CB_BEG;
constexpr int kAvBeg = AV_BEG;
constexpr int kAvLen = AV_LEN;
constexpr int kBurstLen = CB_CYCLES * CRT_CB_FREQ;
// picture size the RGB encoders scale to (crt_ntsc.c:131-132, 148-172)
constexpr int kDestW = kBloom ? (kAvLen * 55500) >> 16 : kAvLen;
constexpr int kDestH = kBloom ? ((CRT_BOT - CRT_TOP) * 63500) >> 16 : ((CRT_BOT - CRT_TOP) * 64500) >> 16;
constexpr int kWhite = WHITE_LEVEL;
// The white scale WHITE_LEVEL * white_point / 100 of the RGB encoders (crt_ntsc.c:318; the same line in crt_ntscvhs.c,
// crt_snes.c, crt_template.c, crt_pv1k.c and crt_nesrgb.c).  Signed overflow being undefined, gcc -O3 folds the
// expression to white_point where WHITE_LEVEL is 100 -- every system that computes it -- so the compiled reference's
// scale is white_point itself, also where 100 * white_point would wrap.  Any other level wraps like the reference's
// multiplication.
__host__ __device__ constexpr int white_scale(int white_point) {
    return kWhite == 100 ? white_point : (int) ((unsigned) kWhite * (unsigned) white_point) / 100;
}
constexpr int kBurst = BURST_LEVEL;
constexpr int kBlack = BLACK_LEVEL;
constexpr int kBlank = BLANK_LEVEL;
constexpr int kSync = SYNC_LEVEL;
#if (CRT_SYSTEM == CRT_SYSTEM_NES) || (CRT_SYSTEM == CRT_SYSTEM_NESRGB)
constexpr int kNesVsyncEnd = PPUpx2pos(327); // crt_nes.c:91, crt_nesrgb.c:33
#endif
// NES_BORDER 1 (crt_nes.c:64-69; crt_b200.h): the NES encoder draws the border colour on lines kTop .. kBot + 2 from
// LAV_BEG on (crt_nes.c:138-161)
constexpr bool kNesBorder = (NES_BORDER != 0);
#if (CRT_SYSTEM == CRT_SYSTEM_NES)
constexpr int kLavBeg = LAV_BEG;
constexpr int kBorderLo = kTop, kBorderHi = kBot + 2; // (inclusive)
#endif

// Slack after each signal buffer: the reference reads its decode windows up to one line past
// inp[] when sync is lost (crt_core.c:438-441,458,511); those reads are outside the parity
// domain but must stay inside our allocation.
constexpr int kSignalPad = 4096;
constexpr int kSignalBytes = ((kInputSize + kSignalPad + 255) / 256) * 256;

// ---------------------------------------------------------------------------------------
// 14-bit-angle sine/cosine (crt_core.c:19-61)
// ---------------------------------------------------------------------------------------
#define CRT_QUARTER15                                                                    \
    { 0x0000, 0x0c88, 0x18f8, 0x2528, 0x30f8, 0x3c50, 0x4718, 0x5130, 0x5a80, 0x62f0,    \
      0x6a68, 0x70e0, 0x7640, 0x7a78, 0x7d88, 0x7f60, 0x8000, 0x7f60 }

constexpr int kQuarter15[18] = CRT_QUARTER15;

constexpr int quarter_c(int a)
{
    return kQuarter15[(a >> 8) & 0xff]
         + (((kQuarter15[((a >> 8) & 0xff) + 1] - kQuarter15[(a >> 8) & 0xff]) * (a & 0xff)) >> 8);
}

constexpr int sin14_c(int n)
{
    return ((n & 16383) >= 8192 ? -1 : 1)
         * (((n & 8191) >= 4096) ? quarter_c(8192 - (n & 8191)) : quarter_c(n & 8191));
}

// host run-time version (used by the exported crt_sincos14 and by host-side set-up)
inline void sincos14_host(int *s, int *c, int n)
{
    n &= 16383;
    int h = n & 8191;
    if (h >= 4096) {
        *c = -quarter_c(h - 4096);
        *s = quarter_c(8192 - h);
    } else {
        *c = quarter_c(4096 - h);
        *s = quarter_c(h);
    }
    if (n >= 8192) {
        *c = -*c;
        *s = -*s;
    }
}

// ---------------------------------------------------------------------------------------
// decoder equaliser coefficients (crt_core.c:171-196, 272-280), EQ_P = 16
// ---------------------------------------------------------------------------------------
constexpr int khz2l(int khz) { return kHres * (khz * 100) / 1431818; }
constexpr int eq_frac(int khz) { return 2 * (sin14_c(8192 * khz2l(khz) / kHres) << 1); }

constexpr int kEqYlf = eq_frac(1500), kEqYhf = eq_frac(3000);
constexpr int kEqIlf = eq_frac(80), kEqIhf = eq_frac(1150);
constexpr int kEqQlf = eq_frac(80), kEqQhf = eq_frac(1000);
// band gains, Q16 (crt_core.c:278-280): Y {65536, 8192, 9175}, I {65536, 65536, 1311},
// Q {65536, 65536, 0}
// with five samples per chroma period Y's gains are {65536, 12192, 7775} (crt_core.c:282)
constexpr int kEqYg1 = (kCc == 5) ? 12192 : 8192, kEqYg2 = (kCc == 5) ? 7775 : 9175, kEqIg2 = 1311;

#if CRT_B200_NTSC_FAMILY
static_assert(kHres == 910 && kAvBeg == 156 && kAvLen == 753 && kCbBeg == 97 && kSyncBeg == 21
              && kBwBeg == 88, "NTSC timing (SURVEY.md 8a)");
static_assert(kEqYlf == 42156 && kEqYhf == 79824 && kEqIlf == 2252 && kEqIhf == 32636
              && kEqQlf == 2252 && kEqQhf == 28248, "equaliser fractions (SURVEY.md 8a)");
#endif

#if (CRT_SYSTEM == CRT_SYSTEM_SNES) || ((CRT_SYSTEM == CRT_SYSTEM_NESRGB) && (CRT_CHROMA_PATTERN == 2))
static_assert(kHres == 909 && kAvBeg == 197 && kAvLen == 682 && kCbBeg == 101 && kSyncBeg == 23 && kBwBeg == 90
              && kInputSize == 238158, "SNES timing (crt_snes.h:20-109, probed from the compiled reference)");
#endif

// ---------------------------------------------------------------------------------------
// encoder band-limit coefficients (crt_ntsc.c:25-106)
// ---------------------------------------------------------------------------------------
constexpr int exp_q11_c(int n)
{
    // only ever evaluated for -2048 < n < 0 here (idx == 0 branch of crt_ntsc.c:41-83)
    long long a = n < 0 ? -(long long) n : n;
    long long term = 2048, sum = 0, fact = 1;
    for (int k = 1; k < 17; k++) {
        sum += term / fact;
        term = (term * a) >> 11;
        fact *= k;
        if (fact > term || term <= 0 || fact <= 0) break;
    }
    long long res = (2048 * sum) >> 11;
    if (n < 0) res = (2048LL << 11) / res;
    return (int) res;
}

constexpr int bandlimit_c(int limit)
{
    return 2048 - exp_q11_c(-((6434 << 9) / ((1431818 << 9) / limit)));
}

#if (CRT_SYSTEM == CRT_SYSTEM_PV1K)
static_assert(kHres == 1920 && kInputSize == 503040 && kSyncBeg == 81 && kBwBeg == 162 && kCbBeg == 216 && kAvBeg == 432
              && kAvLen == 1487 && kBurstLen == 50 && kVper == 5, "PV-1000 timing (crt_pv1k.h:36-101)");
static_assert(kEqYlf == 42252 && kEqYhf == 80024 && kEqIlf == 2104 && kEqIhf == 32636 && kEqQlf == 2104 && kEqQhf == 28444,
              "PV-1000 equaliser fractions (crt_core.c:171-196 with CRT_HRES 1920; probed from the compiled reference)");
#endif

#if (CRT_SYSTEM == CRT_SYSTEM_NTSC) || (CRT_SYSTEM == CRT_SYSTEM_TEMP) || (CRT_SYSTEM == CRT_SYSTEM_PV1K) // crt_ntsc.h:86-90, crt_template.h:117-121, crt_pv1k.h:108-112
constexpr int kIirY = bandlimit_c(420000), kIirI = bandlimit_c(150000), kIirQ = bandlimit_c(55000);
static_assert(kIirY == 1233 && kIirI == 574 && kIirQ == 232, "NTSC band-limit (SURVEY.md 8a)");
#elif (CRT_SYSTEM == CRT_SYSTEM_NTSCVHS)
constexpr int kIirY = bandlimit_c(300000), kIirI = bandlimit_c(62700), kIirQ = bandlimit_c(62700);
static_assert(kIirY == 987 && kIirI == 262 && kIirQ == 262, "VHS band-limit (SURVEY.md 8a)");
#endif

// ---------------------------------------------------------------------------------------
// noise LCG (crt_core.c:359) and its jump-ahead
// ---------------------------------------------------------------------------------------
constexpr uint32_t kLcgMul = 214019u, kLcgAdd = 140327895u;

struct Affine { // x -> x * mul + add (mod 2^32)
    uint32_t mul, add;
};

constexpr Affine lcg_jump(uint32_t n)
{
    uint32_t am = kLcgMul, ac = kLcgAdd, rm = 1u, rc = 0u;
    while (n) {
        if (n & 1u) { rc = rc * am + ac; rm = rm * am; }
        ac = ac * am + ac;
        am = am * am;
        n >>= 1;
    }
    return Affine{ rm, rc };
}

constexpr Affine kLcgField = lcg_jump((uint32_t) kInputSize); // one whole crt_demodulate call
#if (CRT_SYSTEM == CRT_SYSTEM_NTSC)
static_assert(kLcgField.mul == 0x5535b491u && kLcgField.add == 0xf58bfa78u, "SURVEY.md 7.2 K1");
#endif

// pixel formats (crt_core.h:62-67): bytes per pixel, and the byte positions of R, G, B in a pixel (a 4-byte format's
// alpha takes the remaining byte, 6 - r - g - b)
__host__ __device__ inline int bpp_of(int f) { return (f == 0 || f == 1) ? 3 : ((f >= 2 && f <= 5) ? 4 : 0); }
constexpr __host__ __device__ void fmt_positions(int f, int &r, int &g, int &b)
{
    switch (f) {
        case CRT_PIX_FORMAT_RGB:  r = 0; g = 1; b = 2; break;
        case CRT_PIX_FORMAT_BGR:  r = 2; g = 1; b = 0; break;
        case CRT_PIX_FORMAT_ARGB: r = 1; g = 2; b = 3; break;
        case CRT_PIX_FORMAT_RGBA: r = 0; g = 1; b = 2; break;
        case CRT_PIX_FORMAT_ABGR: r = 3; g = 2; b = 1; break;
        default:                  r = 2; g = 1; b = 0; break; // BGRA
    }
}
// the byte position of channel c (0 R, 1 G, 2 B, 3 alpha) at compile time
constexpr int fmt_pos(int f, int c)
{
    int p[4] = { 0, 0, 0, 0 };
    fmt_positions(f, p[0], p[1], p[2]);
    p[3] = 6 - p[0] - p[1] - p[2];
    return p[c];
}

} // namespace crt
