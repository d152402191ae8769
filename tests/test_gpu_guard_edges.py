"""The fast paths at the edges of the ranges their guards admit, bit for bit against the oracle through the batch interface.

Every hot kernel has a fast form that is exact only inside a range, and a guard that picks the path per monitor or launch:
  * the fast equaliser (crt_lines.cuh, crt_lines2.cuh, crt_lines_fir.cuh) while every chroma input (s * wave) >> 9 stays
    within +-16383 -- k_sync admits a line when ((max|s| * wmax) >> 9) + 1 <= 16383 -- and |bright| <= 4096 (2048 on the
    PV-1000);
  * the staged encoder (crt_kernels.cuh) while a chunk's source span fits a stage row: span * bpp + 31 <= 192;
  * its stores, windows aligned to 32-byte sectors of analog[], at every phase of the line start;
  * the burst lock's shortcut for x * 127 / 128 while |x| < 2^23 (crt_sync.cuh).
Each case asserts the path it expects through crtx_get_paths (Batch.paths), so that none passes by falling to the other one,
and sits on both sides of the edge.  The signals are written into analog[] directly (crtx_write_signal) and each pass is
replayed from a saved decoder state (crtx_set_state), so the same field can be decoded with another amplitude or
saturation."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

OUTW, OUTH = 640, 480
GEN, STAGED = 1, 2  # Batch.PATH_GENERIC_EQ, Batch.PATH_STAGED_MOD
KNOBS = dict(blend=0, scanlines=0)


# ---------------------------------------------------------------------------------------------------------------------
# replaying one field from a saved state
# ---------------------------------------------------------------------------------------------------------------------

def _settle(variant, seed=5):
    """one ordinary field through the oracle: the burst lock settles.  Returns (decoder state after it, its signal)."""
    o = S.OracleEngine(variant, OUTW, OUTH)
    o.set(**KNOBS)
    if layout.system_spec(variant).system == layout.SYS_NES:
        o.modulate(S.nes_image(seed=seed), dot_crawl_offset=0)
    else:
        o.modulate(S.rand_image(320, 240, seed=seed), format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
    o.demodulate(0)
    return dict(ccf=o.ccf.copy(), hsync=o.hsync, vsync=o.vsync, rn=o.rn), o.analog


def _oracle_at(variant, state, signal, **knobs):
    o = S.OracleEngine(variant, OUTW, OUTH)
    o.set(**dict(KNOBS, **knobs))
    np.ctypeslib.as_array(o.mon.analog, shape=(o.spec.input_size,))[:] = signal
    ccf = np.asarray(state["ccf"])
    for r in range(ccf.shape[0]):
        for x in range(ccf.shape[1]):
            o.mon.ccf[r][x] = int(ccf[r][x])
    o.mon.hsync, o.mon.vsync, o.mon.rn = state["hsync"], state["vsync"], state["rn"]
    return o


def _probe(variant, state, signal, **knobs):
    """the oracle's sync pass over `signal` from `state`: the decoded lines' records (pos, carrier tables)"""
    o = _oracle_at(variant, state, signal, **knobs)
    o.noise_pass(0)
    _, table = o.sync_pass()
    return [r for r in table if not r.skip]


def _gpu_state(state):
    from ntsc_crt_b200 import capi
    s = (capi.State * 1)()[0]
    ccf = np.asarray(state["ccf"])
    for r in range(ccf.shape[0]):
        for x in range(ccf.shape[1]):
            s.ccf[r][x] = int(ccf[r][x])
    s.hsync, s.vsync, s.rn = state["hsync"], state["vsync"], state["rn"]
    return s


class Replay:
    """a batch of monitors that decode given signals from given states, each pass checked against the oracle"""

    def __init__(self, variant, n=1, lines2=None, **knobs):
        import torch
        from ntsc_crt_b200 import capi
        self.variant, self.n = variant, n
        self.b = capi.Batch(variant, n)
        if lines2 is not None:
            self.b.set_option("lines2", lines2)
        self.outs = [torch.zeros(OUTH, OUTW, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
        self.knobs = [dict(knobs) for _ in range(n)]
        for i in range(n):
            self.b.set_monitor(i, self.outs[i], fmt=layout.PIX_BGRA, **dict(KNOBS, **knobs))
        self.b.commit_monitors()

    def configure(self, i, **knobs):
        for k, v in knobs.items():
            setattr(self.b.monitors[i], k, v)
        self.knobs[i].update(knobs)
        self.b.commit_monitors(i, 1)

    def run(self, items, what=""):
        """items: [(monitor, state, signal)]; one demodulate over the whole batch; returns the monitors' paths"""
        import torch
        from ntsc_crt_b200 import capi
        for i, state, signal in items:
            self.outs[i].zero_()
            self.b.set_state((capi.State * 1)(_gpu_state(state)), first=i)
            self.b.write_signal(i, signal, "analog")
        self.b.demodulate()
        torch.cuda.synchronize()
        for i, state, signal in items:
            o = _oracle_at(self.variant, state, signal, **self.knobs[i])
            o.out[:] = 0
            o.demodulate(0)
            got = self.outs[i].cpu().numpy()
            assert np.array_equal(self.b.signal(i, "inp"), o.inp), "%s monitor %d: inp" % (what, i)
            assert np.array_equal(got, o.out), "%s monitor %d: %s" % (what, i, S.diff_report("out", got, o.out))
        return self.b.paths()


# ---------------------------------------------------------------------------------------------------------------------
# equaliser, chroma
# ---------------------------------------------------------------------------------------------------------------------

def _carrier(rec, cc, i, which):
    """the carrier value the line kernel multiplies sample pos + i by (oracle/crt_oracle.c:1013-1014)"""
    if cc == 4:
        return rec.wave[i & 3] if which == "I" else rec.wave[(i + 3) & 3]
    return rec.wave_i[i % cc] if which == "I" else rec.wave_q[i % cc]


def _wmax(rec, cc):
    return max(abs(x) for x in (list(rec.wave[:4]) if cc == 4 else list(rec.wave_i) + list(rec.wave_q)))


def _unit_pattern(spec, recs, which, run=20):
    """(positions, signs): inside every decoded line's window, away from its ends, the sign of the carrier the I (or Q)
    input is multiplied by, in runs of `run` samples that reverse abruptly -- A * sign drives that input to +-(A * w) >> 9"""
    cc, L = spec.cc_samples, spec.av_len
    pos, sgn = [], []
    i = np.arange(24, L - 24)
    rev = np.where((i // run) % 2 == 0, 1, -1)
    for rec in recs:
        w = np.array([_carrier(rec, cc, int(t), which) for t in range(cc)])
        pos.append(rec.pos + i)
        sgn.append(np.sign(w[i % cc]) * rev)
    pos, sgn = np.concatenate(pos), np.concatenate(sgn)
    keep = pos < spec.input_size
    return pos[keep], sgn[keep].astype(np.int64)


def _picture_lines(spec, state, recs):
    """the decoded lines whose windows lie away from the vertical sync (the PV-1000 and the NES decode lines that hold it)"""
    far = lambda r: min((r.pos // spec.hres - state["vsync"]) % spec.vres, (state["vsync"] - r.pos // spec.hres) % spec.vres)
    return [r for r in recs if far(r) > spec.vsync_window + 2]


def _blank_windows(spec, recs, signal, others=()):
    """the signal with the picture of every line in `recs` cleared (0) from its window's start (or the start of the active
    video, where the picture begins earlier) to the end of the signal line, so that the pattern written over it is the largest sample of the line, and the windows of `others` (lines near
    the vertical sync) limited to the sync level's magnitude, 40"""
    x = signal.copy()
    span = lambda r: slice(min(r.pos, r.pos // spec.hres * spec.hres + spec.av_beg - 8), (r.pos // spec.hres + 1) * spec.hres)
    for rec in others:
        x[span(rec)] = np.clip(x[span(rec)], -40, 40)
    for rec in recs:
        x[span(rec)] = 0
    return x


def _with(signal, pos, values):
    x = signal.copy()
    x[pos] = values
    return x


def _edge_setting(variant, spec, state, signal):
    """(hue, saturation) for the chroma edge: 127 * wmax fails the bound, the edge amplitude lies well above the sync and
    burst levels (64 .. 126), and -- where the hue allows it -- one amplitude puts (A * wmax) >> 9 at 16383 exactly, the
    first value the guard rejects, so that an off-by-one in the bound moves A*.  The carrier scales exactly with the
    saturation (crt_core.c:469-479, 497-508), so each hue needs one probe."""
    best = None
    for hue in range(0, 360, 3):
        w1 = max(_wmax(r, spec.cc_samples) for r in _picture_lines(spec, state, _probe(variant, state, signal, hue=hue, saturation=1)))
        for sat in range(-(-66100 // w1), 130000 // w1 + 1):
            wm = sat * w1
            a = -(-16383 * 512 // wm)  # the least amplitude the bound rejects
            if not 64 < a <= 127:
                continue
            key = (((a * wm) >> 9) == 16383, ((a - 1) * wm) >> 9, -hue, -sat)
            if best is None or key > best[0]:
                best = (key, hue, sat)
        if spec.cc_samples != 4 or best[0][0]:
            break
    return best[1], best[2]


CHROMA_VARIANTS = [("ntsc", 1), ("ntsc", 0), ("ntsc_conv", None), ("nes", None), ("pv1k", None)]


@pytest.mark.parametrize("variant,lines2", CHROMA_VARIANTS)
@pytest.mark.parametrize("which", ["I", "Q"])
def test_fast_equaliser_chroma_edge(variant, lines2, which):
    """A saturation whose 127 * wmax fails the chroma bound; a picture that drives the I (or Q) input to +-(A * w) >> 9.
    The largest amplitude A* the guard admits is found by bisection with the path diagnostic; A* must decode on the fast
    path and A* + 1 on the wrap-exact one, both exactly, on the first pass after a monitor that did not need its lines'
    maximum (k_sync scans the lines itself) and on the next (the maximum measured during the copy)."""
    spec = layout.system_spec(variant)
    cc = spec.cc_samples
    state, x0 = _settle(variant)
    hue, sat = _edge_setting(variant, spec, state, x0)
    every = _probe(variant, state, x0, hue=hue, saturation=sat)
    recs = _picture_lines(spec, state, every)
    wmax = max(_wmax(r, cc) for r in recs)
    assert ((127 * wmax) >> 9) + 1 > 16383 and ((48 * wmax) >> 9) + 1 <= 16383, (sat, wmax)
    pos, sgn = _unit_pattern(spec, recs, which)
    base = _blank_windows(spec, recs, x0, every)
    sig = lambda a: _with(base, pos, a * sgn)
    rp = Replay(variant, 1, lines2=lines2, hue=hue, saturation=sat)

    def generic(a):
        return bool(rp.run([(0, state, sig(a))], "%s %s A=%d" % (variant, which, a))[0] & GEN)

    lo, hi = 48, 127
    assert not generic(lo) and generic(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if generic(mid):
            hi = mid
        else:
            lo = mid
    a_star = lo
    # the replayed pass locked onto the same lines as the probe (the pattern kept clear of sync and burst)
    got = [l for l in rp.b.get_lines(0) if l.beg >= 0]
    assert [(l.pos, l.hsync) for l in got] == [(r.pos, r.hsync) for r in every]
    if cc == 4:
        assert [(l.wave0, l.wave1) for l in got] == [(r.wave[0], r.wave[1]) for r in every]
        # the bisection found exactly the guard's edge: every line's max |s| is A there
        assert ((a_star * wmax) >> 9) + 1 <= 16383 < (((a_star + 1) * wmax) >> 9) + 1, (a_star, wmax)
        assert ((a_star + 1) * wmax) >> 9 == 16383, "the rejected amplitude should sit exactly on the bound"
        print("chroma edge %s %s: hue %d, saturation %d, wmax %d, A* %d, (A* * wmax) >> 9 = %d (bound 16382)" % (
            variant, which, hue, sat, wmax, a_star, (a_star * wmax) >> 9))
    for a, want in ((a_star, 0), (a_star + 1, GEN)):
        rp.configure(0, saturation=1)  # a pass that needs no maximum: the next one scans the lines in k_sync
        rp.run([(0, state, sig(a))], "%s low saturation" % variant)
        rp.configure(0, saturation=sat)
        before = rp.b.lines2_launches
        for kind in ("scanned", "measured"):
            paths = rp.run([(0, state, sig(a))], "%s %s A=%d %s" % (variant, which, a, kind))
            assert paths[0] & GEN == want, (variant, which, a, kind, paths)
        if lines2 == 1 and not want:
            assert rp.b.lines2_launches > before
        if lines2 == 0:
            assert rp.b.lines2_launches == before
    rp.b.close()


def test_fast_equaliser_chroma_struct_tail_pv1k():
    """The PV-1000's last signal line: with hsync above 4 its decode window runs three samples past inp[] into the bytes
    behind it (outw, outh, out_format, 0 -- struct CRT, crt_core.h:74-92), which no clamp or measurement sees.  With
    outw = 640 the first of them is 0x80 = -128.  A carrier with wmax just above 65536 passes the bound for |s| <= 127 but
    puts that sample's chroma input at 16384; k_sync must count |s| = 128 for the line and take the wrap-exact path."""
    variant = "pv1k"
    spec = layout.system_spec(variant)
    H = spec.hres
    state, x0 = _settle(variant)
    # the same field two lines and four samples later: vsync at 260 and hsync 7 put the last decoded line on signal line 261
    x = np.roll(x0, 2 * H + 4)
    state = dict(state, hsync=7, vsync=260)
    # the burst scaled by 0.92 and the hue turned to 152: the largest carrier value of the field (65952 at saturation 16)
    # is the one that multiplies the -128
    burst = (np.arange(spec.vres)[:, None] * H + 5 + spec.cb_beg + np.arange(50)[None, :]).ravel()
    burst = burst[burst < spec.input_size]
    x[burst] = np.round(x[burst].astype(float) * 0.92).astype(np.int8)
    state["ccf"] = np.round(np.asarray(state["ccf"]) * 0.92).astype(np.int64)
    knobs = dict(hue=152, saturation=16)
    recs = _probe(variant, state, x, **knobs)
    tail = [r for r in recs if r.pos + spec.av_len > spec.input_size]
    assert len(tail) == 1 and tail[0].pos // H == spec.vres - 1
    i0 = spec.input_size - tail[0].pos  # the -128 is sample i0 of the line's window
    wmax = max(_wmax(r, 5) for r in recs)
    at_tail = max(abs(tail[0].wave_i[i0 % 5]), abs(tail[0].wave_q[i0 % 5]))
    assert 65536 <= at_tail == wmax and ((127 * wmax) >> 9) + 1 <= 16383 < ((128 * wmax) >> 9) + 1, (at_tail, wmax)
    rp = Replay(variant, 1, **knobs)
    for kind in ("first", "second"):
        paths = rp.run([(0, state, x)], "pv1k struct tail, %s pass" % kind)
        assert paths[0] & GEN, paths
    rp.b.close()


# ---------------------------------------------------------------------------------------------------------------------
# equaliser, luma
# ---------------------------------------------------------------------------------------------------------------------

LUMA_VARIANTS = CHROMA_VARIANTS
PERIODS = (2, 6, 24, 130)


@pytest.mark.parametrize("variant,lines2", LUMA_VARIANTS)
def test_fast_equaliser_luma_edge(variant, lines2):
    """bright = brightness - (black + black_point) at +-4096 (fast) and +-4097 (wrap-exact), +-2048 / +-2049 on the
    PV-1000, under a +-127 square wave of several periods -- the luma cascade's largest overshoot.  One monitor per
    (bright, period), one launch."""
    spec = layout.system_spec(variant)
    edge = 2048 if spec.cc_samples == 5 else 4096
    brights = [edge, -edge, edge + 1, -(edge + 1)]
    state, x0 = _settle(variant)
    recs = _picture_lines(spec, state, _probe(variant, state, x0, saturation=4))
    i = np.arange(24, spec.av_len - 24)
    pos = np.concatenate([r.pos + i for r in recs])
    keep = pos < spec.input_size
    cases = [(b, p) for b in brights for p in PERIODS]
    rp = Replay(variant, len(cases), lines2=lines2, saturation=4)
    items = []
    for m, (bright, period) in enumerate(cases):
        # black_point moves `bright` as well: split the offset between the two knobs
        bp = 3 if bright > 0 else -3
        rp.configure(m, brightness=bright + spec.black + bp, black_point=bp)
        wave = np.where((np.concatenate([i for _ in recs]) // period) % 2 == 0, 127, -127)
        items.append((m, state, _with(x0, pos[keep], wave[keep])))
    before = rp.b.lines2_launches
    paths = rp.run(items, "%s luma edge" % variant)
    for m, (bright, period) in enumerate(cases):
        assert (paths[m] & GEN) == (GEN if abs(bright) > edge else 0), (variant, bright, period, paths[m])
    if lines2 == 1:
        assert rp.b.lines2_launches > before
    rp.b.close()


# ---------------------------------------------------------------------------------------------------------------------
# staged encoder: the span of a chunk
# ---------------------------------------------------------------------------------------------------------------------

K_SPAN, K_ROW, CHUNK = 192, 176, 32  # crt_kernels.cuh: kModSSpan, kModSRow, kModSChunk


def dest_width(variant):
    spec = layout.system_spec(variant)
    return (spec.av_len * 55500) >> 16 if variant.endswith("_bloom") else spec.av_len


def staged_ok(w, destw, bpp):
    """mod_staged_ok (crt_kernels.cuh): the widest source span of a chunk, ceil(32 w / destw) + 1 pixels, plus 15 bytes of
    alignment slack and 16 of copy rounding, fits the 192-byte limit"""
    span = (CHUNK * w + destw - 1) // destw + 1
    return span * bpp + 15 + 16 <= K_SPAN


def widest(destw, bpp):
    w = destw
    while staged_ok(w + 1, destw, bpp):
        w += 1
    return w


def copy_sizes(addr, w, destw, bpp, rows):
    """bytes the staged encoder copies per (row, chunk): the span f0 .. f1 of the chunk's source columns, from the
    16-byte aligned address at or below pixel f0 (crt_kernels.cuh, issue())"""
    out = []
    for row in rows:
        for c in range((destw + CHUNK - 1) // CHUNK):
            f0 = (c * CHUNK) * w // destw
            f1 = min(c * CHUNK + CHUNK - 1, destw - 1) * w // destw
            p = addr + (row * w + f0) * bpp
            out.append(((p & 15) + (f1 - f0 + 1) * bpp + 15) & ~15)
    return out


@pytest.mark.parametrize("variant,destw", [("ntsc", 753), ("ntsc_bloom", 637), ("pv1k", 1487)])
def test_staged_encoder_span_edge(variant, destw):
    """The widest source the staged encoder accepts and one pixel wider (which the gather encoder takes), 4- and 3-byte
    pixels, scaled and raw, at source addresses that make some chunk copy the whole 176-byte stage row: analog[] equal to
    the oracle's, the encoder the diagnostic reports the one expected."""
    import torch
    from ntsc_crt_b200 import capi
    assert dest_width(variant) == destw
    want = {("ntsc", 4): 917, ("ntsc", 3): 1223, ("ntsc_bloom", 4): 776, ("ntsc_bloom", 3): 1035,
            ("pv1k", 4): 1812, ("pv1k", 3): 2416}
    cases = []
    for fmt, bpp in ((layout.PIX_BGRA, 4), (layout.PIX_BGR, 3)):
        w = widest(destw, bpp)
        assert w == want[(variant, bpp)] and staged_ok(w, destw, bpp) and not staged_ok(w + 1, destw, bpp)
        for width in (w, w + 1):
            for raw in (0, 1):
                for skew in ((8, 12) if bpp == 4 else (5,)):
                    cases.append((fmt, bpp, width, raw, skew))
    n = len(cases)
    b = capi.Batch(variant, n)
    outs = [torch.zeros(48, 64, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
    h = 40
    keep, oras, imgs = [], [], []
    full = 0
    for m, (fmt, bpp, width, raw, skew) in enumerate(cases):
        img = S.pack_rgb(S.rand_image(width, h, bpp=3, seed=m), fmt)
        big = torch.zeros(img.size + 64, dtype=torch.uint8, device="cuda")
        base = (-big.data_ptr()) % 16
        dimg = big[base + skew: base + skew + img.size].view(h, width, bpp)
        dimg.copy_(torch.from_numpy(img))
        keep.append(big)
        desth = min(h, 240) if raw else 240  # (every system here decodes 240 picture lines)
        rows = sorted({(y * h) // desth for y in range(desth)})
        sizes = copy_sizes(dimg.data_ptr(), width, destw, bpp, rows)
        if staged_ok(width, destw, bpp):
            assert max(sizes) <= K_ROW
            full += max(sizes) == K_ROW
        b.set_monitor(m, outs[m], fmt=layout.PIX_BGRA, blend=0, scanlines=0)
        b.set_source(m, dimg, format=fmt, as_color=1, raw=raw, field=0, frame=0, dot_crawl_offset=m % 3)
        o = S.OracleEngine(variant, 64, 48)
        o.set(blend=0, scanlines=0)
        o.modulate(img, format=fmt, as_color=1, raw=raw, field=0, frame=0, dot_crawl_offset=m % 3)
        oras.append(o)
        imgs.append(img)
    assert full >= 4, "no staged monitor copies a whole stage row"
    b.commit_monitors()
    b.modulate()
    torch.cuda.synchronize()
    paths = b.paths()
    for m, (fmt, bpp, width, raw, skew) in enumerate(cases):
        assert bool(paths[m] & STAGED) == staged_ok(width, destw, bpp), (variant, cases[m], paths[m])
        got = b.signal(m, "analog")
        assert np.array_equal(got, oras[m].analog), "%s %r: %s" % (variant, cases[m], S.diff_report("analog", got, oras[m].analog))
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# staged encoder: the sector-aligned stores, PV-1000
# ---------------------------------------------------------------------------------------------------------------------

STORE_WIDTHS = (1, 2, 3, 4, 31, 32, 33, 63, 64, 65, 96, 97, 98, 99, 130)


def _store_cases(widths):
    """(raw width, xoffset) pairs: for every width, line starts xo at all 32 residues mod 32 (xo = xo_raw - xo_raw % 5 is a
    multiple of five: 32 consecutive ones, of both parities), half of them with xo_raw itself off the multiple"""
    spec = layout.system_spec("pv1k")
    out = []
    for w in widths:
        base = spec.av_beg + (spec.av_len - w) // 2
        m0 = -(-base // 5)
        for j in range(32):
            out.append((w, 5 * (m0 + j) - base + (j % 2) * 2))
    return out


def _check_store_cases(cases):
    import torch
    from ntsc_crt_b200 import capi
    spec = layout.system_spec("pv1k")
    b = capi.Batch("pv1k", len(cases))
    outs = [torch.zeros(8, 16, 4, dtype=torch.uint8, device="cuda") for _ in cases]
    oras, keep, residues = [], [], set()
    for m, (w, xoff) in enumerate(cases):
        h = 3 + m % 5
        img = S.rand_image(w, h, seed=100 + m)
        dimg = torch.from_numpy(img).cuda()
        keep.append(dimg)
        xo_raw = spec.av_beg + xoff + (spec.av_len - w) // 2
        residues.add((w, (xo_raw - xo_raw % 5) % 32))
        b.set_monitor(m, outs[m], fmt=layout.PIX_BGRA, blend=0, scanlines=0)
        kw = dict(format=layout.PIX_BGRA, as_color=1, raw=1, field=0, frame=m & 1, xoffset=xoff, yoffset=m % 3 - 1,
                  dot_crawl_offset=m % 4)
        b.set_source(m, dimg, **kw)
        o = S.OracleEngine("pv1k", 16, 8)
        o.set(blend=0, scanlines=0)
        o.modulate(img, **kw)
        oras.append(o)
    assert all(len({r for (w2, r) in residues if w2 == w}) == 32 for w in {c[0] for c in cases})
    b.commit_monitors()
    b.modulate()
    torch.cuda.synchronize()
    paths = b.paths()
    for m in range(len(cases)):
        assert paths[m] & STAGED, (cases[m], paths[m])
        got = b.signal(m, "analog")
        assert np.array_equal(got, oras[m].analog), "pv1k %r: %s" % (cases[m], S.diff_report("analog", got, oras[m].analog))
    b.close()


def test_pv1k_staged_encoder_stores_at_every_line_phase():
    """raw pictures 1-4 samples wide (one word cut at both ends), 31-33, 63-65, and several chunks with every tail length
    mod 4, each at all 32 phases of the line start against the 32-byte sectors of analog[], xo even and odd"""
    _check_store_cases(_store_cases(STORE_WIDTHS))


# ---------------------------------------------------------------------------------------------------------------------
# burst lock
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["ntsc", "nes", "pv1k"])
def test_burst_lock_at_the_shortcut_edge(variant):
    """accumulators poked to +-(2^23 - 1), the largest magnitude the shortcut for x * 127 / 128 takes, and +-2^23, the
    smallest it leaves to the exact form (crt_sync.cuh) -- call after call, as in test_burst_lock_from_poked_accumulators"""
    nes = variant == "nes"
    img = S.nes_image(seed=11) if nes else S.rand_image(256, 240, seed=11)
    gpu = S.ProductEngine(variant, 400, 300)
    ora = S.OracleEngine(variant, 400, 300)
    kw = dict(dot_crawl_offset=1) if nes else dict(format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
    vals = [(1 << 23) - 1, -((1 << 23) - 1), 1 << 23, -(1 << 23), (1 << 23) + 1, -((1 << 23) + 1), (1 << 23) - 128]
    for e in (gpu, ora):
        e.set(blend=0, scanlines=1)
        e.modulate(img, **kw)
        tab = e.crt.ccf if hasattr(e, "crt") else e.mon.ccf
        for r in range(e.spec.vper):
            for x in range(e.spec.cc_samples):
                tab[r][x] = vals[(r * e.spec.cc_samples + x) % len(vals)]
    for it in range(3):
        for e in (gpu, ora):
            e.demodulate(0 if it == 0 else 7)
        S.assert_same_state(ora.state(), gpu.state(), "%s ccf at 2^23, call %d" % (variant, it))
