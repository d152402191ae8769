"""A seeded random sweep of the batch interface (include/crtx_batch.h) against one CPU model per monitor.

One launch serves many monitors, and this is where a batch can go wrong while every monitor alone decodes right:
  * crtx_demodulate splits its range into runs of one output geometry (outw, outh, out_format, blend, v_fac, out_pitch)
    and plans each run's line passes from the run's first monitor;
  * k_lines2 (crt_lines2.cuh) decodes two monitors per CTA, reads scanlines, brightness, contrast and the image per lane
    and hands rows between lanes; it is taken only when every image of the run starts on a 16-byte boundary;
  * crtx_modulate groups the staged encoder's launches by source (format, as_color) and leaves the sources too wide for
    a stage row to the gather kernel;
  * crtx_set_monitors uploads only what changed, and rewrites the bytes behind inp[] (the rest of the reference's
    struct CRT, which a decode window can read) when outw, outh or out_format change.
Every draw mixes what those pieces must keep apart: runs of 1 to 4 monitors on geometries on both sides of the kernels'
limits, dense images and windows of larger tensors (16-byte aligned or only 4-byte aligned, in one run), per-lane knobs
that differ inside a run (some far enough out to put a monitor on the wrap-exact equaliser), sources of every format and
size (on the band-limited systems some wider than a stage row), calls on sub-ranges in random order, reconfigurations
and poked sync states between fields.  After every field the whole state of every monitor -- out, analog, inp, ccf,
hsync, vsync, rn -- equals its CPU model's (support.oracle_engine) bit for bit, the 16 bytes behind its signal buffers
hold its geometry, and the paths the batch reports are the ones its configuration implies.  Per variant, the draws must reach each of those cross-monitor cases (COVERAGE): a draw
that stops reaching one fails rather than testing less.

Also here: one context driven from several streams over disjoint ranges, as bench.py does (device images, and
crtx_frames_host with a staging buffer that grows while other streams have work queued), and crt_resize between fields
in the drop-in interface.

The same bodies run on the CPU through the SIMT interpreter, at reduced sizes (tests/test_simt_kernels.py)."""

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import capi, layout

GEN, STAGED, ROW16 = capi.Batch.PATH_GENERIC_EQ, capi.Batch.PATH_STAGED_MOD, capi.Batch.PATH_ROW16
SENT = 0xA7  # the bytes of a canvas outside its window

# sizes of a draw (the interpreter run lowers them)
MAX_MONITORS = 8
FIELDS = 5
MAX_OUTW = 1921
# output widths k_lines2 takes (4-byte pixels, a multiple of 4 in about [528, 1312]) and widths it does not
L2_WIDTHS = (528, 640, 832, 1312)
L1_WIDTHS = (524, 333, 1921, 64)
# output heights below, at and above the 240 decoded lines (the line passes: rows shared by lines, or one pass)
HEIGHTS = (120, 239, 240, 241, 480, 624)
POKES = ((130, 700), (-50, -50), (700, 130))  # (vsync, hsync) set on a monitor before a field
# the draws of each variant; where 1, 2 and 3 did not reach every COVERAGE entry, another seed that reaches the rest
SEEDS = {v: (1, 2, 3) for v in capi.ALL_VARIANTS}
SEEDS.update(ntsc=(1, 2, 3, 4, 5), pv1k=(1, 2, 3, 4, 5), vhs=(1, 2, 3, 4, 5), nes_p1=(1, 2, 3, 10), nes_border=(1, 2, 3, 6),
             ntsc_novsync=(1, 2, 5), template=(1, 2, 5), ntsc_nohsync=(1, 2, 4))

# what every variant's draws must reach, where its build has the path
COVERAGE = ("lines2 pair differing in scanlines", "lines2 pair of a generic and a fast monitor", "demodulate of two runs",
            "modulate of staged and gather sources", "run of ROW16 and other images", "out_format changed alone",
            "outw / outh changed")


def _system(variant):
    return layout.system_spec(variant).system


def _has_lines2(variant):
    """CRTX_HAS_LINES2: the stock IIR decoder (no convolution, no bloom) at four samples per carrier period"""
    return layout.system_spec(variant).cc_samples == 4 and not layout.uses_convolution(variant) and "bloom" not in variant


def _lines2_width(variant, outw):
    """lines2_geometry_ok (crt_lines2.cuh): a multiple of 4 up to 1312 pixels whose 8-pixel blocks span at most 12 samples"""
    dx = ((layout.system_spec(variant).av_len - 1) << 12) // outw
    return outw % 4 == 0 and 16 <= outw <= 1312 and 7 * dx <= 10 * 4096


def _bandlimited(variant):
    """CRT_B200_BANDLIMITED: the RGB encoders with a staged and a gather picture kernel"""
    return _system(variant) in (layout.SYS_NTSC, layout.SYS_VHS, layout.SYS_TEMP, layout.SYS_PV1K)


def reachable(variant):
    """the COVERAGE entries the variant's build has"""
    got = set(COVERAGE)
    if not _has_lines2(variant):
        got -= {COVERAGE[0], COVERAGE[1]}
    if not _bandlimited(variant):
        got.discard(COVERAGE[3])
    if "bloom" in variant:  # (the bloom build never writes 16-byte rows)
        got.discard(COVERAGE[4])
    return got


# ---------------------------------------------------------------------------------------------------------------------
# the draw
# ---------------------------------------------------------------------------------------------------------------------

def _ri(rng, lo, hi):
    return int(rng.integers(lo, hi))


def draw_geometry(rng, kind="any"):
    """one run's output geometry: size, pixel format, blend, v_fac, and the canvas its images are windows of (cw, the
    canvas width in pixels, None for dense images) with where in it they sit (align).  kind "lines2": 4-byte pixels, a
    width k_lines2 takes and rows for every line, dense or 16-byte aligned windows; "mixed": 4-byte pixels in 16-byte
    aligned and unaligned windows of one pitch; "any": anywhere in the pools."""
    widths = [w for w in L2_WIDTHS + L1_WIDTHS if w <= MAX_OUTW]
    g = dict(outw=int(rng.choice(widths)), outh=int(rng.choice(HEIGHTS)), fmt=_ri(rng, 0, 6), blend=_ri(rng, 0, 2),
             v_fac=_ri(rng, 1, 6) if rng.random() < 0.15 else 0, cw=None, align="any")
    if kind != "any":
        g["fmt"] = int(rng.choice([layout.PIX_ARGB, layout.PIX_RGBA, layout.PIX_ABGR, layout.PIX_BGRA]))
        if kind == "lines2":
            g.update(outw=int(rng.choice([w for w in L2_WIDTHS if w <= MAX_OUTW])), outh=int(rng.choice([h for h in HEIGHTS if h >= 240])),
                     align="all16")
        else:
            g.update(outw=int(rng.choice([w for w in widths if w % 4 == 0])), align="mixed")
    if g["align"] == "mixed" or rng.random() < 0.4:
        g["cw"] = draw_canvas(rng, g)
    return g


def draw_canvas(rng, g):
    """the width of a canvas whose row-pitched windows hold a run's images: a pitch of 16-byte multiples (always where
    the run's images are to be 16-byte aligned, mostly otherwise) or only of 4"""
    pad = _ri(rng, 4, 17)
    if g["align"] != "any" or rng.random() < 0.75:
        pad += (-(g["outw"] + pad)) % 4
    return g["outw"] + pad


def draw_offset(rng, g, k):
    """the column of the k-th image of a run in its canvas: 16-byte aligned (4-byte pixels at a multiple of 4), or,
    where the run mixes them, aligned and not by turns"""
    room = g["cw"] - g["outw"]
    if g["align"] == "any":
        return _ri(rng, 0, room + 1)
    if g["align"] == "mixed" and k % 2:
        at = 4 * _ri(rng, 0, (room - 1) // 4 + 1)
        return at + _ri(rng, 1, min(3, room - at) + 1)
    return 4 * _ri(rng, 0, room // 4 + 1)


def draw_knobs(rng, g):
    k = dict(hue=_ri(rng, 0, 360), brightness=_ri(rng, -20, 21), contrast=_ri(rng, 150, 211), saturation=_ri(rng, 0, 20),
             black_point=_ri(rng, 0, 8), white_point=_ri(rng, 88, 101), scanlines=_ri(rng, 0, 2), blend=g["blend"],
             v_fac=g["v_fac"])
    if rng.random() < 0.15:  # far out: the wrap-exact equaliser (|bright| above 4096, or a large carrier)
        if rng.random() < 0.7:
            k["brightness"] = int(rng.choice([-1, 1])) * _ri(rng, 4300, 6000)
        else:
            k["saturation"] = _ri(rng, 40, 120)
    return k


def draw_monitor(rng, variant, g, k):
    m = dict(outw=g["outw"], outh=g["outh"], fmt=g["fmt"], noise=_ri(rng, 0, 40) if rng.random() < 0.8 else 0,
             knobs=draw_knobs(rng, g), geo=g)
    if g["cw"] is not None:
        m["off"] = draw_offset(rng, g, k)
    if _system(variant) == layout.SYS_VHS:
        m["seed"] = _ri(rng, 0, 1 << 31)
    return m


def draw_monitors(rng, variant, n):
    """n monitors in runs of 1 to 4 that share a geometry, the runs' kinds (draw_geometry) taken in turn from a shuffled
    list of the three"""
    mons, kinds = [], []
    while len(mons) < n:
        kinds = kinds or [str(k) for k in rng.permutation(["lines2", "mixed", "any"])]
        kind = kinds.pop()
        g = draw_geometry(rng, kind)
        size = _ri(rng, 2, 5) if kind != "any" else _ri(rng, 1, 5)
        for k in range(min(size, n - len(mons))):
            mons.append(draw_monitor(rng, variant, g, k))
    return mons


def _reads_row_h(variant, h, raw):
    """whether the reference's band-limited encoders read row h, one past an image of h rows, in field 1: the field's
    row offset pushes the last picture row's source row to h (crt_ntsc.c:258-263), whose bytes are not the image's"""
    full = (layout.system_spec(variant).lines * (63500 if "bloom" in variant else 64500)) >> 16
    desth = min(h, full) if raw else full
    return ((desth - 1) * h) // desth + (h + desth) // desth // 2 >= h


def draw_source(rng, variant, m, it):
    """(numpy image, batch settings) of one monitor's field"""
    sysm = _system(variant)
    seed = _ri(rng, 0, 1 << 30)
    if sysm == layout.SYS_NES:
        img = S.nes_image(_ri(rng, 32, 257), _ri(rng, 32, 241), seed=seed)
        kw = dict(dot_crawl_offset=_ri(rng, 0, 3), hue=_ri(rng, 0, 360), xoffset=_ri(rng, 0, 13), yoffset=_ri(rng, 0, 3),
                  reinit=int(it == 0 or rng.random() < 0.2))
        if layout.system_spec(variant).border:
            kw["border_color"] = _ri(rng, 0, 512)
        return img, kw
    fmt = _ri(rng, 0, 6)
    wide = _bandlimited(variant) and rng.random() < 0.3  # wider than a stage row: the gather encoder
    w, h = (_ri(rng, 1100, 2200), _ri(rng, 8, 120)) if wide else (_ri(rng, 16, 700), _ri(rng, 8, 300))
    img = S.rand_image(w, h, bpp=layout.bpp4fmt(fmt), seed=seed)
    kw = dict(format=fmt, hue=_ri(rng, 0, 360), xoffset=_ri(rng, 0, 13), yoffset=_ri(rng, 0, 3), dot_crawl_offset=_ri(rng, 0, 4))
    if sysm == layout.SYS_NESRGB:
        kw["reinit"] = int(it == 0 or rng.random() < 0.2)
        return img, kw
    kw.update(as_color=int(rng.random() < 0.8), raw=int(rng.random() < 0.2), field=_ri(rng, 0, 2), frame=_ri(rng, 0, 2))
    if sysm != layout.SYS_SNES and _reads_row_h(variant, h, kw["raw"]):
        kw["field"] = 0
    if sysm == layout.SYS_VHS:  # (aberrations on monitors without blend, as tests/test_gpu_sync_switches.py)
        kw["do_aberration"] = int(not m["knobs"]["blend"] and rng.random() < 0.3)
    return img, kw


def draw_calls(rng, n):
    """one field's calls: [(first, count)] for the modulates and, separately ordered, the demodulates.  Either the whole
    batch, or two or three disjoint sub-ranges in random order, some of which may sit the field out."""
    if n < 2 or rng.random() < 0.5:
        return [(0, n)], [(0, n)]
    cuts = sorted(rng.choice(np.arange(1, n), size=min(n - 1, _ri(rng, 1, 3)), replace=False).tolist())
    parts = [(a, b - a) for a, b in zip([0] + cuts, cuts + [n])]
    parts = [p for p in parts if rng.random() < 0.8] or parts[:1]
    mod = [parts[k] for k in rng.permutation(len(parts))]
    dem = [parts[k] for k in rng.permutation(len(parts))]
    return mod, dem


# ---------------------------------------------------------------------------------------------------------------------
# images
# ---------------------------------------------------------------------------------------------------------------------

def make_out(m):
    """(image tensor, (canvas, column offset) or None): a dense zeroed image, or a zeroed window of a SENT canvas"""
    import torch
    bpp = max(1, layout.bpp4fmt(m["fmt"]))
    g = m["geo"]
    if g["cw"] is None:
        return torch.zeros(m["outh"], m["outw"], bpp, dtype=torch.uint8, device="cuda"), None
    canvas = torch.full((m["outh"], g["cw"], bpp), SENT, dtype=torch.uint8, device="cuda")
    view = canvas[:, m["off"]:m["off"] + m["outw"]]
    view.zero_()
    return view, (canvas, m["off"])


def describe(m):
    g = m["geo"]
    return "%dx%d fmt %d blend %d v_fac %d %s noise %d knobs %s%s" % (
        m["outw"], m["outh"], m["fmt"], g["blend"], g["v_fac"],
        "dense" if g["cw"] is None else "window at px %d of %d" % (m["off"], g["cw"]), m["noise"],
        {k: v for k, v in m["knobs"].items() if k not in ("blend", "v_fac")}, " seed %d" % m["seed"] if "seed" in m else "")


# ---------------------------------------------------------------------------------------------------------------------
# the sweep
# ---------------------------------------------------------------------------------------------------------------------

def _runs(rig, first, count):
    """the line-pass runs of crtx_demodulate over [first, first + count): consecutive monitors of one geometry"""
    key = lambda i: (rig.mons[i]["outw"], rig.mons[i]["outh"], rig.mons[i]["fmt"], rig.b.monitors[i].blend,
                     rig.b.monitors[i].v_fac, rig.b.monitors[i].out_pitch)
    runs, lo = [], first
    for i in range(first + 1, first + count + 1):
        if i == first + count or key(i) != key(lo):
            runs.append(list(range(lo, i)))
            lo = i
    return runs


def sweep(variant, seed):
    """one seeded draw of monitors and fields on `variant`, checked after every field; returns the COVERAGE entries it
    reached"""
    import torch
    rng = np.random.default_rng([seed, sum(map(ord, variant))])
    n = int(rng.choice(np.arange(1, MAX_MONITORS + 1), p=np.arange(1, MAX_MONITORS + 1) / (MAX_MONITORS * (MAX_MONITORS + 1) / 2)))
    mons = draw_monitors(rng, variant, n)
    made = [make_out(m) for m in mons]
    canvases = [c for _, c in made]
    rig = S.BatchRig(variant, mons, outs=[o for o, _ in made])
    lines2 = _has_lines2(variant)
    reached = set()
    pending = {}  # monitor -> the COVERAGE entry of its reconfiguration, reached once the monitor is next decoded
    history = []

    def where(it, i=None):
        return "%s seed %d field %d%s (reproduce: test_gpu_batch_fuzz.sweep(%r, %d)); history %s" % (
            variant, seed, it, "" if i is None else " monitor %d [%s]" % (i, describe(rig.mons[i])), variant, seed,
            "; ".join(history[-6:]))

    for it in range(FIELDS):
        # reconfigurations and pokes between fields
        if it > 0 and rng.random() < 0.5:
            for i in sorted(rng.choice(n, size=_ri(rng, 1, max(2, n // 2 + 1)), replace=False).tolist()):
                old = rig.mons[i]
                kind = str(rng.choice(["format", "size", "knobs", "image"], p=[0.3, 0.3, 0.2, 0.2]))
                g = dict(old["geo"])
                if kind == "format":
                    g["fmt"] = int(rng.choice([f for f in range(6) if f != old["fmt"]]))
                elif kind == "size":
                    g2 = draw_geometry(rng)
                    g.update(outw=g2["outw"], outh=g2["outh"], cw=None)
                elif kind == "image":  # (at another pitch: its run's neighbours keep the geometry, not the pitch)
                    g["cw"] = None if g["cw"] is not None and rng.random() < 0.5 else draw_canvas(rng, g)
                m = dict(old, fmt=g["fmt"], outw=g["outw"], outh=g["outh"], geo=g)
                if kind == "knobs":
                    m["knobs"] = draw_knobs(rng, g)
                    m["noise"] = _ri(rng, 0, 40)
                keep = kind == "knobs" or (kind == "format" and layout.bpp4fmt(g["fmt"]) == layout.bpp4fmt(old["fmt"]))
                if keep:
                    rig.reconfigure(i, m)
                else:
                    if g["cw"] is not None:
                        m["off"] = draw_offset(rng, g, _ri(rng, 0, 2))
                    out, canvases[i] = make_out(m)
                    rig.reconfigure(i, m, out)
                if kind == "format":
                    pending[i] = "out_format changed alone"
                elif kind == "size":
                    pending[i] = "outw / outh changed"
                history.append("field %d: monitor %d %s -> %s" % (it, i, kind, describe(m)))
        if it > 0 and rng.random() < 0.3:
            i = _ri(rng, 0, n)
            vs, hs = POKES[_ri(rng, 0, len(POKES))]
            st = rig.b.get_state(first=i, count=1)
            st[0].vsync, st[0].hsync = vs, hs
            rig.b.set_state(st, first=i)
            rig.oras[i].set(vsync=vs, hsync=hs)
            history.append("field %d: monitor %d poked vsync %d hsync %d" % (it, i, vs, hs))

        for i in range(n):
            img, kw = draw_source(rng, variant, rig.mons[i], it)
            rig.source(i, img, **kw)
        mod, dem = draw_calls(rng, n)
        history.append("field %d: modulate %s, demodulate %s" % (it, mod, dem))
        for first, count in mod:
            rig.modulate(first, count)
            paths = rig.b.paths(first, count)
            if _bandlimited(variant):
                takes = [bool(p & STAGED) for i, p in zip(range(first, first + count), paths)
                         if layout.bpp4fmt(rig.b.sources[i].format)]
                if any(takes) and not all(takes):
                    reached.add("modulate of staged and gather sources")
        for first, count in dem:
            before = rig.b.lines2_launches
            rig.demodulate(first, count)
            paths = dict(zip(range(first, first + count), rig.b.paths(first, count)))
            runs = _runs(rig, first, count)
            reached.update(pending.pop(i) for i in range(first, first + count) if i in pending)
            if len(runs) > 1:
                reached.add("demodulate of two runs")
            want = 0
            for run in runs:
                row16 = [bool(paths[i] & ROW16) for i in run]
                if any(row16) and not all(row16):
                    reached.add("run of ROW16 and other images")
                m0 = rig.mons[run[0]]
                if lines2 and all(row16) and _lines2_width(variant, m0["outw"]) and m0["outh"] + m0["knobs"]["v_fac"] >= rig.b.spec.lines:
                    want += 1  # k_lines2: one pass of the run, two monitors per CTA
                    for a in range(0, len(run) - 1, 2):
                        x, y = rig.mons[run[a]]["knobs"], rig.mons[run[a + 1]]["knobs"]
                        # (scanlines shortens the rows a line writes only where lines own more than one row)
                        if x["scanlines"] != y["scanlines"] and m0["outh"] + m0["knobs"]["v_fac"] > rig.b.spec.lines:
                            reached.add("lines2 pair differing in scanlines")
                        if bool(paths[run[a]] & GEN) != bool(paths[run[a + 1]] & GEN):
                            reached.add("lines2 pair of a generic and a fast monitor")
            assert rig.b.lines2_launches - before == want, "%s: %d k_lines2 launches, the runs %s imply %d" % (
                where(it), rig.b.lines2_launches - before, runs, want)
        try:
            rig.check(where(it))
        except AssertionError as e:
            raise AssertionError("%s\n%s" % (e, where(it))) from None
        torch.cuda.synchronize()
        for i, c in enumerate(canvases):
            if c is not None:
                a, off = c[0].cpu().numpy(), c[1]
                pad = np.concatenate([a[:, :off], a[:, off + rig.mons[i]["outw"]:]], axis=1)
                assert (pad == SENT).all(), "a byte outside the image changed: %s" % where(it, i)
    rig.close()
    return reached


@pytest.mark.gpu
@pytest.mark.parametrize("variant", capi.ALL_VARIANTS)
def test_random_batches_match_the_oracle(variant):
    """every seed of the variant's sweep, then the cross-monitor cases the seeds reached together"""
    reached = set()
    for seed in SEEDS[variant]:
        reached |= sweep(variant, seed)
    missing = reachable(variant) - reached
    assert not missing, "%s: seeds %s never reached %s" % (variant, SEEDS[variant], sorted(missing))


# ---------------------------------------------------------------------------------------------------------------------
# several streams over one context
# ---------------------------------------------------------------------------------------------------------------------

def make_streams(k):
    """k CUDA streams for one context (the interpreter run gives stand-ins)"""
    import torch
    return [torch.cuda.Stream() for _ in range(k)]


def on_stream(s):
    """the torch context that enqueues copies on s"""
    import torch
    return torch.cuda.stream(s)


STREAM_GEOMETRIES = ((832, 624, layout.PIX_BGRA, 1), (524, 300, layout.PIX_RGB, 0), (640, 480, layout.PIX_BGRA, 0),
                     (333, 241, layout.PIX_ARGB, 1))


def check_streams(variant, host, n_streams=3, per=2, fields=4):
    """n_streams streams, each owning `per` monitors of mixed geometries, enqueue `fields` fields with no host
    synchronisation between them; after each field's decode every image is copied, on its stream, into a buffer of its
    own.  One synchronisation, then every field's image and the final state against the CPU models.  host: the fields
    go through crtx_frames_host on page-locked images, and in field 2 the last stream's first monitor gets a source
    larger than any before, so the staging buffer grows while the other streams have work queued."""
    import torch
    n = n_streams * per
    rng = np.random.default_rng(7)
    mons = []
    for i in range(n):
        w, h, fmt, blend = STREAM_GEOMETRIES[i % len(STREAM_GEOMETRIES)]
        m = dict(outw=w, outh=h, fmt=fmt, noise=5 * i, knobs=dict(blend=blend, scanlines=i & 1, hue=11 * i, saturation=8 + i))
        if _system(variant) == layout.SYS_VHS:
            m["seed"] = 10 + i
        mons.append(m)
    rig = S.BatchRig(variant, mons)
    nes = _system(variant) == layout.SYS_NES
    srcs = []  # [field][monitor] = (numpy image, settings, device or page-locked host tensor)
    for it in range(fields):
        row = []
        for i in range(n):
            big = host and it == 2 and i == (n_streams - 1) * per
            if nes:
                img = S.nes_image(256 if big else 200, 240 if big else 180, seed=100 * it + i)
                kw = dict(dot_crawl_offset=(it + i) % 3, reinit=int(it == 0))
            else:
                w, h = (700, 480) if big else (int(rng.integers(200, 320)), int(rng.integers(150, 200)))
                img = S.rand_image(w, h, seed=100 * it + i)
                kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=(it >> 1) & 1, dot_crawl_offset=it % 3)
            t = torch.from_numpy(img.view(np.int16) if nes else img)
            row.append((img, kw, t.pin_memory() if host else t.cuda()))
        srcs.append(row)
    snaps = [[torch.empty_like(o) for o in rig.outs] for _ in range(fields)]
    hosts = [torch.zeros(tuple(o.shape), dtype=torch.uint8).pin_memory() for o in rig.outs]
    streams = make_streams(n_streams)
    torch.cuda.synchronize()  # (the uploads above ran on the default stream, which the side streams do not wait for)
    for it in range(fields):
        for q, s in enumerate(streams):
            first = q * per
            for i in range(first, first + per):
                img, kw, t = srcs[it][i]
                rig.b.set_source(i, t, **kw)
            if host:
                rig.b.frames_host([hosts[i].data_ptr() for i in range(first, first + per)], stream=s.cuda_stream, first=first,
                                  count=per)
            else:
                rig.b.modulate(stream=s.cuda_stream, first=first, count=per)
                rig.b.demodulate(stream=s.cuda_stream, first=first, count=per)
            with on_stream(s):
                for i in range(first, first + per):
                    snaps[it][i].copy_(rig.outs[i])
    torch.cuda.synchronize()
    for it in range(fields):
        for i in range(n):
            img, kw, _ = srcs[it][i]
            rig.oras[i].modulate(img, **S.oracle_settings(rig.b.spec.system, kw))
            rig.oras[i].demodulate(mons[i]["noise"])
            got, want = snaps[it][i].cpu().numpy(), rig.oras[i].out
            assert np.array_equal(got, want), "%s host %d field %d monitor %d (stream %d): %s" % (
                variant, host, it, i, i // per, S.diff_report("out", got, want))
    rig.check("%s host %d, after %d fields on %d streams" % (variant, host, fields, n_streams))
    if host:
        for i in range(n):  # rows no field wrote are zero on both sides
            assert np.array_equal(hosts[i].numpy(), rig.oras[i].out), "%s host image of monitor %d" % (variant, i)
    rig.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host", [0, 1])
@pytest.mark.parametrize("variant", ["ntsc", "pv1k", "nes", "vhs"])
def test_streams_over_disjoint_ranges_of_one_context(variant, host):
    check_streams(variant, host)


# ---------------------------------------------------------------------------------------------------------------------
# crt_resize between fields, in the drop-in interface
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ntsc", "pv1k"])
def test_dropin_resize_between_fields(variant):
    gpu, ora, ref = S.trio(variant, 640, 480)
    engines = [e for e in (gpu, ora, ref) if e is not None]
    for e in engines:
        e.set(blend=1, scanlines=1)
    S.resize_sequence(variant, engines, lambda what: S.check(gpu, ora, ref, what))
