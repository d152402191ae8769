"""Stage-by-stage GPU diagnostics (not a pytest file): run on an H100, prints where the CUDA
pipeline first departs from the oracle.  python tests/gpu_diag.py [variant]"""
import sys
import traceback

import numpy as np

import os
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import support as S
from ntsc_crt_b200 import capi, layout


def stage_check(variant, outw, outh, noise, generic, blend=1, scanlines=1, fields=2):
    import torch
    spec = layout.system_spec(variant)
    tag = "%s %dx%d noise=%d generic=%d" % (variant, outw, outh, noise, generic)
    print("=== " + tag)
    nes = spec.system == layout.SYS_NES
    img = S.nes_image(seed=5) if nes else S.rand_image(832, 624, seed=3)
    dimg = torch.from_numpy(img.view(np.int16) if nes else img).cuda()
    b = capi.Batch(variant, 1)
    b.set_option("generic_eq", generic)
    out = torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda")
    b.set_monitor(0, out, noise=noise, blend=blend, scanlines=scanlines)
    b.commit_monitors()
    ora = S.OracleEngine(variant, outw, outh)
    ora.set(blend=blend, scanlines=scanlines)
    ok = True
    for f in range(fields):
        if nes:
            kw = dict(dot_crawl_offset=f % 3, hue=0)
            b.set_source(0, dimg, reinit=1 if f == 0 else 0, **kw)
        else:
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=0)
            b.set_source(0, dimg, **kw)
        b.modulate()
        ora.modulate(img, **kw)
        torch.cuda.synchronize()
        a = b.signal(0, "analog")
        print(" field %d " % f + S.diff_report("analog", a, ora.analog))
        if not np.array_equal(a, ora.analog):
            ok = False
            bad = np.argwhere(a != ora.analog)[:, 0]
            ln, col = bad // spec.hres, bad % spec.hres
            print("   lines with diffs:", sorted(set(ln.tolist()))[:20], "cols min/max", col.min(), col.max())
            b.write_signal(0, ora.analog, "analog")  # continue downstream from the correct signal
        st = b.get_state()
        ccf = np.array([[st[0].ccf[r][x] for x in range(4)] for r in range(spec.vper)])
        if not np.array_equal(ccf, ora.ccf):
            ok = False
            print("   ccf after modulate differs: got %r want %r" % (ccf.tolist(), ora.ccf.tolist()))
        b.demodulate()
        ora.noise_pass(noise)
        field, table = ora.sync_pass()
        ora.line_pass(table)
        torch.cuda.synchronize()
        i = b.signal(0, "inp")
        print(" field %d " % f + S.diff_report("inp", i, ora.inp))
        ok &= np.array_equal(i, ora.inp)
        lines = b.get_lines(0)
        nbad = 0
        for k in range(spec.lines):
            g, w = lines[k], table[k]
            want = (w.pos, w.wave[0], w.wave[1], -1 if w.skip else w.beg, -1 if w.skip else w.end, w.hsync)
            got = (g.pos, g.wave0, g.wave1, g.beg, g.end, g.hsync)
            if w.skip:
                want, got = want[3:], got[3:]
            if got != want:
                if nbad < 4:
                    print("   line %d table: got %r want %r" % (k, got, want))
                nbad += 1
        print(" field %d line table: %d/%d lines differ" % (f, nbad, spec.lines))
        ok &= nbad == 0
        st = b.get_state()
        got = (st[0].hsync, st[0].vsync, st[0].rn)
        want = (ora.hsync, ora.vsync, ora.rn)
        print(" field %d state hsync/vsync/rn: got %r want %r %s" % (f, got, want, "OK" if got == want else "DIFF"))
        ok &= got == want
        o = out.cpu().numpy()
        print(" field %d " % f + S.diff_report("out", o, ora.out))
        if not np.array_equal(o, ora.out):
            ok = False
            bad = np.argwhere(o != ora.out)
            rows = sorted(set(bad[:, 0].tolist()))
            print("   rows with diffs: %d, first %r; cols min/max %d %d; channels %r" % (
                len(rows), rows[:12], bad[:, 1].min(), bad[:, 1].max(), sorted(set(bad[:, 2].tolist()))))
            r0 = rows[0]
            cols = bad[bad[:, 0] == r0][:, 1]
            print("   row %d: %d bad px, first cols %r" % (r0, len(set(cols.tolist())), sorted(set(cols.tolist()))[:10]))
            c0 = int(cols[0])
            print("   got  ", o[r0, c0:c0 + 4].tolist())
            print("   want ", ora.out[r0, c0:c0 + 4].tolist())
            out.copy_(torch.from_numpy(ora.out))
    b.close()
    print(" RESULT %s: %s" % (tag, "PASS" if ok else "FAIL"))
    return ok


def main():
    variants = sys.argv[1:] or ["ntsc"]
    results = []
    for v in variants:
        for cfg in [dict(noise=0, generic=1), dict(noise=0, generic=0), dict(noise=24, generic=0)]:
            try:
                results.append(stage_check(v, 832, 624, **cfg))
            except Exception:
                traceback.print_exc()
                results.append(False)
        try:
            results.append(stage_check(v, 640, 480, 12, 0, blend=0, scanlines=1, fields=3))
            results.append(stage_check(v, 256, 240, 0, 0, blend=0, scanlines=0, fields=2))
        except Exception:
            traceback.print_exc()
            results.append(False)
    print("DIAG SUMMARY: %d/%d stage checks passed" % (sum(bool(r) for r in results), len(results)))


if __name__ == "__main__":
    main()
