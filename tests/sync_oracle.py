"""TEST INFRASTRUCTURE: the CPU model of the decoder with its sync searches off (CRT_DO_VSYNC 0 / CRT_DO_HSYNC 0,
crt_core.h:71-72), on top of the stock oracle.

The switches change only the sync pre-pass of crt_demodulate:
  * CRT_DO_VSYNC 0 (crt_core.c:323-342): the 2W candidate lines around vsync are searched in analog[] -- before any noise
    -- for the field only; vsync is set to -3 and the lines are decoded from there.  The "gave up" case leaves
    j == CRT_HRES, so field 1, as the stock search does.
  * CRT_DO_HSYNC 0 (crt_core.c:446-450): the hsync search still runs but its result is dropped: hsync is 0 after every
    decoded line.  The search has no side effect, so the model does not run it.
SyncOracleEngine runs support.OracleEngine's encoders, noise pass and line pass and does this sync pass itself, in the
oracle's 32-bit arithmetic.  It is pinned against the reference built with the switches off (oracle/Makefile) by
tests/test_oracle_sync_switches.py.
"""
import ctypes as C

import numpy as np

import support as S

# every system of the reference, under the name of its stock library, and the three switch sets (layout.SYNC_SUFFIXES)
SYSTEMS = ("ntsc", "vhs", "nes", "snes", "nesrgb", "template", "pv1k")
SWITCHES = ("novsync", "nohsync", "nosync")
OCRT_PAD = 2048  # oracle/crt_oracle.h: slack after the oracle's signal buffers


def _i32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def _cdiv(a, b):
    """C's truncating division"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _cmod(a, b):
    return a - b * _cdiv(a, b)


class SyncOracleEngine(S.OracleEngine):
    """support.OracleEngine for a build with CRT_DO_VSYNC and / or CRT_DO_HSYNC off"""

    def __init__(self, variant, *a, **kw):
        super().__init__(variant, *a, **kw)
        assert not (self.spec.do_vsync and self.spec.do_hsync), variant

    def demodulate(self, noise=0):
        if self.lib.ocrt_bpp(self.mon.out_format) == 0:  # crt_core.c:312-315
            return
        self.noise_pass(noise)
        field, table = self.sync_pass()
        self.line_pass(table)

    def _sincos(self, n):
        sn, cs = C.c_int(), C.c_int()
        self.lib.ocrt_sincos14(C.byref(sn), C.byref(cs), n)
        return sn.value, cs.value

    def sync_pass(self):
        """crt_core.c:318-320, 323-342, 369-479 with the switches of this build: fills one record per decoded line,
        updates vsync, hsync and ccf, and returns the field"""
        o, m, spec = self.sys.contents, self.mon, self.spec
        H, V, CC = o.hres, o.vres, o.cc_samples
        table = (S.OLine * o.lines)()
        analog = np.ctypeslib.as_array(m.analog, shape=(o.input_size,)).astype(np.int64)
        inp_arr = np.ctypeslib.as_array(m.inp, shape=(o.input_size + OCRT_PAD,)).astype(np.int64)
        inp = inp_arr.tolist()
        sn, cs = self._sincos(_cdiv(_i32((_cmod(m.hue, 360) + 33) * 8192), 180))
        huesn, huecs = sn >> 11, cs >> 11

        # vsync: the stock search in inp[] (crt_core.c:379-396), or the field search in analog[] (crt_core.c:323-341)
        sig = inp_arr if spec.do_vsync else analog
        thresh = o.vsync_thresh * o.sync_level
        line, j = 0, 0
        for i in range(-o.vsync_window, o.vsync_window):
            line = (m.vsync + i) % V
            hit = np.nonzero(np.cumsum(sig[line * H:(line + 1) * H]) <= thresh)[0]
            if len(hit):
                j = int(hit[0])
                break
            j = H
        m.vsync = line if spec.do_vsync else -3
        field = int(j > H // 2)
        ratio = (_cdiv(_i32(m.outh << 16), o.lines) + 32768) >> 16  # crt_core.c:404-405
        field *= _cdiv(ratio, 2)

        span = (m.outh + m.v_fac) & 0xFFFFFFFF
        hthresh = o.hsync_thresh * o.sync_level
        for k in range(o.lines):
            rec = table[k]
            line = o.top + k
            rec.beg = _i32(((k * span) & 0xFFFFFFFF) // o.lines + (field & 0xFFFFFFFF))  # crt_core.c:428-432
            rec.end = _i32((((k + 1) * span) & 0xFFFFFFFF) // o.lines + (field & 0xFFFFFFFF))
            if rec.beg >= m.outh:
                rec.skip = 1
                rec.hsync = m.hsync
                continue
            if rec.end > m.outh:
                rec.end = m.outh
            ln = ((line + m.vsync) % V) * H
            if spec.do_hsync:  # crt_core.c:437-447
                base = ln + m.hsync + o.sync_beg
                assert base - o.hsync_window >= 0, "hsync window before the signal (outside the parity domain)"
                acc, i = 0, o.hsync_window
                for t in range(-o.hsync_window, o.hsync_window):
                    acc += inp[base + t]
                    if acc <= hthresh:
                        i = t
                        break
                m.hsync = (i + m.hsync) % H
            else:  # crt_core.c:448-449
                m.hsync = 0
            hs = m.hsync
            rec.hsync = hs
            ypos = (line + m.vsync + 3) % V  # crt_core.c:452-454 (xnudge -3, ynudge +3)
            rec.pos = (o.av_beg + hs - 3) % H + ypos * H

            row = ypos % o.cc_vper  # crt_core.c:456-467
            ccr = [m.ccf[row][p] for p in range(CC)]
            start = ln + ((hs & ~3) if CC == 4 else hs - _cmod(hs, CC))
            for i in range(o.cb_beg, o.cb_beg + o.burst_len):
                p = i % CC
                ccr[p] = _i32(_cdiv(_i32(ccr[p] * 127), 128) + inp[start + i])
            for p in range(CC):
                m.ccf[row][p] = ccr[p]

            sat = m.saturation
            if CC == 4:  # crt_core.c:469-479
                pa = hs & 3
                dci = _i32(ccr[(pa + 1) & 3] - ccr[(pa + 3) & 3])
                dcq = _i32(ccr[(pa + 2) & 3] - ccr[pa])
                w0 = _i32((_i32(_i32(dci * huecs) - _i32(dcq * huesn)) >> 4) * sat)
                w1 = _i32((_i32(_i32(dcq * huecs) + _i32(dci * huesn)) >> 4) * sat)
                rec.wave[0], rec.wave[1], rec.wave[2], rec.wave[3] = w0, w1, _i32(-w0), _i32(-w1)
            else:  # crt_core.c:480-509
                pa = hs % CC
                peak = pa + CC // 4
                dci = _i32(ccr[peak % CC] - _cdiv(_i32(ccr[(peak + CC // 2) % CC] + ccr[(peak + CC // 2 + 1) % CC]), 2))
                dcq = _i32(ccr[(pa + CC // 2) % CC] - ccr[pa])
                ang = _cmod(m.hue, 360)
                for i in range(CC):
                    sn, cs = self._sincos(_cdiv(_i32(ang * 8192), 180))
                    rec.wave_i[i] = _i32((_i32(_i32(dci * cs) + _i32(dcq * sn)) >> 15) * sat)
                    sn, cs = self._sincos(_cdiv(_i32((ang + 90) * 8192), 180))
                    rec.wave_q[i] = _i32((_i32(_i32(dci * cs) + _i32(dcq * sn)) >> 15) * sat)
                    ang += 360 // CC
        return field, table

