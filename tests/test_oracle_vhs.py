"""The random VHS cases of tests/test_gpu_vhs.py, run on the CPU between the oracle and the COMPILED REFERENCE
(oracle/_ref, else its states recorded in tests/golden/ref_states.json): every case the GPU tests draw lies inside the
reference's defined behaviour, so a GPU mismatch there is a bug of the library, never an artefact of undefined reads.

The reference draws from libc rand(): RefEngine(seed=s) calls srand(s) before the reference runs, and the oracle runs
its replica of glibc's generator from the same seed.

Where the sync pulses of the last lines are lost -- to an aberration, to loud noise, or to the head-switching wobble the
VHS noise pass puts on the bottom of every field -- hsync can run away, and the reference then reads a decode window
past inp[] into the rest of struct CRT, which holds a pointer.  Those rows are outside the parity
domain and are masked in both images, as tests/test_oracle_vs_ref.py::test_vhs does; blend 0 keeps them from leaking
into later fields.  `CRT_RECORD_REF=1 python -m pytest tests/test_oracle_vhs.py` records the reference's side afresh.
"""
import numpy as np
import pytest

import support as S
import test_gpu_vhs as V
from ntsc_crt_b200 import layout


def demodulate_masked(ref, ora, noise):
    """demodulate both (the oracle in its three stages, to see every line's decode window) and return both states with
    the rows whose window leaves inp[] zeroed, in the states and in both images"""
    ref.demodulate(noise)
    ora.noise_pass(noise)
    _, table = ora.sync_pass()
    ora.line_pass(table)
    a, b = ref.state(), ora.state()
    for rec in table:
        if not rec.skip and rec.pos + ora.spec.av_len > ora.spec.input_size:
            b["out"][rec.beg:rec.end] = 0
            ora.out[rec.beg:rec.end] = 0
            if not isinstance(a, S.RecordedState):  # (a recorded state was recorded masked)
                a["out"][rec.beg:rec.end] = 0
                ref.out[rec.beg:rec.end] = 0
    return a, b


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5, 6])
def test_gpu_vhs_cases_are_inside_the_reference_domain(seed):
    rng = np.random.default_rng(3000 + seed)  # the stream test_gpu_vhs.test_dropin_random_cases consumes
    for case in range(V.SWEEP_CASES):
        c = V.draw_case(rng)
        ref = S.RefEngine("vhs", c["outw"], c["outh"], c["fmt"], seed=c["seed"])
        ora = S.OracleEngine("vhs", c["outw"], c["outh"], c["fmt"], seed=c["seed"])
        for e in (ref, ora):
            e.set(**c["knobs"])
        for call in range(V.SWEEP_CALLS):
            kw, noise = V.draw_call(rng, c)
            assert not kw["do_aberration"] or c["knobs"]["blend"] == 0
            assert abs(noise) <= 1 << 23
            what = "seed %d case %d call %d (%r, noise %d)" % (seed, case, call, kw, noise)
            for e in (ref, ora):
                e.modulate(c["img"], **kw)
            S.assert_same_state(ref.state(), ora.state(), "modulate " + what)
            a, b = demodulate_masked(ref, ora, noise)
            S.assert_same_state(a, b, "demodulate " + what)


@pytest.mark.parametrize("seed", [1, 0xFFFFFFFF])
def test_unknown_source_format_draws_no_aberration(seed):
    """a field whose source has an unknown format and do_aberration set, then ordinary fields: the reference returns
    before the aberration draw (crt_ntscvhs.c:191-193 against :205-207), so the first modulate draws nothing"""
    img = S.bars_image(400, 300)
    ref = S.RefEngine("vhs", 400, 300, seed=seed)
    ora = S.OracleEngine("vhs", 400, 300, seed=seed)
    for e in (ref, ora):
        e.set(blend=0, scanlines=1)
    for it, (fmt, aberr) in enumerate([(9, 1), (layout.PIX_BGRA, 0), (-1, 1), (layout.PIX_BGRA, 1)]):
        for e in (ref, ora):
            e.modulate(img, format=fmt, as_color=1, field=it & 1, frame=0, do_aberration=aberr)
        S.assert_same_state(ref.state(), ora.state(), "field %d (format %d, aberration %d) modulate" % (it, fmt, aberr))
        a, b = demodulate_masked(ref, ora, 24)
        S.assert_same_state(a, b, "field %d (format %d, aberration %d) demodulate" % (it, fmt, aberr))
