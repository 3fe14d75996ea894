"""Self-checks of the numpy fp8 epilogue restatement (tests/fp8_epilogue_ref.py) that the GPU accuracy tests
compare the kernels with: its emulated fmaf rounds once, it agrees with float64 where every step is exact, and the
bias search finds elements that tell each wrong epilogue from the documented one."""
from fractions import Fraction

import numpy as np
import pytest

from tests.fp8_epilogue_ref import (F32, MUTATIONS, _fma32, differ, discriminating_bias, epilogue,
                                   reciprocal_trap_scale)


def _round_f32(q):
    """Fraction -> nearest float32, ties to even"""
    r = np.float32(float(q))
    best = None
    for c in (np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))):
        d = abs(Fraction(float(c)) - q)
        if best is None or d < best[0] or (d == best[0] and int(np.array(c).view(np.int32)) % 2 == 0):
            best = (d, c)
    return best[1]


def test_emulated_fmaf_rounds_once():
    rng = np.random.default_rng(0)
    a = rng.integers(-3000, 3000, size=3000).astype(F32)
    b = (rng.standard_normal(3000) * 1e-4).astype(F32)
    c = (rng.standard_normal(3000) * np.exp2(rng.integers(-30, 5, size=3000))).astype(F32)
    # exact ties of the float64 sum: c chosen so that a * b + c sits a quarter float32 ulp off a tie
    got = _fma32(a, b, c)
    for i in range(len(a)):
        want = _round_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
        assert got[i] == want, (a[i], b[i], c[i], got[i], want)
    two_step = (a * b) + c
    assert (got != two_step).any(), "no element where fused and two-step rounding differ"


@pytest.mark.parametrize("out", ["f32", "f16", "bf16", "e4m3"])
def test_exact_grid_cannot_tell_the_variants_apart(out):
    """integer acc, power-of-two scales, biases on a 1/8 grid: every variant equals float64 rounded once, which is
    why the exact-grid tests cannot catch them"""
    rng = np.random.default_rng(1)
    acc = rng.integers(-200, 200, size=(500, 8)).astype(np.float64)
    w = (2.0 ** rng.integers(-2, 2, size=8)).astype(F32)
    bias = (rng.integers(-16, 17, size=8) / 8).astype(F32)
    add = rng.integers(-3, 4, size=(500, 8)).astype(np.float64)
    kw = dict(in_scale=0.125, w_scale=w, bias=bias, add=add, add_scale=0.5, act="leaky_relu", alpha=0.25, out=out,
              out_scale=0.25)
    ref = epilogue(acc, **kw)
    y = acc * (0.125 * w.astype(np.float64)) + bias + add * 0.5
    y = np.where(y >= 0, y, y * 0.25)
    if out == "e4m3":
        y = y / 0.25
    from tests.fp8_epilogue_ref import round_out
    assert not differ(ref, round_out(y.astype(F32), out)).any()
    for v in MUTATIONS:
        assert not differ(ref, epilogue(acc, variant=v, **kw)).any(), v


@pytest.mark.parametrize("out", ["f16", "bf16", "e4m3"])
@pytest.mark.parametrize("act", ["none", "relu", "leaky_relu"])
def test_bias_search_finds_discriminating_elements(out, act):
    rng = np.random.default_rng(2)
    acc = rng.integers(-60, 60, size=2000).astype(np.float64)
    in_scale, w_k = F32(3.1 / 448), F32(0.77 / 448)
    add = rng.standard_normal(2000).astype(F32) * 1e-3
    o = reciprocal_trap_scale(7e-6)
    assert abs(float(o) / 7e-6 - 1) < 1e-4
    for v in MUTATIONS if out == "e4m3" else ("fma", "assoc"):
        b, hits = discriminating_bias(acc, in_scale, w_k, F32(1e-3), add, F32(0.37), act, 0.1, out, o, v)
        assert hits > 0, v
        kw = dict(in_scale=in_scale, w_scale=np.array([w_k]), bias=np.array([b]), add=add[:, None], add_scale=0.37,
                  act=act, alpha=0.1, out=out, out_scale=o)
        assert differ(epilogue(acc[:, None], **kw), epilogue(acc[:, None], variant=v, **kw)).sum() == hits
