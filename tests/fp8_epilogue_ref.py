"""numpy float32 restatement of the fp8 epilogue (gemm.cuh fp8_epilogue, spx_implicit_gemm_fwd_fp8), one
rounding per step, and three plausible wrong versions of it that give the same bits whenever every scale is a
power of two:

    "fma"    fmaf(acc, s, bias) instead of two rounded steps
    "assoc"  (acc * in_scale) * w_scale[k] instead of acc * (in_scale * w_scale[k])
    "recip"  y * (1 / out_scale) instead of y / out_scale (e4m3 output)

A test of the kernel against `epilogue` can only tell it from a wrong version if some output element differs
between the two; `discriminating_bias` finds, for one output channel, a bias that puts some rows of that channel
on an output rounding boundary where the wrong version lands on the other side.
"""
import numpy as np
import torch

from tests.test_fp8_cpu import e4m3_rne

F32 = np.float32
MUTATIONS = ("fma", "assoc", "recip")
# (significant bits, smallest normal exponent) of each output type
_GRID = {"f16": (11, -14), "bf16": (8, -126), "e4m3": (4, -6)}


def _fma32(a, b, c):
    """float32 fmaf(a, b, c) on float32 arrays: a * b is exact in float64 (48 bits); the sum is taken exactly as
    hi + lo (TwoSum) and rounded once to float32, with the float64 rounding of hi undone where it sits on a
    float32 tie"""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    hi = p + c64
    bb = hi - p
    lo = (p - (hi - bb)) + (c64 - bb)
    r = hi.astype(F32)
    # hi exactly halfway between two float32 values and lo != 0: the exact sum lies on lo's side of the tie
    up = np.nextafter(r, F32(np.inf)).astype(np.float64)
    dn = np.nextafter(r, F32(-np.inf)).astype(np.float64)
    r64 = r.astype(np.float64)
    tie_lo = (hi == (r64 + dn) / 2)          # r rounded up from a tie with dn
    tie_hi = (hi == (r64 + up) / 2)          # r rounded down from a tie with up
    r = np.where(tie_lo & (lo < 0), np.nextafter(r, F32(-np.inf)), r)
    r = np.where(tie_hi & (lo > 0), np.nextafter(r, F32(np.inf)), r)
    return r.astype(F32)


def round_out(y, out):
    """float32 epilogue value -> the output type, as float64 (fp16 / bf16 / e4m3 values already divided)"""
    if out == "f32":
        return y.astype(np.float64)
    if out == "f16":
        return y.astype(np.float16).astype(np.float64)
    if out == "bf16":
        return torch.from_numpy(np.ascontiguousarray(y)).to(torch.bfloat16).double().numpy()
    return e4m3_rne(y.astype(np.float64))


def epilogue(acc, in_scale, w_scale, bias, add, add_scale, act, alpha, out, out_scale, variant=None):
    """acc [rows, K] exact integers (float64) -> the output as float64; `variant` one of MUTATIONS or None.
    in_scale / add_scale / out_scale scalars, w_scale and bias [K], add [rows, K] (values of the output type)."""
    a = np.asarray(acc).astype(F32)
    assert np.array_equal(a.astype(np.float64), acc), "acc must be exact in fp32"
    i_s, w_s = F32(in_scale), np.asarray(w_scale, dtype=F32)
    s = i_s * w_s                                                    # s_k, one rounding
    if variant == "assoc":
        y = (a * i_s) * w_s
    else:
        y = a * s
    if bias is not None:
        b = np.broadcast_to(np.asarray(bias, dtype=F32), y.shape)
        y = _fma32(a, np.broadcast_to(s, y.shape), b) if variant == "fma" else y + b
    if add is not None:
        y = y + np.asarray(add, dtype=F32) * F32(1.0 if add_scale is None else add_scale)
    if act == "relu":
        y = np.where(y > 0, y, F32(0))
    elif act == "leaky_relu":
        y = np.where(y >= 0, y, y * F32(alpha))
    else:
        assert act == "none", act
    y = y.astype(F32)
    if out == "e4m3":
        o = F32(out_scale)
        y = y * (F32(1) / o) if variant == "recip" else y / o
    return round_out(y.astype(F32), out)


def differ(a, b):
    """bool mask: a and b (float64) differ in value, sign of zero or NaN-ness"""
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    return (nan_a != nan_b) | (~nan_a & ~nan_b & ((a != b) | (np.signbit(a) != np.signbit(b))))


def _midpoint(v, out):
    """the output-grid rounding boundary nearest above |v| (in y / out_scale space), with v's sign"""
    p, emin = _GRID[out]
    av = np.abs(v)
    e = np.maximum(np.floor(np.log2(np.where(av > 0, av, 1.0))), emin)
    ulp = np.ldexp(1.0, (e - (p - 1)).astype(int))
    return np.copysign((np.floor(av / ulp) + 0.5) * ulp, v)


def discriminating_bias(acc_col, in_scale, w_k, b0, add_col, add_scale, act, alpha, out, out_scale, variant,
                        rows=64):
    """A float32 bias for one output channel (acc_col [rows]) near which `variant` changes some output element
    from what `epilogue` gives; (bias, number of such elements), (b0, 0) when none is found.  Candidates put the
    exact epilogue value of sampled rows on a rounding boundary of the output type (for e4m3 the boundary times
    out_scale), and up to 8 float32 steps either side of it."""
    if out == "f32":
        return F32(b0), 0
    acc_col = np.asarray(acc_col, dtype=np.float64)
    s = F32(in_scale) * F32(w_k)
    add_term = (np.zeros(len(acc_col), F32) if add_col is None else
                np.asarray(add_col, dtype=F32) * F32(1.0 if add_scale is None else add_scale))
    pick = np.linspace(0, len(acc_col) - 1, min(rows, len(acc_col))).astype(int)
    p = acc_col[pick].astype(F32) * s
    base = p.astype(np.float64) + add_term[pick].astype(np.float64) + float(b0)
    if act == "relu":
        base = np.abs(base)
    o = 1.0 if out != "e4m3" else float(F32(out_scale))
    target = _midpoint(base / o, out) * o
    b = (target - p.astype(np.float64) - add_term[pick].astype(np.float64)).astype(F32)
    cands = [b]
    for _ in range(8):
        cands.append(np.nextafter(cands[-1], F32(np.inf)))
    down = [b]
    for _ in range(8):
        down.append(np.nextafter(down[-1], F32(-np.inf)))
    cands = np.unique(np.concatenate(cands + down[1:]))
    cands = cands[np.isfinite(cands)]
    best, hits = F32(b0), 0
    col = acc_col[:, None]
    for chunk in np.array_split(cands, max(1, len(cands) // 64)):
        kw = dict(in_scale=in_scale, w_scale=np.full(len(chunk), w_k, F32), bias=chunk,
                  add=None if add_col is None else np.repeat(np.asarray(add_col)[:, None], len(chunk), 1),
                  add_scale=add_scale, act=act, alpha=alpha, out=out, out_scale=out_scale)
        accs = np.repeat(col, len(chunk), 1)
        n = differ(epilogue(accs, **kw), epilogue(accs, variant=variant, **kw)).sum(0)
        j = int(n.argmax())
        if n[j] > hits:
            best, hits = F32(chunk[j]), int(n[j])
    return best, hits


def reciprocal_trap_scale(scale, steps=64):
    """the float32 value within `steps` float32 steps of `scale` whose float32 reciprocal is furthest (relative)
    from the exact one: an output scale where y * (1 / out_scale) most often lands on the other side of a rounding
    boundary than y / out_scale"""
    c = [F32(scale)]
    for _ in range(steps):
        c.append(np.nextafter(c[-1], F32(np.inf)))
    c = np.array(c, dtype=F32)
    err = np.abs((F32(1) / c).astype(np.float64) * c.astype(np.float64) - 1.0)
    return F32(c[int(err.argmax())])
