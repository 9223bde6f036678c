"""The error model of the W4A16 linear kernels, and LLM-shaped test data.  TEST INFRASTRUCTURE ONLY.

Error model
-----------
Every forward output y of a linear kernel is held to its fp64 value y64 = X . W (+ bias), where W is the weight the
stored tensors encode (the bit-exact fp16 dequantisation for the GEMM and GEMV layouts, q*s + sz in fp64 for the
GEMVFast layout):

    |y - y64| <= 2^-10 |y64|  +  wr (|X| . |W|)  +  2^-24 r Omega sum_g s_g sum_{k in g} |x_k|  +  1e-6

  * 2^-10 |y64|: the final rounding to fp16 (2^-11) with a factor 2 of slack;
  * wr (|X| . |W|): the weights and the fp32 sums of the products;
  * the fold term: kernels that apply zero point and scale once per (group, column) round sums whose magnitude is
    Omega sum |x|, not |q - z| |x|; their error does not shrink with the weights, and on a column whose every q equals
    its group's z (exact output 0) it is the whole error;
  * 1e-6: absolute floor (fp16 subnormal steps, fixed-point split-K partials).

Families (the route-to-family map of the C ABI is in tests/test_gpu_llm_data.py):

  exact-dequant  dequant.cu; the wgmma GEMM and the small-M kernel (gemm_tc.cu) with the GEMM- and GEMV-layout
                 loaders; moe_tc_kernel.  The tensor-core A operand is W16 itself, bit-exact: wr = 2^-16, no fold term.
  fast-dequant   the wgmma kernels with the GEMVFast-layout loader: fp16(q*s + sz) per weight (gemm_tc.cu
                 FastLayoutLoader), one fp16 rounding per weight away from the fp64 truth: wr = 2^-11, no fold term.
  offset-fold    the persistent GEMV gemv_v3 and gemv_v3_moe, the register-staged GEMV, moe_grouped_kernel, and the
                 stream / batched decode programs: the tensor core accumulates S = sum x (1024 + c q) and
                 X = sum x in fp32 and the fold is s (S - (1024 + c z) X) / c.  wr = 2^-11, Omega = 1039 (kind A,
                 c = 1: 1024 + 15; kind B, c = 16: (1024 + 16 q) / 16 <= 79 is covered).
  code-fold      the warp-per-row fp32-FMA kernels of the GEMV and GEMVFast layouts (gemv.cu): S = sum x q,
                 X = sum x, fold s (S - z X) (GEMV) or s S + sz X (GEMVFast).  wr = 2^-11, Omega = 15 (|z|, and
                 |sz| / s).

Counting r, the fp32 roundings on the fold path, each of magnitude at most Omega sum_{k in g} |x_k| (u = 2^-24 each):
2 per mma.sync accumulation (the tensor core aligns the addends and truncates; it does not round each add the IEEE
way), 1 per fp32 add of warp or unit partials inside a group, 1 per fp32 FMA / add of a sequential sum, and 2 for the
fold itself (the product (1024 + c z) X and the subtraction).  Per kernel, at group size G:

  offset-fold
    gemv_v3 / gemv_v3_moe (gemv.cu:561-567, gemv_tile.cuh:v3_tile_mma, v3_fold_reg): one warp accumulates the S and X
        chains over the 64-row tiles of its run until the group (or the run) ends, at most G / 16 mma each:
        r = 2 G/16 + 2 G/16 + 2 = G/4 + 2                                                    (34 at G = 128)
    register-staged GEMV (gemv.cu:119-144, 174-197) and moe_grouped_kernel (moe.cu:207-266): RW / 16 mma per warp
        chain, then the raw sums of the warps sharing a group added in fp32; an add replaces two or more mma
        roundings, so r <= G/4 + 2 as above (RW = G: 2 G/16 per chain, no adds).
    stream / batched decode programs (program_stream.cuh:455-474, program_batch.cuh:74-98, X from
        program_stream_body.inc:458-469): F = min(G, 128) / 16 k16 blocks in two chains of F / 2 mma, added once:
        S: F + 1; X: 8 fp16 values per lane summed in pairs and sequentially (depth 4), then log2(UK / 8) shuffle
        adds: 4 + log2(UK / 8); fold 2.                                                        (19 at G = 128)
    r = max of the two expressions above.
  code-fold
    GEMV layout (gemv.cu:857-890): per 32-k chunk, S of each nibble class is 16 sequential FMAs (15 roundings), X is 16
        pair adds plus 16 sequential adds (depth 16), the fold adds the classes, multiplies z X and subtracts (3):
        r = 15 + 16 + 3 = 34.
    GEMVFast layout (gemv.cu:1034-1055): S and X as above, the fold adds the classes, multiplies by s, multiplies sz X
        and adds (4): r = 35.
    r = 35.

r comes from the order of the arithmetic, not from any measurement: if a kernel exceeds its bound, the order above
misses a rounding of that kernel.
"""
from __future__ import annotations

import numpy as np

from oracle import awq_oracle as O

RTOL = 2.0**-10
WR_EXACT = 2.0**-16
WR_FOLD = 2.0**-11
ATOL = 1e-6
U32 = 2.0**-24
FP16_MAX = 65504.0
# the band of exact values that a correct kernel may round either way: below it fp16 is finite, above it inf
BAND_LO, BAND_HI = 65504.0, 65520.0
OVF_LOW = FP16_MAX * (1 - 2.0**-9)
OVF_HIGH = 65520.0 * (1 + 2.0**-8)
CANCEL_HALF = 2.0**17

FAMILIES = ("exact-dequant", "fast-dequant", "offset-fold", "code-fold")
_WR = {"exact-dequant": WR_EXACT, "fast-dequant": WR_FOLD, "offset-fold": WR_FOLD, "code-fold": WR_FOLD}
_OMEGA = {"offset-fold": 1039.0, "code-fold": 15.0}


def fold_r(family: str, G: int) -> int:
    """r of the family at group size G (see the module docstring); 0 for the families without a fold."""
    if family == "offset-fold":
        uk = min(G, 128)
        program = (uk // 16 + 1) + (4 + int(np.log2(uk // 8))) + 2
        return max(G // 4 + 2, program)
    if family == "code-fold":
        return 35
    if family in ("exact-dequant", "fast-dequant"):
        return 0
    raise ValueError(family)


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def forward_tolerance(x, case, family: str, cols=None, y64=None):
    """Per-element bound on |y - y64| for the rows `x` [M, K] and the columns `cols` (all when None) of `case`:
    a dict with "w" [K, N] (the weight the stored tensors encode), "scales" [K/G (or more rows), N] and
    "group_size".  `y64` (the fp64 result of those columns, bias included) is computed when not given."""
    if family not in _WR:
        raise ValueError(family)
    w = case["w"] if cols is None else case["w"][:, cols]
    xa = np.abs(_f64(x))
    if y64 is None:
        y64 = _f64(x) @ _f64(w)
        if case.get("bias") is not None:
            y64 = y64 + _f64(case["bias"] if cols is None else case["bias"][cols])
    tol = RTOL * np.abs(y64) + _WR[family] * (xa @ np.abs(_f64(w))) + ATOL
    r = fold_r(family, case["group_size"])
    if r:
        K = xa.shape[-1]
        G = case["group_size"]
        ng = K // G
        s = _f64(case["scales"])[:ng]
        s = s if cols is None else s[:, cols]
        xg = xa.reshape(xa.shape[0], ng, G).sum(axis=2)         # sum_{k in g} |x_k|, per row and group
        tol = tol + U32 * r * _OMEGA[family] * (xg @ np.abs(s))
    return tol


def check_forward(y, x, case, family: str, what: str, cols=None, y64=None):
    """Assert |y - y64| <= forward_tolerance on the columns `cols` of y ([M, N] or already [M, len(cols)]);
    returns the largest error / bound ratio.  y64 (bias included) is computed when not given."""
    w = case["w"] if cols is None else case["w"][:, cols]
    if y64 is None:
        y64 = _f64(x) @ _f64(w)
        if case.get("bias") is not None:
            y64 = y64 + _f64(case["bias"] if cols is None else case["bias"][cols])
    got = _f64(y)
    if cols is not None and got.shape[-1] != len(cols):
        got = got[..., cols]
    tol = forward_tolerance(x, case, family, cols=cols, y64=y64)
    err = np.abs(got - y64)
    bad = ~(err <= tol)                                          # NaN counts as outside
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError(f"{what} [{family}]: {int(bad.sum())} / {bad.size} outside tolerance, first at "
                             f"{tuple(int(v) for v in i)}: got {got[tuple(i)]!r} want {y64[tuple(i)]!r} "
                             f"bound {tol[tuple(i)]:.3e}; max err / bound {np.nanmax(err / tol):.3e}")
    return float((err / tol).max()) if err.size else 0.0


# ------------------------------------------------------------------------------------------ which family runs where
# The route each C-ABI entry point takes (cabi.cu:127-190), restated so that every check names the family of the
# kernel that ran.  `knobs` holds the non-default knob values of the call.
def gemm_route_family(M: int, K: int, N: int, G: int, knobs=None) -> str:
    """b200awq_gemm_forward: M <= knob 2 (default 8, lowered to 4 where the small-M wgmma kernel applies) on shapes the
    tensor-pipe GEMV takes -> gemv_v3 (knob 5 = 0) or the register-staged GEMV: offset-fold; else gemm_tc."""
    knobs = knobs or {}
    G = K if G in (-1, 0) else G
    gemv_max = knobs.get(2, 8)
    tcq = knobs.get(19, 0) != 1 and G >= 64 and K % 128 == 0 and N % 128 == 0 and M <= 128
    if gemv_max == 8 and M > 4 and tcq:
        gemv_max = 4
    if M <= gemv_max and M <= 8 and N % 32 == 0 and G % 32 == 0:
        return "offset-fold"
    return "exact-dequant"


def gemv_route_family(M: int, K: int, knobs=None) -> str:
    """b200awq_gemv_forward: M <= knob 2 and (M <= 2 or K % 64 != 0) -> the warp-per-row kernel; else gemm_tc."""
    knobs = knobs or {}
    return "code-fold" if M <= knobs.get(2, 8) and (M <= 2 or K % 64 != 0) else "exact-dequant"


def fast_route_family(M: int, knobs=None) -> str:
    """b200awq_fast_forward: M <= min(knob 2, 2) -> the warp-per-row kernel; else gemm_tc with the GEMVFast loader."""
    knobs = knobs or {}
    return "code-fold" if M <= min(knobs.get(2, 8), 2) else "fast-dequant"


# ------------------------------------------------------------------------------------------------- LLM-shaped data
ZERO_COLS = (0, 7, 8, 255, 256)          # and N - 1: the 8-column word, 16-column set and 256-column tile edges


def _massive_channels(K, G, avoid_groups, rng, n=6):
    ok = np.ones(K, dtype=bool)
    for g in avoid_groups:
        ok[g * G:(g + 1) * G] = False
    ch = np.sort(rng.choice(np.nonzero(ok)[0], size=n, replace=False))
    mag = 2.0 ** rng.uniform(8, 12, size=n)
    sign = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    rng.shuffle(sign)
    return ch, sign * mag


def _pin_column(scales, col, d, xsum_g, target, groups):
    """Scales of `col` over `groups` such that sum_g s_g d X_g ~= target: a common fp16 scale slightly short of the
    target, the last group's scale filling in the rest (fp16 rounding of one group's share remains)."""
    groups = list(groups)
    tot = float(xsum_g[groups].sum())
    s0 = np.float16(target / (d * tot) * (1 - 2.0**-6))
    scales[groups[:-1], col] = s0
    part = float(s0) * d * float(xsum_g[groups[:-1]].sum())
    scales[groups[-1], col] = np.float16((target - part) / (d * float(xsum_g[groups[-1]])))


def make_llm_case(K: int, N: int, G: int, M: int, seed: int, kind: str = "llm"):
    """Deterministic LLM-shaped linear: returns a dict with x [M, K] fp16, the canonical integers (intweight [K, N],
    zeros [K/G, N], scales [K/G, N] fp16), the GEMM-layout words (qweight, qzeros), w = the bit-exact fp16
    dequantisation, bias (kind "llm") and the designated columns / groups.

    kind "llm": N(0,1) activations with six massive channels (2^8..2^12, mixed signs, the same channels in every row),
      row 1 all small (~2^-10), row 2 with fp16-subnormal entries; AWQ-like codes q = clip(z + round(N(0, sigma)),
      0, 15), sigma 0.7 / 2.5 alternating per 8 columns, zeros over 0..15 with both ends; log-uniform scales in
      [2^-12, 2^-4], one group with fp16-subnormal scales and one with scale 1; all-zero columns (every q equals its
      group's z) at ZERO_COLS and N - 1, and one whole group with q == z in every column.
    kind "overflow": positive activations (rows alternate in sign); columns whose exact output is +-OVF_LOW
      ("ovf_low") and +-OVF_HIGH ("ovf_high"), each built from same-sign contributions.
    kind "cancel": positive activations (rows alternate in sign); columns ("cancel") whose first- and second-half-of-K
      partial sums are about +-2^17 while the total is O(1).
    The generator asserts its own claims (finite fp16 inputs, where the zero columns / groups are, the fp16 range of
    every exact output, and that every overflow column's bound stays inside its side of the fp16 overflow band)."""
    assert K % G == 0 and N % 8 == 0 and N > 256 and K // G >= 4
    rng = np.random.default_rng(seed)
    ng = K // G
    z = rng.integers(0, 16, size=(ng, N)).astype(np.uint8)
    z[0, :N // 2], z[0, N // 2:] = 0, 15                         # both ends of the zero-point range
    sigma = np.where((np.arange(N) // 8) % 2 == 0, 0.7, 2.5)
    zk = np.repeat(z, G, axis=0).astype(np.int64)
    q = np.clip(zk + np.rint(rng.standard_normal((K, N)) * sigma[None, :]), 0, 15).astype(np.int64)
    scales = (2.0 ** rng.uniform(-12, -4, size=(ng, N))).astype(np.float16)
    out = dict(group_size=G, kind=kind, zero_cols=np.array([], dtype=np.int64), zero_groups=np.array([], dtype=np.int64),
               ovf_low=np.array([], dtype=np.int64), ovf_high=np.array([], dtype=np.int64),
               cancel=np.array([], dtype=np.int64), bias=None)
    if kind == "llm":
        g_sub, g_one, g_zero = 1, 2, 3
        scales[g_sub] = (rng.integers(1, 1024, size=N) * 2.0**-24).astype(np.float16)   # fp16 subnormals
        scales[g_one] = 1.0
        zero_cols = np.unique([c for c in ZERO_COLS if c < N] + [N - 1])
        q[:, zero_cols] = zk[:, zero_cols]
        q[g_zero * G:(g_zero + 1) * G] = zk[g_zero * G:(g_zero + 1) * G]
        ch, val = _massive_channels(K, G, (g_one,), rng)
        x = rng.standard_normal((M, K))
        x[:, ch] = val[None, :] * (1 + 0.01 * rng.standard_normal((M, len(ch))))
        if M > 1:
            x[1] = rng.standard_normal(K) * 2.0**-10
        if M > 2:
            sub = np.arange(0, K, 3)
            x[2, sub] = rng.integers(1, 1024, size=sub.size) * 2.0**-24 * np.where(rng.random(sub.size) < 0.5, -1, 1)
        x = x.astype(np.float16)
        if M > 2:
            sub_x = x[2, np.arange(0, K, 3)]
            assert ((sub_x != 0) & (np.abs(sub_x) < 2.0**-14)).all(), "row 2 lost its fp16 subnormals"
        out.update(zero_cols=zero_cols, zero_groups=np.array([g_zero]), massive=ch,
                   bias=(rng.standard_normal(N) * 0.5).astype(np.float16))
    else:
        x0 = (0.5 + np.abs(rng.standard_normal(K)) * 0.5).astype(np.float16).astype(np.float64)
        x = (x0[None, :] * np.where(np.arange(M) % 2 == 0, 1.0, -1.0)[:, None]).astype(np.float16)
        xsum_g = x0.reshape(ng, G).sum(axis=1)
        d = 8
        picks = rng.choice(np.arange(1, N - 1), size=16, replace=False)

        def set_sign(col, sign, groups):
            rows = np.concatenate([np.arange(g * G, (g + 1) * G) for g in groups])
            gz = np.asarray(groups)
            z[gz, col] = rng.integers(0, 8, size=gz.size) if sign > 0 else rng.integers(8, 16, size=gz.size)
            q[rows, col] = np.repeat(z[gz, col].astype(np.int64), G) + sign * d

        if kind == "overflow":
            low, high = picks[:8], picks[8:]
            for i, c in enumerate(np.concatenate([low, high])):
                sign = 1 if i % 2 == 0 else -1
                set_sign(c, sign, range(ng))
                _pin_column(scales, c, d * sign, xsum_g, sign * (OVF_LOW if i < 8 else OVF_HIGH), range(ng))
            out.update(ovf_low=np.sort(low), ovf_high=np.sort(high))
        elif kind == "cancel":
            half = ng // 2
            for c in picks[:8]:
                set_sign(c, 1, range(half))
                set_sign(c, -1, range(half, ng))
                _pin_column(scales, c, d, xsum_g, CANCEL_HALF, range(half))
                p1 = float(_f64(scales[:half, c]) @ (d * xsum_g[:half]))
                _pin_column(scales, c, -d, xsum_g, -(p1 - 0.75), range(half, ng))
            out.update(cancel=np.sort(picks[:8]))
        else:
            raise ValueError(kind)
    iw = q.astype(np.uint8)
    qweight, qzeros = O.pack_gemm(iw, z)
    w = O.dequantize_gemm(qweight, qzeros, scales, G)
    out.update(x=x, intweight=iw, zeros=z, scales=scales, qweight=qweight, qzeros=qzeros, w=w)
    _assert_claims(out)
    return out


def _assert_claims(c):
    x, w, s, G = c["x"], c["w"], c["scales"], c["group_size"]
    for name in ("x", "scales", "bias"):
        if c.get(name) is not None:
            assert c[name].dtype == np.float16 and np.isfinite(c[name]).all(), name
    assert (c["intweight"] <= 15).all() and (c["zeros"] <= 15).all()
    for col in c["zero_cols"]:
        assert not w[:, col].any(), f"column {col} is not all zero"
    for g in c["zero_groups"]:
        assert not w[g * G:(g + 1) * G].any(), f"group {g} is not all zero"
    if c["kind"] == "llm":
        assert (c["zeros"] == 0).any() and (c["zeros"] == 15).any()
        assert ((s > 0) & (s < 2.0**-14)).any() and (s == 1).any()
    worst = {f: forward_tolerance(x, c, f) for f in ("offset-fold", "code-fold", "exact-dequant")}
    bound = np.maximum(np.maximum(worst["offset-fold"], worst["code-fold"]), worst["exact-dequant"])
    y64 = _f64(x) @ _f64(w) + (_f64(c["bias"]) if c.get("bias") is not None else 0.0)
    special = np.zeros(w.shape[1], dtype=bool)
    special[c["ovf_low"]] = special[c["ovf_high"]] = True
    a = np.abs(y64)
    assert (a[:, ~special] + bound[:, ~special] <= FP16_MAX * (1 - 2.0**-4)).all(), "an output near the fp16 limit"
    if len(c["ovf_low"]):
        lo, hi = c["ovf_low"], c["ovf_high"]
        assert (np.abs(a[:, lo] - OVF_LOW) < 2.0).all() and (np.abs(a[:, hi] - OVF_HIGH) < 2.0).all()
        assert (a[:, lo] + bound[:, lo] < BAND_LO).all(), "a low overflow column's bound reaches the band"
        assert (a[:, hi] - bound[:, hi] > BAND_HI).all(), "a high overflow column's bound reaches the band"
    K = w.shape[0]
    for col in c["cancel"]:
        p1 = _f64(x[:, :K // 2]) @ _f64(w[:K // 2, col])
        assert (np.abs(p1) > 2.0**16).all() and (np.abs(y64[:, col]) < 8).all(), f"cancel column {col}"
