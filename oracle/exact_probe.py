"""Exact-arithmetic probes for the W4A16 linear kernels.  TEST INFRASTRUCTURE ONLY (numpy, no torch, no GPU).

A probe is a quantised linear and a batch of activations chosen so that the true product is exactly representable
and every partial sum a kernel can form, in any order, is exact in fp32.  Every summation order then gives the same
bits, a test can demand equality on every output element, and one dropped, duplicated or misplaced product moves an
output by at least one unit - which a rounding tolerance that grows with K cannot see (DESIGN.md section 4).

Construction (all integers; `unit` is the smallest scale, a power of two):
  * weights q in 0..15, zero points z in 0..15, scales in unit * {1, 2, 4} (optionally 0 on whole columns);
    w[k, n] = (q - z) * s is an integer of magnitude <= 60 in units;
  * activations are small integers, mostly 0, else -2, -1, 1 or 2.  The supports of consecutive token rows are
    consecutive chunks of a random permutation of 0..K-1, so rows differ and the first `cover_rows` rows touch
    every k exactly once;
  * the number of non-zeros per row follows from K-independent arithmetic: the output is a random walk of `nnz`
    steps, and `nnz` is chosen so that 8 standard deviations stay inside the 2048 units an fp16 holds exactly.

What `make_exact_case` asserts before it returns, so that no case is exact by luck:
  * |y_exact| (+ bias) <= 2048 units everywhere: every output is an fp16 value;
  * sum_k |x| * 1264 < 2^20 per token row: the GEMV and stream kernels accumulate the raw codes, S = sum x *
    (1024 + c q) with c in {1, 16}, and fold (1024 + c z) * sum x per group; 1024 + 16 * 15 = 1264 bounds both, and
    the bound on the whole row covers any group, tile or K-split of it;
  * max_row(sum_k |x|) * max|w| < 2^20 units: every prefix of sum x w in any order is an exact fp32 integer, with
    room for the alignment of addends inside a tensor-core instruction (hence 2^20, not 2^24);
  * -(z * s) is an fp16 value (the GEMVFast layout stores it rounded);
  * token rows are pairwise different, neighbouring output columns differ, every k is covered by the first
    `cover_rows` rows, and every k-row has a non-zero (q - z) * s in most live columns.
"""
from __future__ import annotations

import numpy as np

from . import awq_oracle as O

FP16_EXACT_INT = 2048          # |integers| up to here are fp16 values
PARTIAL_LIMIT = 1 << 20        # bound on any partial sum, in units
RAW_CODE = 1264                # 1024 + 16 * 15: the largest raw code 1024 + c q (and 1024 + c z), c in {1, 16}
X_VALUES = np.array([-2, -1, 1, 2], dtype=np.int8)
X_PROBS = np.array([0.1, 0.4, 0.4, 0.1])
SCALE_STEPS = np.array([1, 2, 4], dtype=np.int8)
SCALE_PROBS = np.array([0.6, 0.3, 0.1])
BIAS_MAX = 64                  # |bias| in units


def weight_units(intweight, zeros, scale_steps, group_size: int) -> np.ndarray:
    """(q - z) * (s / unit) as int8 [K, N]."""
    rep = lambda a: np.repeat(a, group_size, axis=0)  # noqa: E731
    return ((intweight.astype(np.int8) - rep(zeros.astype(np.int8))) * rep(scale_steps.astype(np.int8))).astype(np.int8)


def pick_nnz(K: int, w_units: np.ndarray, limit: int) -> int:
    """Non-zeros per activation row, at most K / 4: the output random walk keeps 8 sigma inside `limit` units at the
    mean step variance over the matrix, and 5.5 sigma in the column with the largest weights (with one group per
    column a column of scale 4 walks four times as far as one of scale 1).  A choice, not a proof: make_exact_case
    asserts the outcome."""
    x_var = float((X_PROBS * X_VALUES.astype(np.float64) ** 2).sum())
    col_var = np.square(w_units.astype(np.int16)).mean(axis=0, dtype=np.float64)
    n = min((limit / 8.0) ** 2 / (x_var * max(col_var.mean(), 1e-9)), (limit / 5.5) ** 2 / (x_var * max(col_var.max(), 1e-9)))
    return int(max(4, min(K // 4, n)))


def activation_rows(K: int, M: int, nnz: int, rng) -> np.ndarray:
    """[M, K] int8: row r is non-zero on the r-th chunk of `nnz` entries of a random permutation of 0..K-1 (a new
    permutation once one is used up; a chunk never straddles two permutations, so supports within a cover are
    disjoint)."""
    x = np.zeros((M, K), dtype=np.int8)
    per = K // nnz + (K % nnz != 0)
    for r0 in range(0, M, per):
        perm = rng.permutation(K)
        for r in range(r0, min(M, r0 + per)):
            idx = perm[(r - r0) * nnz:(r - r0 + 1) * nnz]
            x[r, idx] = rng.choice(X_VALUES, size=idx.size, p=X_PROBS)
    return x


def contract_units(x_units: np.ndarray, w_units: np.ndarray) -> np.ndarray:
    """X . W for integer operands, as float64.  The products run through BLAS in fp32 over column blocks: with every
    |partial sum| < 2^20 (which the caller asserts) each fp32 operation is exact, so the result is the integer
    contraction; tests/test_exact_probe_cpu.py checks it against int64 arithmetic."""
    xf = x_units.astype(np.float32)
    out = np.empty((x_units.shape[0], w_units.shape[1]), dtype=np.float64)
    for n0 in range(0, w_units.shape[1], 4096):
        out[:, n0:n0 + 4096] = xf @ w_units[:, n0:n0 + 4096].astype(np.float32)
    return out


def make_exact_case(K: int, N: int, G: int, M: int, seed: int, bias: bool = False, zero_col_frac: float = 0.0,
                    unit: float = 2.0**-6, nnz: int | None = None, layouts=("gemm", "gemv", "fast"),
                    reference: bool = True) -> dict:
    """One exact probe (see the module docstring).  G = -1 means one group per column (G = K).

    Returns intweight / zeros / scales (canonical), group_size, the requested packings (`qweight`, `qzeros` for
    "gemm"; `gemv` = (qweight, qzeros, scales); `fast` = (qweight, scales, scaled_zeros)), x [M, K] fp16, bias [N]
    fp16 or None, y_exact [M, N] float64 (bias included; None when reference=False), unit, nnz, cover_rows (the
    first that many rows touch every k exactly once) and w_units.  `nnz` overrides the density chosen from the
    weights (chains of linears pass a small one)."""
    rng = np.random.default_rng(seed)
    Gs = K if G == -1 else G
    assert K % Gs == 0 and N % 8 == 0
    iw = rng.integers(0, 16, size=(K, N), dtype=np.uint8)
    iz = rng.integers(0, 16, size=(K // Gs, N), dtype=np.uint8)
    steps = rng.choice(SCALE_STEPS, size=(K // Gs, N), p=SCALE_PROBS)
    if zero_col_frac > 0:
        steps[:, rng.random(N) < zero_col_frac] = 0
    scales = (steps.astype(np.float32) * np.float32(unit)).astype(np.float16)
    w_units = weight_units(iw, iz, steps, Gs)
    b_units = rng.integers(-BIAS_MAX, BIAS_MAX + 1, size=N).astype(np.int64) if bias else None
    limit = FP16_EXACT_INT - (BIAS_MAX if bias else 0)
    if nnz is None:
        nnz = pick_nnz(K, w_units, limit)
    assert 1 <= nnz <= K
    x_units = activation_rows(K, M, nnz, rng)
    cover_rows = K // nnz + (K % nnz != 0)

    # ---- the guarantees ---------------------------------------------------------------------------------
    row_abs = np.abs(x_units).astype(np.int64).sum(axis=1)
    assert int(row_abs.max()) * RAW_CODE < PARTIAL_LIMIT, "raw-code partial sums may leave the exact fp32 range"
    assert int(row_abs.max()) * int(np.abs(w_units).max()) < PARTIAL_LIMIT, "partial sums may leave the exact range"
    sz = -(scales.astype(np.float32) * iz.astype(np.float32))
    assert np.array_equal(sz.astype(np.float16).astype(np.float32), sz), "-(z * s) is not an fp16 value"
    if M > 1:
        assert np.unique(x_units, axis=0).shape[0] == M, "two token rows are equal"
    if M >= cover_rows:
        assert ((x_units[:cover_rows] != 0).sum(axis=0) == 1).all(), "a k-row is not covered exactly once"
    live = steps.any(axis=0)
    if zero_col_frac < 0.5:
        assert ((w_units[:, live] != 0).mean(axis=1) > 0.75).all(), "a k-row is zero in too many columns"

    y_exact = None
    if reference:
        y_units = contract_units(x_units, w_units)
        if bias:
            y_units += b_units
        assert np.abs(y_units).max() <= FP16_EXACT_INT, "an output is not an fp16 value: lower nnz"
        if N > 1 and M >= 4 and live.all():
            assert (y_units[:, 1:] != y_units[:, :-1]).any(axis=0).all(), "two neighbouring columns are equal"
        y_exact = y_units * float(unit)
        assert np.array_equal(y_exact.astype(np.float16).astype(np.float64), y_exact)

    c = dict(intweight=iw, zeros=iz, scales=scales, scale_steps=steps, group_size=Gs, w_units=w_units,
             x=x_units.astype(np.float16), x_units=x_units, unit=float(unit), nnz=nnz, cover_rows=cover_rows,
             bias=(b_units * float(unit)).astype(np.float16) if bias else None, y_exact=y_exact)
    if "gemm" in layouts:
        c["qweight"], c["qzeros"] = O.pack_gemm(iw, iz)
    if "gemv" in layouts:
        c["gemv"] = O.pack_gemv(iw, iz, scales, Gs)
    if "fast" in layouts:
        c["fast"] = O.pack_gemv_fast(iw, iz, scales, Gs)
    return c


def mismatch_report(got, want, unit: float, limit: int = 8) -> str:
    """First few wrong (row, column) pairs and their difference in units: the position locates the faulty boundary."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    bad = np.argwhere(got != want)
    head = ", ".join(f"({r}, {c}): {(got[r, c] - want[r, c]) / unit:+g}" for r, c in bad[:limit])
    cols = np.unique(bad[:, 1])
    return (f"{len(bad)} / {got.size} elements differ in {np.unique(bad[:, 0]).size} rows and {cols.size} columns "
            f"(columns {cols.min()}..{cols.max()}); first (row, col): units = {head}")
