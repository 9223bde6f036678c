"""Exact-arithmetic probes for the W4A16 linear kernels.  TEST INFRASTRUCTURE ONLY (numpy; the MoE probes' weights
and reference use torch on whatever device they are given).

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

`make_exact_moe_case` extends the probes to whole MoE blocks (sparse_moe, qwen3_moe, deepseek_moe): the test chooses
the routing through one-hot router rows, and the SiLU * mul of the gate|up finish becomes exact because every gate
column is 0, +32 or -64 (see its docstring).  Its expert weights are drawn with torch on the device that runs them
(`moe_weights`), and `moe_expected` is the exact reference of every buffer the block leaves behind.
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


# ------------------------------------------------------------------------------------------------------ MoE blocks
MOE_LOGIT = 32.0                 # a selected expert's router logit: Wg[e, r_e] = 32 and x[r_e] = 1
GATE_ON, GATE_OFF = 32.0, -64.0  # gate column values: silu(32) = 32 in fp32, silu(-64) * u rounds to 0 in fp16
GATE_SCALE, GATE_ZERO = 8.0, 8   # the control groups' gate scale and zero point: q = 12 gives +32, q = 0 gives -64
W_VAR = 42.5 * float((SCALE_PROBS * SCALE_STEPS.astype(np.float64) ** 2).sum())   # E[((q - z) step)^2]
W_VAR_MAX = 42.5 * 16.0                                                           # ... in a column at step 4
X_VAR = float((X_PROBS * X_VALUES.astype(np.float64) ** 2).sum())
Y_LIMIT = 1023                   # |per-slot down output| in units: one unit of y moves c = y w by more than an ulp
ROUTE_PER_GROUP = 16             # routing coordinates per quantisation group at most


def _designed_weight(op: str, k: int, renormalize: bool, scoring: str, rsf: float) -> float:
    """The routing weight every selected slot gets when k logits are 32 and the rest 0 or -32, in the kernels' fp32
    arithmetic (slot-order sums; the unselected experts' exp(-32) vanish below one fp32 ulp of k)."""
    f32 = np.float32
    if op == "deepseek" and scoring == "sigmoid":
        w = np.full(k, f32(1), dtype=f32)                   # sigmoid(32) = 1 / (1 + exp(-32)) = 1.0f
        if renormalize:
            den = f32(0)
            for v in w:
                den = f32(den + v)
            w = (w / f32(den + f32(1e-20))).astype(f32)
        return float(f32(w[0] * f32(rsf)))
    p = np.full(k, f32(1) / f32(k), dtype=f32)              # exp(0) / sum
    if op == "deepseek":
        return float(f32(p[0] * f32(rsf)))
    if renormalize:
        den = f32(0)
        for v in p:
            den = f32(den + v)
        p = (p / den).astype(f32)
    return float(np.float16(p[0])) if op == "qwen3" else float(p[0])


def _teams(rng, E: int, k: int, n_group: int, topk_group: int) -> list:
    """One round of selections: every expert in exactly one team of k (the last team is filled up with experts from
    other teams); with expert groups a team spans at most topk_group of the n_group groups, so the group rule keeps
    it."""
    gsz = E // n_group
    left = list(rng.permutation(E))
    teams = []
    while left:
        team, groups = [], set()
        for e in list(left):
            if len(team) < k and (e // gsz in groups or len(groups) < topk_group):
                team.append(e)
                groups.add(e // gsz)
                left.remove(e)
        for e in rng.permutation(E):                      # fill the last team from the groups it already spans
            if len(team) < k and e not in team and e // gsz in groups:
                team.append(int(e))
        assert len(team) == k, "cannot form a team within topk_group expert groups"
        teams.append(np.array(team, dtype=np.int64))
    return teams


def make_exact_moe_case(op: str, E: int, top_k: int, H: int, I: int, G: int, seed: int, I_s: int = 0,
                        renormalize: bool = True, scoring: str = "softmax", n_group: int = 1, topk_group: int = 1,
                        rsf: float = 1.0, order: str = "ascending", unit: float = 2.0**-6,
                        unit2: float = 2.0**-6) -> dict:
    """The run plan of an exact probe of one MoE block: op "sparse" (sparse_moe), "qwen3" (qwen3_moe) or "deepseek"
    (deepseek_moe with a shared expert of intermediate size I_s).

    Reserved coordinates of x: one routing coordinate r_e per expert (at most ROUTE_PER_GROUP per quantisation group)
    and m control coordinates (in "control groups").  The router weight is one-hot, Wg[e, r_e] = 32, so
    logit_e = 32 x[r_e]: x[r_e] = 1 selects e (logit 32), 0 or -1 does not (0 or -32).  Softmax then gives the
    selected experts exactly 1 / k, sigmoid exactly 1.0 (and 0.5 or ~0 to the rest), so every scoring rule and
    renormalisation gives a known weight (_designed_weight), and the k selected experts tie: their slots follow the
    kernels' documented tie rule, ascending id.  order="descending" (sigmoid only) sets e_score_correction_bias[e] =
    e 2^-12 instead of 0, which orders the same selection by descending id and leaves the weights (taken from s) as
    they are.
    Gate half of every w1 (the shared expert's too): zero (q = z) except on the control rows, where the control groups
    have scale 8, zero point 8 and q = 12 (g = +32) on the columns of the row's class, q = 0 (g = -64) elsewhere.
    Every routed column belongs to one of m classes, and so does every shared column.
    Up half: ordinary probe weights, except that the groups holding reserved rows have scale step 1, the control rows
    have q - z = +-1, and the routing rows q - z = +-1 on a few "routing columns" (one in each of the first classes)
    and q = z elsewhere.  w2 (and the shared down): ordinary probe weights in units of unit2.

    Two kinds of runs (one token each), each round a new random partition of the experts into teams of k:
      "up" runs cover the k-rows of gate|up: a chunk of the other coordinates (probe values), x[r_e] = 1 for the team
      and -1 for every other expert, no control row.  Every gate is 0, so act, the down outputs and out are 0.
      "down" runs cover the k-rows of down: x[r_e] = 1 for the team, one control row = 1 (class c), nothing else.
      Each up value is then the control row's +-1, or on a routing column a sum of k + 1 terms +-1 (odd for even
      k), never 0, and act = 32 u on the class-c columns, 0 elsewhere: every class-c k-row of down meets a non-zero
      activation, and |y| <= 60 sum |u| bounds every down output whatever the weights.
    The number of classes keeps that bound within Y_LIMIT units (2048 for the shared expert).  What it asserts: the
    raw-code and partial-sum limits of the module docstring for both expert ops, the fp32 routing arithmetic, that
    silu(-64) u rounds to 0, that every (expert, k-row) pair of gate|up and of down is hit by a run (and every
    (shared, k-row) pair), and the slot positions of experts 0 and E - 1.  The data-dependent limits (outputs that
    are fp16 values) are asserted by moe_expected on the generated weights.

    Returns the plan: x_units [R, H] int8, ids [R, k] (designed slot order), kind [R] (0 up, 1 down), ctl [R] (class
    or -1), route_rows [E], ctl_rows [m], classes [I] / classes_s [I_s], weight (the designed fp32 / fp16 routing
    weight), bias [E] (sigmoid), the sizes and units, and the coverage counts."""
    assert op in ("sparse", "qwen3", "deepseek") and (op == "deepseek" or I_s == 0)
    assert scoring == "softmax" or op == "deepseek"
    assert order == "ascending" or scoring == "sigmoid"
    assert n_group == 1 or scoring == "sigmoid"
    assert top_k % 2 == 0, "the down runs' up values are sums of top_k + 1 terms +-1: odd (non-zero) for even top_k"
    assert H % G == 0 and I % G == 0 and I_s % G == 0 and E % n_group == 0 and 1 <= topk_group <= n_group
    rng = np.random.default_rng(seed)
    k, k1 = top_k, top_k + 1
    ngr = H // G

    # ---- classes: in a down run an up value is the control row's +-1, or on the few "routing columns" (where the
    #      routing rows' up weights are +-1 too) a sum of k + 1 terms +-1; a class of n columns with one routing column
    #      gives |y| <= (n - 1 + k + 1) 60 units whatever the weights: within Y_LIMIT per slot, 2048 for the shared one
    n_on = Y_LIMIT // 60 - k
    n_on_s = FP16_EXACT_INT // 60 - k
    assert n_on >= 1
    m = max(-(-I // n_on), -(-I_s // n_on_s) if I_s else 1)
    classes = (rng.permutation(I) % m).astype(np.int32)
    classes_s = (rng.permutation(I_s) % m).astype(np.int32)
    # one routing column in each of the first classes (at most one per class), the rows' k-row coverage in up
    n_rc = min(m, 8)
    route_cols = np.array([rng.choice(np.flatnonzero(classes == q)) for q in range(n_rc)], dtype=np.int64)
    route_cols_s = (np.array([rng.choice(np.flatnonzero(classes_s == q)) for q in range(n_rc)], dtype=np.int64)
                    if I_s else np.zeros(0, dtype=np.int64))

    # ---- reserved coordinates
    n_rg, n_cg = -(-E // ROUTE_PER_GROUP), -(-m // G)
    assert n_rg + n_cg < ngr, "no quantisation group left for the probe coordinates"
    gperm = rng.permutation(ngr)
    route_groups, ctl_groups = np.sort(gperm[:n_rg]), np.sort(gperm[n_rg:n_rg + n_cg])
    route_rows = np.empty(E, dtype=np.int64)
    per = -(-E // n_rg)
    for i, g in enumerate(route_groups):
        es = np.arange(i, E, n_rg)
        route_rows[es] = g * G + rng.choice(G, size=es.size, replace=False)
    assert per <= ROUTE_PER_GROUP
    ctl_pool = (ctl_groups[:, None] * G + np.arange(G)[None, :]).reshape(-1)
    ctl_rows = np.sort(rng.choice(ctl_pool, size=m, replace=False))
    reserved = np.zeros(H, dtype=bool)
    reserved[route_rows] = reserved[ctl_rows] = True
    probe_rows = np.flatnonzero(~reserved)

    # ---- up runs: probe chunks as make_exact_case sizes them, at the up half's column variance, plus the E
    #      routing terms +-1
    nnz = int(max(4, min(probe_rows.size // 4, ((FP16_EXACT_INT / 8.0) ** 2 - E) / (X_VAR * W_VAR),
                         ((FP16_EXACT_INT / 5.5) ** 2 - E) / (X_VAR * W_VAR_MAX))))
    n_chunks = -(-probe_rows.size // nnz)
    chunk_perm = rng.permutation(probe_rows)

    xs, ids, kind, ctl = [], [], [], []

    def team_order(team):
        return np.sort(team)[::-1] if order == "descending" else np.sort(team)

    for ch in range(n_chunks):
        for team in _teams(rng, E, k, n_group, topk_group):
            x = np.zeros(H, dtype=np.int8)
            rows = chunk_perm[ch * nnz:(ch + 1) * nnz]
            x[rows] = rng.choice(X_VALUES, size=rows.size, p=X_PROBS)
            x[route_rows] = -1
            x[route_rows[team]] = 1
            xs.append(x), ids.append(team_order(team)), kind.append(0), ctl.append(-1)
    for c in range(m):
        for team in _teams(rng, E, k, n_group, topk_group):
            x = np.zeros(H, dtype=np.int8)
            x[route_rows[team]] = 1
            x[ctl_rows[c]] = 1
            xs.append(x), ids.append(team_order(team)), kind.append(1), ctl.append(c)
    x_units = np.stack(xs)
    ids = np.stack(ids).astype(np.int32)
    kind, ctl = np.array(kind, dtype=np.int8), np.array(ctl, dtype=np.int32)
    R = x_units.shape[0]

    # ---- the guarantees that follow from the plan
    f32 = np.float32
    row_abs = np.abs(x_units).astype(np.int64).sum(axis=1)
    assert int(row_abs.max()) * RAW_CODE < PARTIAL_LIMIT, "gate|up raw-code sums may leave the exact fp32 range"
    assert int(row_abs.max()) * 60 < PARTIAL_LIMIT, "gate|up partial sums may leave the exact range"
    for cls, rc, limit in ((classes, route_cols, Y_LIMIT), (classes_s, route_cols_s, FP16_EXACT_INT)):
        if cls.size:
            # sum |u| over a class's columns in a down run, and the down outputs' bound
            u_abs = np.bincount(cls, minlength=m) + k * np.bincount(cls[rc], minlength=m)
            assert int(u_abs.max()) * 60 <= limit, "a down output may leave its limit"
            assert int(u_abs.max()) * RAW_CODE < PARTIAL_LIMIT, "down raw-code sums may leave the exact fp32 range"
    assert f32(f32(k) + f32(E * np.exp(-32.0))) == f32(k), "exp(-32) of the unselected experts shows in the sum"
    assert f32(1) / (f32(1) + f32(np.exp(-MOE_LOGIT))) == f32(1)          # sigmoid(32) = 1, sigmoid(0) = 0.5
    # silu(-64) u with |u| <= k + 1 units (down runs; up runs have g = 0): below half the smallest fp16 subnormal
    assert 64.0 * np.exp(-64.0) * k1 * unit < 2.0**-25
    assert GATE_ON * k1 * unit <= FP16_EXACT_INT * 2.0**-5                # act = 32 u: an fp16 value
    sel_mask = np.zeros((R, E), dtype=bool)
    np.put_along_axis(sel_mask, ids.astype(np.int64), True, axis=1)
    assert (sel_mask.sum(axis=1) == k).all(), "a team repeats an expert"
    # every selected expert's logit is 32, every other one's 0 or -32
    assert (x_units[:, route_rows][sel_mask] == 1).all() and (x_units[:, route_rows][~sel_mask] <= 0).all()
    if n_group > 1:
        gsz = E // n_group
        assert all(np.unique(r // gsz).size <= topk_group for r in ids), "a team spans too many expert groups"

    # ---- coverage: (expert, k-row) of gate|up and of down, slots
    nz = (x_units != 0)
    cov_gu = np.zeros((E, H), dtype=bool)
    cov_dn = np.zeros((E, I), dtype=bool)
    for e in range(E):
        runs = np.flatnonzero(sel_mask[:, e])
        cov_gu[e] = nz[runs].any(axis=0)
        on = np.unique(ctl[runs][kind[runs] == 1])
        cov_dn[e] = np.isin(classes, on)
    assert cov_gu.all(), f"{int((~cov_gu).sum())} (expert, gate|up k-row) pairs are not hit"
    assert cov_dn.all(), f"{int((~cov_dn).sum())} (expert, down k-row) pairs are not hit"
    if I_s:
        assert nz.any(axis=0).all() and np.isin(classes_s, ctl[kind == 1]).all(), "a shared-expert k-row is not hit"
    slot_hits = np.zeros((E, k), dtype=np.int64)
    np.add.at(slot_hits, (ids.astype(np.int64), np.broadcast_to(np.arange(k), ids.shape)), 1)
    first, last = (E - 1, 0) if order == "descending" else (0, E - 1)
    assert slot_hits[first, 0] > 0 and slot_hits[last, k - 1] > 0
    bias = (np.arange(E, dtype=np.float32) * f32(2.0**-12) if order == "descending" else np.zeros(E, dtype=np.float32))

    return dict(op=op, E=E, top_k=k, H=H, I=I, G=G, I_s=I_s, renormalize=renormalize, scoring=scoring,
                n_group=n_group, topk_group=topk_group, rsf=rsf, order=order, unit=float(unit), unit2=float(unit2),
                seed=seed, x_units=x_units, ids=ids, kind=kind, ctl=ctl, route_rows=route_rows, ctl_rows=ctl_rows,
                route_groups=route_groups, ctl_groups=ctl_groups, classes=classes, classes_s=classes_s, m=m,
                route_cols=route_cols, route_cols_s=route_cols_s,
                nnz=nnz, runs=R, weight=_designed_weight(op, k, renormalize, scoring, rsf), bias=bias,
                cov_gu=cov_gu, cov_dn=cov_dn, slot_hits=slot_hits)


def _pack_words_torch(v):
    """[.., 8C] ints 0..15 (torch) -> [.., C] int32 with the AWQ interleave (O.pack_gemm_words)."""
    import torch

    v = v.to(torch.int32).reshape(*v.shape[:-1], -1, O.PACK)
    w = torch.zeros(v.shape[:-1], dtype=torch.int32, device=v.device)
    for j in range(O.PACK):
        w |= v[..., j] << (4 * int(O.AWQ_REVERSE_ORDER[j]))
    return w


def unpack_words_torch(w):
    """Inverse of _pack_words_torch: [.., C] int32 -> [.., 8C] int16 in 0..15."""
    import torch

    sh = torch.tensor([4 * int(O.AWQ_REVERSE_ORDER[j]) for j in range(O.PACK)], dtype=torch.int32, device=w.device)
    return ((w.unsqueeze(-1) >> sh) & 0xF).reshape(*w.shape[:-1], -1).to(torch.int16)


def _expert_w1(c, gen, device, n_cols, cls, route_cols):
    """One expert's [H, 2 n_cols] gate | up as GEMM-layout (qweight, scales, qzeros) (see make_exact_moe_case)."""
    import torch

    H, G, ngr = c["H"], c["G"], c["H"] // c["G"]
    N = 2 * n_cols
    q = torch.randint(0, 16, (H, N), generator=gen, device=device, dtype=torch.int16)
    z = torch.randint(0, 16, (ngr, N), generator=gen, device=device, dtype=torch.int16)
    probs = torch.tensor(SCALE_PROBS, device=device, dtype=torch.float32)
    steps = torch.tensor(SCALE_STEPS, device=device, dtype=torch.float32)[
        torch.multinomial(probs, ngr * N, replacement=True, generator=gen)].view(ngr, N)
    route_g = torch.as_tensor(c["route_groups"], device=device)
    ctl_g = torch.as_tensor(c["ctl_groups"], device=device)
    # gate half: zero everywhere but the control rows
    q[:, :n_cols] = z[:, :n_cols].repeat_interleave(G, dim=0)
    z[ctl_g, :n_cols] = GATE_ZERO
    for g in c["ctl_groups"]:
        q[g * G:(g + 1) * G, :n_cols] = GATE_ZERO
    ctl_rows = torch.as_tensor(c["ctl_rows"], device=device)
    cls_t = torch.as_tensor(cls, device=device, dtype=torch.int64)
    on = cls_t[None, :] == torch.arange(c["m"], device=device)[:, None]                  # [m, n_cols]
    q[ctl_rows, :n_cols] = torch.where(on, 12, 0).to(torch.int16)
    s = steps * c["unit"]
    s[ctl_g, :n_cols] = GATE_SCALE
    # up half: step 1 in the groups holding reserved rows, q - z = +-1 on the reserved rows
    spec = torch.cat([route_g, ctl_g])
    s[spec, n_cols:] = c["unit"]
    res = torch.cat([torch.as_tensor(c["route_rows"], device=device), ctl_rows])
    zr = z[res // G, n_cols:]
    sign = torch.where(torch.rand(zr.shape, generator=gen, device=device) < 0.5, -1, 1).to(torch.int16)
    sign = torch.where(zr == 0, 1, torch.where(zr == 15, -1, sign)).to(torch.int16)
    keep = torch.zeros((res.numel(), n_cols), dtype=torch.bool, device=device)
    keep[c["E"]:] = True                                                                   # control rows: every column
    keep[:c["E"], torch.as_tensor(route_cols, device=device)] = True                       # routing rows: routing columns
    q[res, n_cols:] = torch.where(keep, zr + sign, zr).to(torch.int16)
    return _pack_words_torch(q), s.half(), _pack_words_torch(z)


def _expert_w2(c, gen, device, K):
    import torch

    H, G = c["H"], c["G"]
    q = torch.randint(0, 16, (K, H), generator=gen, device=device, dtype=torch.int16)
    z = torch.randint(0, 16, (K // G, H), generator=gen, device=device, dtype=torch.int16)
    probs = torch.tensor(SCALE_PROBS, device=device, dtype=torch.float32)
    steps = torch.tensor(SCALE_STEPS, device=device, dtype=torch.float32)[
        torch.multinomial(probs, (K // G) * H, replacement=True, generator=gen)].view(K // G, H)
    return _pack_words_torch(q), (steps * c["unit2"]).half(), _pack_words_torch(z)


def moe_weights(c: dict, device) -> dict:
    """The block's tensors for a plan, drawn with torch on `device` from the plan's seed, expert by expert (distinct
    weights per expert): gate [E, H] fp16 (one-hot 32), w1 / w2 stacked GEMM-layout (qweight, scales, qzeros), ws1 /
    ws2 (2-D, DeepSeek) and bias [E] fp32."""
    import torch

    E, H, I, G = c["E"], c["H"], c["I"], c["G"]
    gen = torch.Generator(device=device).manual_seed(int(c["seed"]) * 7919 + 17)
    gate = torch.zeros((E, H), dtype=torch.float16, device=device)
    gate[torch.arange(E, device=device), torch.as_tensor(c["route_rows"], device=device)] = MOE_LOGIT
    w1 = [torch.empty((E, H, 2 * I // 8), dtype=torch.int32, device=device),
          torch.empty((E, H // G, 2 * I), dtype=torch.float16, device=device),
          torch.empty((E, H // G, 2 * I // 8), dtype=torch.int32, device=device)]
    w2 = [torch.empty((E, I, H // 8), dtype=torch.int32, device=device),
          torch.empty((E, I // G, H), dtype=torch.float16, device=device),
          torch.empty((E, I // G, H // 8), dtype=torch.int32, device=device)]
    for e in range(E):
        for dst, src in zip(w1, _expert_w1(c, gen, device, I, c["classes"], c["route_cols"])):
            dst[e] = src
        for dst, src in zip(w2, _expert_w2(c, gen, device, I)):
            dst[e] = src
    out = dict(gate=gate, w1=tuple(w1), w2=tuple(w2), bias=torch.as_tensor(c["bias"], device=device))
    if c["I_s"]:
        out["ws1"] = _expert_w1(c, gen, device, c["I_s"], c["classes_s"], c["route_cols_s"])
        out["ws2"] = _expert_w2(c, gen, device, c["I_s"])
    return out


def dequant_torch(qweight, scales, qzeros):
    """fp64 [K, N] (q - z) s of one GEMM-layout weight: exact (integers times fp16 scales)."""
    import torch

    q = unpack_words_torch(qweight).to(torch.float64)
    G = q.shape[0] // scales.shape[0]
    z = unpack_words_torch(qzeros).to(torch.float64).repeat_interleave(G, dim=0)
    return (q - z) * scales.to(torch.float64).repeat_interleave(G, dim=0)


def moe_dequant(W: dict, which: str, e) -> "torch.Tensor":  # noqa: F821
    """fp64 weights of expert e's w1 / w2, or ("ws1" / "ws2", None) of the shared expert."""
    return dequant_torch(*W[which]) if which in ("ws1", "ws2") else dequant_torch(*(t[e] for t in W[which]))


def _fp16_exact(t, what):
    import torch

    bad = t.to(torch.float16).to(torch.float64) != t
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} values are not fp16 values (the probe is not exact)"


def moe_expected(c: dict, W: dict, runs=None, read=None, deq=None) -> dict:
    """The exact buffers of the block on the plan's runs (all, or the index array `runs`), one token per run, on W's
    device: logits, topk_ids, topk_weights, gate_up, act, down (the per-slot c), out, and shared_out (DeepSeek), in the
    moe_buffers layout with a leading run axis.  Asserts the data-dependent limits: every gate|up value, every per-slot
    down output (within Y_LIMIT units), every shared down output and act are fp16 values, and every gate is 0, +32 or
    -64.  c = fp16(fp32(y) w) and the combine are the kernels' documented roundings applied to exact values.

    Fault models for the CPU tests: read[r, s] names the expert whose weights slot s of run r reads (default: the
    recorded id); deq(which, e) replaces moe_dequant (the fp64 weights the block contracts)."""
    import torch

    op, E, k, H, I, I_s = c["op"], c["E"], c["top_k"], c["H"], c["I"], c["I_s"]
    dev = W["gate"].device
    f64, f16, f32 = torch.float64, torch.float16, torch.float32
    runs = np.arange(c["runs"]) if runs is None else np.asarray(runs)
    R = runs.size
    x = torch.as_tensor(c["x_units"][runs], device=dev).to(f64)
    ids = torch.as_tensor(c["ids"][runs].astype(np.int64), device=dev)
    rd = ids if read is None else torch.as_tensor(np.asarray(read)[runs].astype(np.int64), device=dev)
    deq = deq or (lambda which, e: moe_dequant(W, which, e))
    w1_of, w2_of = (lambda e: deq("w1", e)), (lambda e: deq("w2", e))
    gu = torch.zeros((R, k, 2 * I), dtype=f64, device=dev)
    for e in torch.unique(rd).tolist():
        rr, ss = torch.nonzero(rd == e, as_tuple=True)
        gu[rr, ss] = x[rr] @ w1_of(e)
    _fp16_exact(gu, "gate|up")

    def act_of(g_u, n):
        g, u = g_u[..., :n], g_u[..., n:]
        assert bool(((g == 0) | (g == GATE_ON) | (g == GATE_OFF)).all()), "a gate is not 0, +32 or -64"
        a = torch.where(g == GATE_ON, GATE_ON * u, torch.zeros_like(u))
        _fp16_exact(a, "act")
        return a

    act = act_of(gu, I)
    ulim = float(2 * FP16_EXACT_INT * c["unit"])
    assert bool((gu[..., I:].abs() <= ulim).all())
    y = torch.zeros((R, k, H), dtype=f64, device=dev)
    for e in torch.unique(rd).tolist():
        rr, ss = torch.nonzero(rd == e, as_tuple=True)
        y[rr, ss] = act[rr, ss] @ w2_of(e)
    g_y = GATE_ON * c["unit"] * c["unit2"]
    assert float(y.abs().max()) <= Y_LIMIT * g_y, f"a down output is past {Y_LIMIT} units: more classes"
    _fp16_exact(y, "down y")
    w = torch.full((R, k), c["weight"], dtype=f32, device=dev)
    cc = (y.to(f32) * w.unsqueeze(-1)).to(f16)                       # c = fp16(fp32(y) w): one unit of y shows in c
    cmax = float(cc.abs().max().float())
    if cmax > 0:
        assert 2.0 ** (np.floor(np.log2(cmax)) - 10) < g_y * c["weight"], "one unit of y can hide in c's rounding"
    order_ = torch.argsort(ids, dim=1, stable=True)                   # the combine runs in ascending expert id
    cs = torch.gather(cc, 1, order_.unsqueeze(-1).expand(R, k, H))
    if op == "sparse":
        out = cs.to(f32).sum(dim=1).to(f16)                           # fp32 sum over the slots, rounded once
    else:
        out = torch.zeros((R, H), dtype=f16, device=dev)
        for j in range(k):
            out = (out.to(f32) + cs[:, j].to(f32)).to(f16)            # fp16(out + c)
    res = dict(topk_ids=ids.to(torch.int32), gate_up=gu.to(f16), act=act.to(f16), down=cc, out=out)
    logit = MOE_LOGIT * x[:, torch.as_tensor(c["route_rows"], device=dev)]
    res["logits"] = logit.to(f32 if op == "deepseek" else f16)
    res["topk_weights"] = w.to(f16) if op == "qwen3" else w
    if I_s:
        gus = x @ deq("ws1", None)
        _fp16_exact(gus, "shared gate|up")
        acts = act_of(gus, I_s)
        ys = acts @ deq("ws2", None)
        assert float(ys.abs().max()) <= FP16_EXACT_INT * g_y, "a shared down output is not an fp16 value"
        _fp16_exact(ys, "shared down")
        res["gate_up"] = torch.cat([res["gate_up"].reshape(R, -1), gus.to(f16)], dim=1)
        res["act"] = torch.cat([res["act"].reshape(R, -1), acts.to(f16)], dim=1)
        res["shared_out"] = ys.to(f16)
        res["out"] = (out.to(f32) + ys.to(f32)).to(f16)              # out = fp16(r + y_s)
    return res
