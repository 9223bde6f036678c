"""CPU checks of the error model (oracle/llm_data.forward_tolerance) on the LLM-shaped data, against float32 models of
the three families' arithmetic written from the kernel source:

  offset-fold: each k16 block's sum of x (1024 + c q) and of x rounded to fp32 once (the mma.sync result), the blocks of
               a group summed in fp32, folded s/c (S - (1024 + c z) X) in fp32 (gemv_tile.cuh:v3_fold_reg);
  code-fold:   per 32-k chunk sequential fp32 sums of x q and of x, folded s (S - z X) (gemv.cu:857-890);
  exact-dequant: fp16 dequantised weights, each k16 block's sum of products rounded to fp32, blocks summed in fp32.

They show that the bound holds for the arithmetic with room to spare, that the fold term is forced by it (the old bound
without it fails on the zero columns), and that it is tight enough to catch a kernel that keeps a sum in fp16."""
import numpy as np
import pytest

from oracle import llm_data as L

K, N, G, M = 2048, 512, 128, 6
CASES = [(kind, seed) for kind in ("llm", "overflow", "cancel") for seed in (0, 1)]


@pytest.fixture(scope="module", params=CASES, ids=[f"{k}-{s}" for k, s in CASES])
def case(request):
    kind, seed = request.param
    return L.make_llm_case(K, N, G, M, seed=seed + 11, kind=kind)


def _kind_c(n):
    return np.where(((np.arange(n) & 7) >> 1) & 1, 16.0, 1.0)


def _blocks_f32(x, a, blk):
    """[M, K] x [K, N] -> [M, K/blk, N]: each block's exact sum rounded to fp32 once."""
    Mx, Kx = x.shape
    xb = x.astype(np.float64).reshape(Mx, Kx // blk, blk)
    ab = a.astype(np.float64).reshape(Kx // blk, blk, -1)
    return np.einsum("mbk,bkn->mbn", xb, ab).astype(np.float32)


def _seq_f32(parts, axis):
    acc = np.zeros(np.delete(parts.shape, axis), dtype=np.float32)
    for i in range(parts.shape[axis]):
        acc = (acc + np.take(parts, i, axis=axis)).astype(np.float32)
    return acc


def offset_fold_model(c, x, x_block_fp16=False, s_fp16=False, partial_fp16=False):
    q = c["intweight"].astype(np.float64)
    z = c["zeros"].astype(np.float64)
    s = c["scales"].astype(np.float32)
    cc = _kind_c(q.shape[1])
    codes = 1024.0 + cc[None, :] * q
    Sb = _blocks_f32(x, codes, 16)                                   # [M, K/16, N]
    Xb = _blocks_f32(x, np.ones((x.shape[1], 1)), 16)[:, :, 0]       # [M, K/16]
    if x_block_fp16:
        Xb = Xb.astype(np.float16).astype(np.float32)
    nb = G // 16
    ng = x.shape[1] // G
    with np.errstate(over="ignore", invalid="ignore"):
        S = _seq_f32(Sb.reshape(x.shape[0], ng, nb, -1), 2)          # [M, ng, N]
        X = _seq_f32(Xb.reshape(x.shape[0], ng, nb), 2)               # [M, ng]
        if s_fp16:
            S = S.astype(np.float16).astype(np.float32)
        zoff = (1024.0 + cc[None, :] * z).astype(np.float32)          # [ng, N]
        t = ((S - (zoff[None] * X[:, :, None]).astype(np.float32)).astype(np.float32)
             * (s / cc[None, :].astype(np.float32))[None]).astype(np.float32)
        halves = [_seq_f32(t[:, :ng // 2], 1), _seq_f32(t[:, ng // 2:], 1)]   # split-K: two K halves
        if partial_fp16:
            halves = [h.astype(np.float16).astype(np.float32) for h in halves]
        y = (halves[0] + halves[1]).astype(np.float32)
        return _finish(c, y)


def code_fold_model(c, x):
    q = c["intweight"].astype(np.float32)
    z = c["zeros"].astype(np.float32)
    s = c["scales"].astype(np.float32)
    Mx, Kx = x.shape
    xf = x.astype(np.float32)
    nch = Kx // 32
    S = np.zeros((Mx, nch, q.shape[1]), dtype=np.float32)
    X = np.zeros((Mx, nch), dtype=np.float32)
    for i in range(32):
        k = np.arange(nch) * 32 + i
        S = (S + xf[:, k, None] * q[None, k, :]).astype(np.float32)   # exact product, one fp32 rounding
        X = (X + xf[:, k]).astype(np.float32)
    g = (np.arange(nch) * 32) // G
    with np.errstate(over="ignore", invalid="ignore"):
        t = (s[g][None] * (S - (z[g][None] * X[:, :, None]).astype(np.float32))).astype(np.float32)
        return _finish(c, _seq_f32(t, 1))


def exact_dequant_model(c, x):
    with np.errstate(over="ignore", invalid="ignore"):
        return _finish(c, _seq_f32(_blocks_f32(x, c["w"], 16), 1))


def _finish(c, y):
    if c.get("bias") is not None:
        y = (y + c["bias"].astype(np.float32)[None]).astype(np.float32)
    with np.errstate(over="ignore"):
        return y.astype(np.float16)


def _y64(c, x):
    y = x.astype(np.float64) @ c["w"].astype(np.float64)
    return y + (c["bias"].astype(np.float64) if c.get("bias") is not None else 0.0)


def _ratio(c, y, family):
    """Largest error / bound over the columns that must come back finite; the high overflow columns must be inf with
    the sign of the exact value."""
    x = c["x"]
    y64 = _y64(c, x)
    hi = c["ovf_high"]
    if len(hi):
        assert np.isinf(y[:, hi]).all() and (np.sign(y[:, hi]) == np.sign(y64[:, hi])).all()
    keep = np.setdiff1d(np.arange(y.shape[1]), hi)
    tol = L.forward_tolerance(x, c, family, cols=keep, y64=y64[:, keep])
    err = np.abs(y[:, keep].astype(np.float64) - y64[:, keep])
    assert np.isfinite(err).all()
    return float((err / tol).max())


def _old_bound(c, x, wr):
    y64 = _y64(c, x)
    return L.RTOL * np.abs(y64) + wr * (np.abs(x.astype(np.float64)) @ np.abs(c["w"].astype(np.float64))) + L.ATOL


def test_fold_models_use_at_most_half_of_their_bound(case):
    assert _ratio(case, offset_fold_model(case, case["x"]), "offset-fold") <= 0.5
    assert _ratio(case, code_fold_model(case, case["x"]), "code-fold") <= 0.5


def test_fold_term_is_forced_on_zero_columns(case):
    if case["kind"] != "llm":
        pytest.skip("zero columns live in the llm cases")
    x, zc = case["x"], case["zero_cols"]
    y = offset_fold_model(case, x).astype(np.float64)
    err = np.abs(y - _y64(case, x))
    old = _old_bound(case, x, L.WR_FOLD)
    assert (err[:, zc] > old[:, zc]).any(), "the offset fold met the bound without a fold term on the zero columns"
    # and the new bound holds there
    tol = L.forward_tolerance(x, case, "offset-fold", cols=zc)
    assert (err[:, zc] <= tol).all()


def test_exact_dequant_meets_the_old_bound(case):
    x = case["x"]
    y = exact_dequant_model(case, x)
    assert _ratio(case, y, "exact-dequant") <= 1.0
    keep = np.setdiff1d(np.arange(N), case["ovf_high"])
    err = np.abs(y.astype(np.float64) - _y64(case, x))[:, keep]
    assert (err <= _old_bound(case, x, L.WR_EXACT)[:, keep]).all()
    if len(case["zero_cols"]):
        want = np.broadcast_to(case["bias"][case["zero_cols"]], (M, len(case["zero_cols"])))
        assert np.array_equal(y[:, case["zero_cols"]], want)


def _exceeds(c, y, family):
    x = c["x"]
    y64 = _y64(c, x)
    keep = np.setdiff1d(np.arange(y.shape[1]), c["ovf_high"])
    tol = L.forward_tolerance(x, c, family, cols=keep, y64=y64[:, keep])
    err = np.abs(y[:, keep].astype(np.float64) - y64[:, keep])
    return bool((~(err <= tol)).any())


@pytest.mark.parametrize("fault", ["x_block_fp16", "s_fp16", "partial_fp16"])
def test_precision_faults_exceed_the_bound(fault):
    hits = []
    for kind, seed in CASES:
        c = L.make_llm_case(K, N, G, M, seed=seed + 11, kind=kind)
        y = offset_fold_model(c, c["x"], **{fault: True})
        hits.append(_exceeds(c, y, "offset-fold"))
        if fault == "partial_fp16" and kind == "cancel":
            assert not np.isfinite(y[:, c["cancel"]]).all(), "fp16 split-K partials stayed finite on cancelling columns"
    assert any(hits), f"{fault}: within the bound on every case"


def test_fold_r_is_derived_not_fitted():
    assert L.fold_r("offset-fold", 128) == 34 and L.fold_r("code-fold", 128) == 35
    assert L.fold_r("exact-dequant", 128) == 0 and L.fold_r("fast-dequant", 128) == 0
    assert L.fold_r("offset-fold", 32) == 11 and L.fold_r("offset-fold", 4096) == 1026
