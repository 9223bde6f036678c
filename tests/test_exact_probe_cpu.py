"""CPU tests of the exact-arithmetic probes (oracle/exact_probe.py).

Three things: the generator's guarantees hold at every shape tests/test_gpu_exact_probes.py uses; its reference is
the oracle's (fp64 contraction of the bit-exact dequantised weights, already an fp16 value); and the reason the
probes exist - index faults injected into the reference product are ALL flagged by exact comparison on a probe,
while the rounding tolerance of the forward tests, on their Gaussian data at the `down` shape, lets several pass.
"""
import numpy as np
import pytest

from oracle import awq_oracle as O
from oracle import exact_probe as E

# every (K, N, G) of tests/test_gpu_exact_probes.py (kept in step by test_shapes_are_the_gpu_tests)
MODEL_SHAPES = [(4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096), (8192, 1280), (1024, 8192), (8192, 7168),
                (3584, 8192)]
EDGE_SHAPES = [(1024, 1936, 128), (512, 96, 128), (256, 40, -1), (384, 256, 128), (1152, 384, 128), (1152, 384, 64),
               (512, 256, 32), (2048, 640, -1), (576, 128, 64)]


def test_shapes_are_the_gpu_tests():
    import ast
    import os

    src = open(os.path.join(os.path.dirname(__file__), "test_gpu_exact_probes.py")).read()
    consts = {n.targets[0].id: ast.literal_eval(n.value) for n in ast.parse(src).body
              if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Name)
              and n.targets[0].id in ("MODEL_SHAPES", "EDGE_SHAPES")}
    assert [tuple(s[1:]) for s in consts["MODEL_SHAPES"]] == MODEL_SHAPES
    assert consts["EDGE_SHAPES"] == EDGE_SHAPES


@pytest.mark.parametrize("K,N,G", [(K, N, 128) for K, N in MODEL_SHAPES] + EDGE_SHAPES)
def test_generator_guarantees(K, N, G):
    """The assertions inside make_exact_case pass (bounds only: no product, no packing), rows cover every k, and the
    density keeps the activations mostly zero."""
    c = E.make_exact_case(K, N, G, 64, seed=K % 97 + N % 89, bias=True, layouts=(), reference=False)
    M = max(2, c["cover_rows"])
    c = E.make_exact_case(K, N, G, M, seed=K % 97 + N % 89, bias=True, layouts=(), reference=False)
    xu = c["x_units"]
    assert ((xu[:c["cover_rows"]] != 0).sum(axis=0) == 1).all()            # 100 % of k, each exactly once
    assert set(np.unique(xu)) <= {-2, -1, 0, 1, 2} and (xu != 0).mean() <= 0.25
    assert np.array_equal(c["x"].astype(np.int8), xu)
    assert set(np.unique(c["scale_steps"])) == {1, 2, 4}
    assert np.abs(c["w_units"]).max() <= 60 and c["bias"] is not None


@pytest.mark.parametrize("K,N,G,M", [(512, 256, 128, 21), (1152, 384, 64, 9), (256, 40, -1, 5), (4096, 4096, 128, 33),
                                     (576, 128, 64, 3)])
def test_reference_is_the_oracles(K, N, G, M):
    c = E.make_exact_case(K, N, G, M, seed=3, bias=True, zero_col_frac=0.1)
    Gs = c["group_size"]
    w = O.dequantize_gemm(c["qweight"], c["qzeros"], c["scales"], Gs)
    assert np.array_equal(w.astype(np.float64), c["w_units"] * c["unit"])
    y64 = O.gemm_f64(c["x"], w) + c["bias"].astype(np.float64)
    assert np.array_equal(y64, c["y_exact"])
    assert np.array_equal(y64.astype(np.float16).astype(np.float64), y64)       # its own fp16 rounding
    assert np.array_equal(O.wqlinear_forward(c["x"], c["qweight"], c["qzeros"], c["scales"], Gs, c["bias"]),
                          c["y_exact"].astype(np.float16))
    # the integer contraction behind y_exact, in int64
    yi = c["x_units"].astype(np.int64) @ c["w_units"].astype(np.int64)
    assert np.array_equal((c["y_exact"] - c["bias"].astype(np.float64)) / c["unit"], yi)
    # the three packings hold the same matrix
    assert np.array_equal(O.dequantize_gemv(*c["gemv"], Gs), w)
    assert np.array_equal(O.dequantize_gemv_fast_f64(*c["fast"], Gs), w.astype(np.float64))
    assert (c["scales"][:, ~c["scale_steps"].any(axis=0)] == 0).all() and (~c["scale_steps"].any(axis=0)).any()


def test_generator_refuses_a_case_that_is_not_exact():
    """Dense activation rows: the raw-code sums of the GEMV kernels could pass 2^20, and the generator says so instead
    of returning a case that might be exact by luck."""
    with pytest.raises(AssertionError, match="exact fp32 range"):
        E.make_exact_case(4096, 256, 128, 8, seed=0, nnz=4096)


def test_mismatch_report_names_rows_columns_and_units():
    want = np.zeros((3, 32))
    got = want.copy()
    got[1, 16:32] = 0.5
    msg = E.mismatch_report(got, want, 0.25)
    assert "16 / 96" in msg and "columns 16..31" in msg and "(1, 16): +2" in msg


# ------------------------------------------------------------------------------------------ mutation sensitivity
def _deq(iw_rows, z_row, s_row):
    """fp16((q - z) * s) as float64, the weights every kernel path contracts."""
    return ((iw_rows.astype(np.float16) - z_row.astype(np.float16)) * s_row.astype(np.float16)).astype(np.float64)


def _mutations(x, w, y, iw, iz, s, G, k):
    """name -> the product a kernel with that index fault would return (fp64), from the true product y = x . w.
    k: the k-row the row faults hit (k + 1 in the same group, k >= G)."""
    K = w.shape[0]
    g = k // G
    rows = slice(g * G, (g + 1) * G)
    out = {
        "drop row k": y - np.outer(x[:, k], w[k]),
        "drop last row": y - np.outer(x[:, K - 1], w[K - 1]),
        "row K-1 reads row K-2": y + np.outer(x[:, K - 1], w[K - 2] - w[K - 1]),
        "swap rows k, k+1": y + np.outer(x[:, k] - x[:, k + 1], w[k + 1] - w[k]),
        "row k counted twice": y + np.outer(x[:, k], w[k]),
        "neighbour group's scales": y + x[:, rows] @ (_deq(iw[rows], iz[g], s[g - 1]) - w[rows]),
        "neighbour group's zeros": y + x[:, rows] @ (_deq(iw[rows], iz[g - 1], s[g]) - w[rows]),
    }
    sh = y.copy()
    sh[:, 32:48] = y[:, 48:64]
    out["16-column set shifted by one set"] = sh
    if y.shape[0] > 1:
        ex = y.copy()
        ex[[0, 1]] = y[[1, 0]]
        out["two token rows exchanged"] = ex
    return out


K_DOWN, N_DOWN, G_DOWN = 14336, 4096, 128


def test_exact_probe_flags_every_injected_fault():
    c = E.make_exact_case(K_DOWN, N_DOWN, G_DOWN, 64, seed=7, layouts=())
    assert c["cover_rows"] <= 64                                            # so every k meets a non-zero activation
    x = c["x"].astype(np.float64)
    w = c["w_units"] * c["unit"]
    # faults at a tile boundary inside a group, in the first row of a group, and next to the end
    for k in (128 + 63, 5 * 128, K_DOWN - 2):
        muts = _mutations(x, w, c["y_exact"], c["intweight"], c["zeros"], c["scales"], G_DOWN, k)
        assert len(muts) == 9
        for name, ym in muts.items():
            got = ym.astype(np.float16)                                     # what a kernel would store
            assert not np.array_equal(got.astype(np.float64), c["y_exact"]), f"k={k}: '{name}' goes unnoticed"
    # a single-row call sees the faults of the k-rows its support covers: the GPU test rotates over cover_rows calls
    one = np.flatnonzero(c["x_units"][0])[0]
    assert not np.array_equal(c["y_exact"][:1] - np.outer(x[:1, one], w[one]), c["y_exact"][:1])


def test_rounding_tolerance_misses_faults_at_the_down_shape():
    """The recipe of tests/test_gpu_shapes.py at 14336 x 4096, M = 1 (same seeds, scales, tolerance and column
    sample), with the fault injected into the fp64 product and the result rounded to fp16."""
    K, N, G = K_DOWN, N_DOWN, G_DOWN
    c = O.make_case(K, N, G, seed=K % 97 + N % 89)
    s = (c["scales"].astype(np.float32) / (6.1 * 0.0108 * np.sqrt(K))).astype(np.float16)
    w = O.dequantize_gemm(c["qweight"], c["qzeros"], s, G).astype(np.float64)
    x = np.random.default_rng(K + N).standard_normal((1, K)).astype(np.float16).astype(np.float64)
    cols = np.unique(np.concatenate([np.arange(0, N, 61), [0, 1, 7, 8, 255, 256, N - 9, N - 8, N - 1]]))
    assert cols.size == 75
    y = x @ w
    tol = 2.0**-10 * np.abs(y) + 2.0**-11 * (np.abs(x) @ np.abs(w)) + 1e-6
    # a k-row inside a group (not its edge) whose activation has the median magnitude
    inner = np.arange(K - 1)[(np.arange(K - 1) % G != G - 1) & (np.arange(K - 1) >= G)]
    k = int(inner[np.argsort(np.abs(x[0, inner]))[inner.size // 2]])
    assert 0.6 < abs(x[0, k]) < 0.75
    muts = _mutations(x, w, y, c["intweight"], c["zeros"], s, G, k)
    bad = {name: np.abs(ym.astype(np.float16).astype(np.float64) - y) > tol for name, ym in muts.items()}
    n_all = {name: int(b.sum()) for name, b in bad.items()}
    n_cols = {name: int(b[:, cols].sum()) for name, b in bad.items()}
    # passes unseen on every one of the 4096 columns
    assert n_all["drop last row"] == 0 and n_all["row K-1 reads row K-2"] == 0, n_all
    # a dropped or double-counted row of median weight moves a handful of outputs out of 4096 past the tolerance, none
    # of them on the sampled columns
    for name in ("drop row k", "row k counted twice", "swap rows k, k+1"):
        assert n_all[name] <= 8 and n_cols[name] == 0, (name, n_all[name], n_cols[name])
    # what the tolerance does see: a whole group's scales or zeros, and misplaced columns
    for name in ("neighbour group's scales", "neighbour group's zeros", "16-column set shifted by one set"):
        assert n_all[name] > 0, name
    # the unfaulted product rounds inside the tolerance, of course
    assert not (np.abs(y.astype(np.float16).astype(np.float64) - y) > tol).any()
