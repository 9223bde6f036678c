"""The tensor-core kernels under programmatic dependent launch (knob 4: what bench.py runs with) inside a CUDA graph.

A launch under PDL may start while its predecessor still runs; every kernel must wait (`griddepcontrol.wait`) before it
touches the activations, the split-K workspace or its output.  The rest of the GPU suite runs without the attribute,
so this test replays graphs of back-to-back linears with and without it:

  * independent launches on different weights and token counts: the small-M kernel (5 <= M <= 128), the general
    kernel above 128 tokens, with and without split-K, and the register-staged kernel at small M (knob 19);
  * dependent chains: the output buffer of the first linear is cleared inside the graph and then read by the second,
    so a consumer that reads its activations before the producer finished sees zeros or partial sums.

Every output is checked against the fp64 oracle, and the split-K workspace must be all-zero afterwards."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O

pytestmark = pytest.mark.gpu

G = 128
# (K, N, M): small-M kernel tiles 16 / 32 / 64 / 128, ragged M; then M > 128 split-K (4 tiles x 64 k-steps) and M > 128
# whole tiles
INDEPENDENT = [(1024, 1792, 16), (2048, 640, 64), (1024, 1792, 8), (512, 256, 100), (4096, 512, 33), (1024, 1792, 128),
               (4096, 512, 160), (2048, 1024, 300)]
CHAINS = [1, 16, 200]   # M of a chain x[M, 1024] -> [M, 2048] -> [M, 512]: GEMV, small-M kernel, general kernel


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _check(y, ref, bud, gemv, what):
    wr = 2.0**-11 if gemv else 2.0**-16       # the GEMV rounds per weight; the tensor-core paths use the exact A tile
    got = y.cpu().numpy().astype(np.float64)
    tol = 2.0**-10 * np.abs(ref) + wr * bud + 1e-6
    bad = int((np.abs(got - ref) > tol).sum()) + int((~np.isfinite(got)).sum())
    assert bad == 0, f"{what}: {bad} / {got.size} outside tolerance, max err {np.nanmax(np.abs(got - ref)):.3e}"


def _workspace_clean(ext):
    torch.cuda.synchronize()
    return sum(int(ws.view(torch.int32).ne(0).sum()) for ws in ext._WS.values()) == 0


def _graph(side, fn):
    with torch.cuda.stream(side):
        fn()                      # warm-up: allocates the stream's workspace outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        for _ in range(3):
            fn()
    return g


@pytest.mark.parametrize("staged", [0, 1], ids=["default", "register-staged"])
@pytest.mark.parametrize("pdl", [0, 1], ids=["plain", "pdl"])
def test_independent_linears_in_graph(pdl, staged):
    from autoawq_b200 import ext

    dev = torch.device("cuda:0")
    cases = []
    for i, (K, N, M) in enumerate(INDEPENDENT):
        c = O.make_case(K, N, G, seed=100 + i)
        x = np.random.default_rng(i).standard_normal((M, K)).astype(np.float16)
        w = O.dequantize_gemm(c["qweight"], c["qzeros"], c["scales"], G)
        cases.append((_t(x, dev), _t(c["qweight"], dev), _t(c["scales"], dev), _t(c["qzeros"], dev), O.gemm_f64(x, w),
                      np.abs(x.astype(np.float64)) @ np.abs(w.astype(np.float64)),
                      torch.empty((M, N), dtype=torch.float16, device=dev)))

    def run():
        for xt, qw, sc, qz, _, _, y in cases:
            ext.linear_forward("gemm", xt, qw, sc, qz, G, out=y)

    ext.set_knob(4, pdl)
    ext.set_knob(19, staged)
    try:
        g = _graph(torch.cuda.Stream(), run)
        for c in cases:
            c[-1].zero_()
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    finally:
        ext.set_knob(4, 0)
        ext.set_knob(19, 0)
    for xt, _, _, _, ref, bud, y in cases:
        M = xt.shape[0]     # the GEMV serves M <= 4, and M <= 8 where the small-M kernel is switched off (knob 19)
        _check(y, ref, bud, M <= (8 if staged else 4), f"pdl={pdl} staged={staged} M={M} N={y.shape[1]}")
    assert _workspace_clean(ext), "split-K workspace not restored"


@pytest.mark.parametrize("M", CHAINS)
@pytest.mark.parametrize("pdl", [0, 1], ids=["plain", "pdl"])
def test_dependent_chain_in_graph(pdl, M):
    from autoawq_b200 import ext

    dev = torch.device("cuda:0")
    c1, c2 = O.make_case(1024, 2048, G, seed=11), O.make_case(2048, 512, G, seed=12)
    w1 = O.dequantize_gemm(c1["qweight"], c1["qzeros"], c1["scales"], G)
    w2 = O.dequantize_gemm(c2["qweight"], c2["qzeros"], c2["scales"], G)
    x = np.random.default_rng(M).standard_normal((M, 1024)).astype(np.float16)
    xt = _t(x, dev)
    a1 = [_t(c1[k], dev) for k in ("qweight", "scales", "qzeros")]
    a2 = [_t(c2[k], dev) for k in ("qweight", "scales", "qzeros")]
    h = torch.empty((M, 2048), dtype=torch.float16, device=dev)
    y = torch.empty((M, 512), dtype=torch.float16, device=dev)

    def run():
        h.zero_()                 # a second linear that reads h too early sees zeros or partial sums
        ext.linear_forward("gemm", xt, *a1, G, out=h)
        ext.linear_forward("gemm", h, *a2, G, out=y)

    ext.set_knob(4, pdl)
    try:
        g = _graph(torch.cuda.Stream(), run)
        y.zero_()
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    finally:
        ext.set_knob(4, 0)
    _check(h, O.gemm_f64(x, w1), np.abs(x.astype(np.float64)) @ np.abs(w1.astype(np.float64)), M <= 4, f"pdl={pdl} first")
    hn = h.cpu().numpy()      # the second linear's reference is built from what the first one left behind
    _check(y, O.gemm_f64(hn, w2), np.abs(hn.astype(np.float64)) @ np.abs(w2.astype(np.float64)), M <= 4, f"pdl={pdl} second")
    assert _workspace_clean(ext), "split-K workspace not restored"
