"""Per-op kernels against the ORACLE (not against themselves) at every (K, N) of BASELINE configs 2 and 5:

  Llama-3-8B (config 2/3):       qkv 4096x6144, o 4096x4096, gate|up 4096x28672, down 14336x4096
  Llama-3-70B / 8 ranks (cfg 5): qkv 8192x1280, o 1024x8192, gate|up 8192x7168,  down 3584x8192

x M in {1, 2, 4, 8, 16, 64, 300} (GEMV kernels, the small-batch kernel, the wgmma kernel) in all three
checkpoint layouts (GEMM / GEMV / GEMVFast), through the awq_ext / awq_v2_ext operator surface.  The oracle is
the fp64 contraction of the bit-exact dequantised weights, evaluated on a strided sample of output columns
(every 61st + the edges: the full product at M = 300 on 4096x28672 would be 70 GFLOP of fp64 per case; each
column is an independent dot product, so a column sample checks the same arithmetic); each route held to
oracle/llm_data.forward_tolerance of the kernel family that ran (oracle/llm_data.*_route_family).
"""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import llm_data as L

pytestmark = pytest.mark.gpu
SHAPES = [
    ("8b.qkv", 4096, 6144), ("8b.o", 4096, 4096), ("8b.gate_up", 4096, 28672), ("8b.down", 14336, 4096),
    ("70b8.qkv", 8192, 1280), ("70b8.o", 1024, 8192), ("70b8.gate_up", 8192, 7168), ("70b8.down", 3584, 8192),
]
MS = [1, 2, 4, 8, 16, 64, 300]
G = 128


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _check(y, x, w, scales, cols, family, what):
    case = dict(w=w[:, cols], scales=np.asarray(scales)[:, cols], group_size=G, bias=None)
    L.check_forward(np.asarray(y)[:, cols], x, case, family, what)


@pytest.fixture(scope="module")
def ext():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext as e

    return e


@pytest.mark.parametrize("name,K,N", SHAPES)
def test_all_layouts_all_m_vs_oracle(ext, name, K, N):
    import awq_ext
    import awq_v2_ext

    c = O.make_case(K, N, G, seed=K % 97 + N % 89)
    # keep the outputs O(1): scales ~ 1 / (6.1 sqrt(K)) (same conditioning as bench.py)
    s = (c["scales"].astype(np.float32) / (6.1 * 0.0108 * np.sqrt(K))).astype(np.float16)
    w = O.dequantize_gemm(c["qweight"], c["qzeros"], s, G)
    cols = np.unique(np.concatenate([np.arange(0, N, 61), [0, 1, 7, 8, 255, 256, N - 9, N - 8, N - 1]]))
    vw, vz, vs = O.pack_gemv(c["intweight"], c["zeros"], s, G)
    fw, fs, fz = O.pack_gemv_fast(c["intweight"], c["zeros"], s, G)
    wfast = O.dequantize_gemv_fast_f64(fw, fs, fz, G)
    qw, qz, sc = _t(c["qweight"]), _t(c["qzeros"]), _t(s)
    tvw, tvz, tvs = _t(vw), _t(vz), _t(vs)
    tfw, tfs, tfz = _t(fw), _t(fs), _t(fz)
    rng = np.random.default_rng(K + N)
    for M in MS:
        x = rng.standard_normal((M, K)).astype(np.float16)
        xt = _t(x)
        y = awq_ext.gemm_forward_cuda(xt, qw, sc, qz, 8)
        assert tuple(y.shape) == (M, N)
        _check(y.cpu().numpy(), x, w, s, cols, L.gemm_route_family(M, K, N, G), f"{name} gemm layout M={M}")
        if M > 8:
            yv = awq_ext.gemmv2_forward_cuda(xt, tvw, tvs, tvz, G, 8)
            yf = awq_v2_ext.gemm_forward_cuda_prefill(xt.unsqueeze(0), tfw, tfs, tfz)[0]
        else:
            yv = awq_ext.gemv_forward_cuda(xt, tvw, tvs, tvz, G)
            yf = awq_v2_ext.gemv_forward_cuda_decode(xt.unsqueeze(1), tfw, tfs, tfz, M, N, K, G)[:, 0]
        _check(yv.cpu().numpy(), x, w, s, cols, L.gemv_route_family(M, K), f"{name} gemv layout M={M}")
        _check(yf.cpu().numpy(), x, wfast, fs, cols, L.fast_route_family(M), f"{name} fast layout M={M}")
    # dequant at this shape, bit-exact on the sampled columns and on a full-row digest
    wd = awq_ext.dequantize_weights_cuda(qw, sc, qz, 0, 0, 0, False).cpu().numpy()
    assert np.array_equal(wd.view(np.uint16), w.view(np.uint16)), f"{name}: dequant not bit-exact"
