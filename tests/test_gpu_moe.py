"""GPU parity tests of the MoE operators (awq_ext.topk_softmax / moe_alig_block_size / grouped_gemm_forward,
awq/modules/fused/moe.py:45-171) against the CPU oracle, through the awq_ext surface (C ABI underneath).
The reference pins none of these (kernels live in the un-vendored autoawq-kernels package); the oracle restates the
contract of the call sites, and the moe_align case below is the worked example of the reference's own docstring."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import llm_data as L

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


@pytest.fixture(scope="module")
def awq_ext():
    import awq_ext as m

    return m


def test_topk_softmax(awq_ext):
    rng = np.random.default_rng(0)
    for M, E, topk in [(1, 8, 2), (7, 8, 2), (33, 64, 6), (5, 160, 8)]:
        g = rng.standard_normal((M, E)).astype(np.float32) * 3
        g[0, :3] = g[0, 3]  # a four-way tie: lowest index wins
        w = torch.empty((M, topk), dtype=torch.float32, device=_dev())
        ids = torch.empty((M, topk), dtype=torch.int32, device=_dev())
        src = torch.empty((M, topk), dtype=torch.int32, device=_dev())
        awq_ext.topk_softmax(w, ids, src, _t(g))
        rw, rids, rsrc = O.topk_softmax(g, topk)
        assert np.array_equal(ids.cpu().numpy(), rids), (M, E, topk)
        assert np.array_equal(src.cpu().numpy(), rsrc)
        np.testing.assert_allclose(w.cpu().numpy(), rw, rtol=2e-6, atol=1e-7)


def _align(awq_ext, ids, block, E):
    numel = ids.size
    sorted_ids = torch.full((numel + E * (block - 1),), numel, dtype=torch.int32, device=_dev())
    expert_ids = torch.full((numel + E,), -1, dtype=torch.int32, device=_dev())
    npost = torch.zeros(1, dtype=torch.int32, device=_dev())
    awq_ext.moe_alig_block_size(_t(ids.astype(np.int32)), E, block, sorted_ids, expert_ids, npost)
    return sorted_ids, expert_ids, npost


def test_moe_align_reference_docstring_example(awq_ext):
    """moe.py:104-113: topk_ids [[2,3,4],[1,2,4],[1,3,4],[1,2,3]], block 4 ->
    [3,6,9,12, 0,4,10,12, 1,7,11,12, 2,5,8,12]."""
    ids = np.array([[2, 3, 4], [1, 2, 4], [1, 3, 4], [1, 2, 3]])
    s, e, n = _align(awq_ext, ids, 4, 5)
    assert int(n.item()) == 16
    assert s[:16].cpu().tolist() == [3, 6, 9, 12, 0, 4, 10, 12, 1, 7, 11, 12, 2, 5, 8, 12]
    assert e[:4].cpu().tolist() == [1, 2, 3, 4]


def test_moe_align_random(awq_ext):
    rng = np.random.default_rng(1)
    for T, topk, E, block in [(1, 2, 8, 16), (5, 2, 8, 16), (300, 2, 8, 16), (64, 6, 64, 16), (3, 1, 4, 8)]:
        ids = np.stack([rng.permutation(E)[:topk] for _ in range(T)])
        s, e, n = _align(awq_ext, ids, block, E)
        rs, re_, rn = O.moe_align_block_size(ids, block, E)
        assert int(n.item()) == rn
        assert np.array_equal(s.cpu().numpy()[:rn], rs[:rn])
        assert np.array_equal(e.cpu().numpy()[: rn // block], re_[: rn // block])


def _experts(E, K, N, G, seed):
    qw, qz, sc, w = [], [], [], []
    for e in range(E):
        c = O.make_case(K, N, G, seed=seed + e)
        s = (c["scales"].astype(np.float32) * (1.0 / (6.1 * 0.0108 * np.sqrt(K)))).astype(np.float16)
        qw.append(c["qweight"])
        qz.append(c["qzeros"])
        sc.append(s)
        w.append(O.dequantize_gemm(c["qweight"], c["qzeros"], s, G))
    return np.stack(qw), np.stack(qz), np.stack(sc), np.stack(w)


@pytest.mark.parametrize("T,topk,E,K,N,G,kernel", [
    (1, 2, 8, 1024, 512, 128, "ring"), (5, 2, 8, 1024, 512, 128, "ring"), (37, 2, 4, 512, 256, 64, "ring"),
    (2, 2, 8, 1024, 512, 128, "ring"), (3, 2, 8, 1024, 512, 128, "ring"),   # the 2- and 4-slot variants of the ring kernel
    (3, 3, 6, 1536, 96, 128, "staged"),            # N not a multiple of 256: the register-staged kernel
    (5, 2, 8, 1024, 512, 128, "staged-forced"),    # knob 12 = 2
])
def test_grouped_gemm_and_full_moe_block(awq_ext, T, topk, E, K, N, G, kernel):
    from autoawq_b200 import ext

    ext.set_knob(12, 2 if kernel == "staged-forced" else 0)
    try:
        _moe_block(awq_ext, T, topk, E, K, N, G, _moe_family(T, topk, E))
    finally:
        ext.set_knob(12, 0)
    for ws in ext._WS.values():
        assert int(ws.count_nonzero()) == 0, "grouped GEMM left the shared workspace dirty"


def _moe_family(T, topk, E):
    """cabi.cu:482-513: moe_tc_kernel from 20 slots per expert (exact-dequant), the ring / register-staged GEMVs below
    (offset-fold)."""
    return "exact-dequant" if T * topk >= 20 * E else "offset-fold"


def _check_slots(y, ref, x_of, w, sc, tids, tw, family, what):
    """Every (token, slot) row of y against the oracle's ref = x_of(t, k) . W[expert] (* tw) under the family's error
    model."""
    T, topk = tids.shape
    G = w.shape[1] // sc.shape[1]
    for t in range(T):
        for k in range(topk):
            e = int(tids[t, k])
            wgt = 1.0 if tw is None else float(tw[t, k])
            case = dict(w=w[e].astype(np.float64) * wgt, scales=sc[e].astype(np.float64) * wgt, group_size=G, bias=None)
            L.check_forward(y[t, k][None, :], x_of(t, k)[None, :], case, family, f"{what} token {t} slot {k}",
                            y64=ref[t, k][None, :])


def _moe_block(awq_ext, T, topk, E, K, N, G, family):
    """apply_moe_weights (moe.py:45-89) end to end: route, align, gate|up grouped GEMM, silu*mul, down grouped GEMM
    with the routing weights, sum over the top-k - every stage against the oracle on the GPU's own inputs."""
    rng = np.random.default_rng(T * 100 + E)
    qw1, qz1, sc1, w1 = _experts(E, K, 2 * N, G, seed=10)      # gate|up: K -> 2N
    x = rng.standard_normal((T, K)).astype(np.float16)
    gating = rng.standard_normal((T, E)).astype(np.float32)
    tw = torch.empty((T, topk), dtype=torch.float32, device=_dev())
    tid = torch.empty((T, topk), dtype=torch.int32, device=_dev())
    src = torch.empty((T, topk), dtype=torch.int32, device=_dev())
    awq_ext.topk_softmax(tw, tid, src, _t(gating))
    tw = tw / tw.sum(dim=-1, keepdim=True)                      # fused_topk renormalize=True (moe.py:169-170)
    s_ids, e_ids, npost = _align(awq_ext, tid.cpu().numpy(), 16, E)
    xt = _t(x).view(T, 1, K)
    gu = awq_ext.grouped_gemm_forward(xt, _t(qw1), _t(sc1), _t(qz1), tw, s_ids, e_ids, npost, False, 8)
    assert gu.shape == (T, topk, 2 * N) and gu.dtype == torch.float16
    ref = O.grouped_gemm_f64(x.reshape(T, 1, K), w1, tw.cpu().numpy(), s_ids.cpu().numpy(), e_ids.cpu().numpy(),
                             int(npost.item()), False)
    tids = tid.cpu().numpy()
    gun = gu.cpu().numpy()
    _check_slots(gun, ref, lambda t, k: x[t], w1, sc1, tids, None, family, "gate|up grouped GEMM")

    # second GEMM: per-slot inputs [T, topk, N'] with the routing weight multiplied in, N' must be a multiple of 512
    if N % 512 == 0:
        act = torch.empty((T, topk, N), dtype=torch.float16, device=_dev())
        awq_ext.silu_and_mul(act, gu)
        qw2, qz2, sc2, w2 = _experts(E, N, K, G, seed=90)
        out = awq_ext.grouped_gemm_forward(act, _t(qw2), _t(sc2), _t(qz2), tw, s_ids, e_ids, npost, True, 8)
        a = act.cpu().numpy()
        ref2 = O.grouped_gemm_f64(a, w2, tw.cpu().numpy(), s_ids.cpu().numpy(), e_ids.cpu().numpy(), int(npost.item()),
                                  True)
        outn = out.cpu().numpy()
        _check_slots(outn, ref2, lambda t, k: a[t, k], w2, sc2, tids, tw.cpu().numpy(), family, "down grouped GEMM")
        final = torch.sum(out, dim=1)                           # moe.py:89
        assert final.shape == (T, K)
