"""GPU tests of the grouped tensor-core kernel (moe_tc_kernel): grouped_gemm_forward at prefill-sized token counts.
The kernel is forced with knob 12 = 3 (and reached through the default routing where the shape is large enough), held to
the fp64 oracle with the tolerance of tests/test_gpu_moe.py, to the register-staged kernel (knob 12 = 2) bit for bit on
exact-arithmetic data, and checked for what it must NOT do: write rows of slots that are not listed, touch memory
around y, dirty the shared workspace, or depend on routing that was current when a CUDA graph was captured."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import exact_probe as XP

pytestmark = pytest.mark.gpu

RTOL = 2.0**-10
WR = 2.0**-11
BLOCK = 16            # the block size awq_ext.grouped_gemm_forward aligns to (moe.py:54-56)
STAGED, FORCED = 2, 3


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


@pytest.fixture(scope="module")
def awq_ext():
    import awq_ext as m

    return m


@pytest.fixture()
def knob12():
    from autoawq_b200 import ext

    yield lambda v: ext.set_knob(12, v)
    ext.set_knob(12, 0)


def _experts(E, K, N, G, seed):
    qw, qz, sc, w = [], [], [], []
    for e in range(E):
        c = O.make_case(K, N, G, seed=seed + e)
        s = (c["scales"].astype(np.float32) * (1.0 / (6.1 * 0.0108 * np.sqrt(K)))).astype(np.float16)
        qw.append(c["qweight"])
        qz.append(c["qzeros"])
        sc.append(s)
        w.append(O.dequantize_gemm(c["qweight"], c["qzeros"], s, c["group_size"]))
    return np.stack(qw), np.stack(qz), np.stack(sc), np.stack(w)


def _random_routing(rng, T, topk, E):
    return np.stack([rng.permutation(E)[:topk] for _ in range(T)]).astype(np.int32)


def _tables(tids, E):
    """Aligned routing tables of topk_ids [T, topk] (the oracle's moe_align_block_size), on the device."""
    s, e, n = O.moe_align_block_size(tids, BLOCK, E)
    return _t(s), _t(e), _t(np.array([n], dtype=np.int32)), (s, e, n)


def _weights_like(rng, T, topk):
    w = rng.random((T, topk)).astype(np.float32) + 0.1
    return (w / w.sum(axis=1, keepdims=True)).astype(np.float32)


def _budget(x_rows, w, tids, scale=None):
    """|x| . |W[expert]| per slot, [T, topk, N] float64; x_rows [T, topk or 1, K]."""
    T, topk = tids.shape
    out = np.empty((T, topk, w.shape[-1]), dtype=np.float64)
    for e in np.unique(tids):
        t, k = np.nonzero(tids == e)
        rows = np.abs(x_rows[t, k if x_rows.shape[1] != 1 else 0].astype(np.float64))
        out[t, k] = rows @ np.abs(w[e].astype(np.float64))
    return out if scale is None else out * scale[..., None]


def _moe_block(awq_ext, set_knob, modes, tids, E, K, N, G, seed=0):
    """apply_moe_weights (moe.py:45-89) from the aligned tables on: gate|up grouped GEMM (x [T, 1, K], no routing
    weight), silu*mul, down grouped GEMM (x [T, topk, N], routing weight multiplied in) - each against the fp64 oracle
    on the GPU's own inputs, once per knob 12 value in `modes`; all modes that run the same kernel must agree exactly."""
    T, topk = tids.shape
    rng = np.random.default_rng(seed + T * 100 + E)
    qw1, qz1, sc1, w1 = _experts(E, K, 2 * N, G, seed=10)
    x = rng.standard_normal((T, K)).astype(np.float16)
    tw = _weights_like(rng, T, topk)
    s_ids, e_ids, npost, (hs, he, hn) = _tables(tids, E)
    d_qw1, d_sc1, d_qz1, d_tw, xt = _t(qw1), _t(sc1), _t(qz1), _t(tw), _t(x).view(T, 1, K)
    ref = O.grouped_gemm_f64(x.reshape(T, 1, K), w1, tw, hs, he, hn, False)
    budget = _budget(x.reshape(T, 1, K), w1, tids)
    outs = []
    for mode in modes:
        set_knob(mode)
        gu = awq_ext.grouped_gemm_forward(xt, d_qw1, d_sc1, d_qz1, d_tw, s_ids, e_ids, npost, False, 8)
        assert gu.shape == (T, topk, 2 * N) and gu.dtype == torch.float16
        err = np.abs(gu.float().cpu().numpy().astype(np.float64) - ref)
        assert (err <= RTOL * np.abs(ref) + WR * budget + 1e-6).all(), f"gate|up, knob 12 = {mode}: max err {err.max():.3e}"
        outs.append(gu)
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), "forced and default routing ran different kernels"
    if N % 64 != 0:
        return
    act = torch.empty((T, topk, N), dtype=torch.float16, device=_dev())
    awq_ext.silu_and_mul(act, outs[0])
    qw2, qz2, sc2, w2 = _experts(E, N, K, G, seed=90)
    d_qw2, d_sc2, d_qz2 = _t(qw2), _t(sc2), _t(qz2)
    a = act.cpu().numpy()
    ref2 = O.grouped_gemm_f64(a, w2, tw, hs, he, hn, True)
    budget2 = _budget(a, w2, tids, scale=tw.astype(np.float64))
    outs = []
    for mode in modes:
        set_knob(mode)
        out = awq_ext.grouped_gemm_forward(act, d_qw2, d_sc2, d_qz2, d_tw, s_ids, e_ids, npost, True, 8)
        err2 = np.abs(out.float().cpu().numpy().astype(np.float64) - ref2)
        assert (err2 <= 2 * RTOL * np.abs(ref2) + WR * budget2 + 1e-6).all(), f"down, knob 12 = {mode}: max err {err2.max():.3e}"
        outs.append(out)
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), "forced and default routing ran different kernels"


def _workspace_clean():
    from autoawq_b200 import ext

    for ws in ext._WS.values():
        assert int(ws.count_nonzero()) == 0, "grouped GEMM left the shared workspace dirty"


@pytest.mark.parametrize("T,topk,E,K,N,G,default_too", [
    (64, 2, 8, 1024, 512, 128, False),       # 16 slots per expert: token tile 32, below the default routing's threshold
    (300, 2, 8, 1024, 512, 128, True),       # 75 per expert: token tile 64
    (1024, 2, 8, 1024, 1024, 64, True),      # 256 per expert: token tile 128, G = 64
    (257, 6, 64, 512, 256, 128, True),       # DeepSeek-style fan-out: 64 experts, top-6
    (96, 3, 6, 1536, 96, 128, True),         # gate|up N = 192: the second column tile is half empty
    (200, 2, 4, 512, 256, 32, True),         # G = 32: two quantisation groups per k-step
    (130, 2, 4, 512, 128, -1, True),         # one group per column (G = K)
])
def test_block_against_oracle(awq_ext, knob12, T, topk, E, K, N, G, default_too):
    rng = np.random.default_rng(T + E)
    assert (T * topk >= 20 * E) == default_too
    _moe_block(awq_ext, knob12, [FORCED, 0] if default_too else [FORCED], _random_routing(rng, T, topk, E), E, K, N, G)
    _workspace_clean()


@pytest.mark.parametrize("kind", ["one-expert", "empty-expert", "bt-plus-one", "single-slots"])
def test_skewed_routing(awq_ext, knob12, kind):
    E, K, N, G = 8, 512, 256, 128
    if kind == "one-expert":                 # every token on expert 5: one run of 300 slots
        tids = np.full((300, 1), 5, dtype=np.int32)
    elif kind == "empty-expert":             # experts 2 and 7 get nothing
        rng = np.random.default_rng(3)
        tids = np.array([0, 1, 3, 4, 5, 6], dtype=np.int32)[_random_routing(rng, 200, 2, 6)]
    elif kind == "bt-plus-one":              # 776 slots over 8 experts pick the 128 tile; runs of 129, 65 and 33
        tids = np.concatenate([np.full(129, 1), np.full(65, 2), np.full(33, 4), np.full(549, 6)]).astype(np.int32)
        tids = tids.reshape(-1, 1)
    else:                                    # every expert has exactly one slot: 8 tiles of one real row each
        tids = np.arange(8, dtype=np.int32).reshape(4, 2)
    _moe_block(awq_ext, knob12, [FORCED], tids, E, K, N, G, seed=7)
    _workspace_clean()


def test_only_rows_of_listed_slots_are_written(knob12):
    """Through the C ABI, y inside a larger buffer pre-filled with a sentinel: rows of listed slots are fully written,
    rows of slots the tables do not list (an expert id outside 0..E-1 never enters sorted_ids) and the guard rows on
    both sides keep the sentinel."""
    from autoawq_b200 import _cabi

    T, topk, E, K, N, G = 150, 2, 8, 512, 192, 128
    rng = np.random.default_rng(5)
    tids = _random_routing(rng, T, topk, E)
    unlisted = rng.random((T, topk)) < 0.1
    tids[unlisted] = E
    qw, qz, sc, w = _experts(E, K, N, G, seed=40)
    x = rng.standard_normal((T, K)).astype(np.float16)
    tw = _weights_like(rng, T, topk)
    s_ids, e_ids, npost, (hs, he, hn) = _tables(tids, E)
    guard = 64
    sentinel = 0x7BFF                        # 65504.0: no output comes near it
    buf = torch.full(((T * topk + 2 * guard) * N,), sentinel, dtype=torch.int16, device=_dev())
    y = buf[guard * N:(guard + T * topk) * N]
    d = [_t(a) for a in (x, qw, sc, qz, tw)]
    knob12(FORCED)
    rc = _cabi.lib.b200awq_grouped_gemm_forward(
        d[0].data_ptr(), 1, d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), s_ids.data_ptr(),
        e_ids.data_ptr(), npost.data_ptr(), y.data_ptr(), T, topk, s_ids.numel(), E, K, N, G, 1, BLOCK, None, 0,
        torch.cuda.current_stream().cuda_stream)
    _cabi.check(rc, "grouped_gemm_forward")
    torch.cuda.synchronize()
    got = buf.cpu().numpy().view(np.uint16).reshape(-1, N)
    assert (got[:guard] == sentinel).all() and (got[guard + T * topk:] == sentinel).all(), "wrote outside y"
    rows = got[guard:guard + T * topk]
    flat_unlisted = unlisted.reshape(-1)
    assert (rows[flat_unlisted] == sentinel).all(), "wrote the row of a slot that is not listed"
    assert (rows[~flat_unlisted] != sentinel).all(), "a listed slot's row is not fully written"
    ref = O.grouped_gemm_f64(x.reshape(T, 1, K), w, tw, hs, he, hn, True).reshape(-1, N)
    vals = rows.view(np.float16).astype(np.float64)
    budget = _budget(x.reshape(T, 1, K), w, np.where(unlisted, 0, tids), scale=tw.astype(np.float64)).reshape(-1, N)
    err = np.abs(vals - ref)[~flat_unlisted]
    assert (err <= 2 * RTOL * np.abs(ref[~flat_unlisted]) + WR * budget[~flat_unlisted] + 1e-6).all()


@pytest.mark.parametrize("T,topk,E,K,N,G,per_slot", [(200, 2, 8, 1024, 512, 128, False), (96, 4, 4, 512, 384, 64, True)])
def test_exact_arithmetic_equals_the_staged_kernel_bit_for_bit(awq_ext, knob12, T, topk, E, K, N, G, per_slot):
    """Integer-valued probes: every summation order is exact, so the wgmma kernel, the register-staged kernel and the
    integer contraction must agree on every bit of every element."""
    rows = T * topk if per_slot else T
    cases = [XP.make_exact_case(K, N, G, rows, seed=300 + e, layouts=("gemm",), reference=False) for e in range(E)]
    x_units = cases[0]["x_units"]
    unit = cases[0]["unit"]
    rng = np.random.default_rng(11)
    tids = _random_routing(rng, T, topk, E)
    s_ids, e_ids, npost, _ = _tables(tids, E)
    x = _t(cases[0]["x"]).view(T, topk if per_slot else 1, K)
    qw, sc, qz = (_t(np.stack([c[k] for c in cases])) for k in ("qweight", "scales", "qzeros"))
    tw = _t(_weights_like(rng, T, topk))
    out = {}
    for mode in (FORCED, STAGED):
        knob12(mode)
        out[mode] = awq_ext.grouped_gemm_forward(x, qw, sc, qz, tw, s_ids, e_ids, npost, False, 8)
    exact = np.empty((T, topk, N), dtype=np.float64)
    xr = x_units.reshape(T, -1, K)
    for e in range(E):
        t, k = np.nonzero(tids == e)
        exact[t, k] = XP.contract_units(xr[t, k if per_slot else 0], cases[e]["w_units"]) * unit
    got = out[FORCED].cpu().numpy().reshape(-1, N)
    want = exact.astype(np.float16).reshape(-1, N)
    assert np.array_equal(got, want), XP.mismatch_report(got, want, unit)
    assert torch.equal(out[FORCED], out[STAGED]), "the wgmma and the register-staged kernel differ on exact data"


def test_mixtral_shaped_call_matches_the_staged_kernel(awq_ext, knob12):
    """Mixtral-8x7B gate|up (4096 -> 28672, g128, 8 experts, top-2) at 512 tokens, default routing (128 slots per
    expert: the wgmma kernel) against the register-staged kernel.  The fp64 oracle at this size is too slow to
    build on the host, so the weights are raw random words generated on the device."""
    from autoawq_b200 import ext

    T, topk, E, K, N, G = 512, 2, 8, 4096, 28672, 128
    gen = torch.Generator(device=_dev()).manual_seed(1)
    qw = torch.randint(-2**31, 2**31 - 1, (E, K, N // 8), dtype=torch.int64, device=_dev(), generator=gen).to(torch.int32)
    qz = torch.randint(-2**31, 2**31 - 1, (E, K // G, N // 8), dtype=torch.int64, device=_dev(), generator=gen).to(torch.int32)
    sc = (torch.rand((E, K // G, N), device=_dev(), generator=gen) * 0.01 + 1e-3).to(torch.float16)
    x = (torch.randn((T, 1, K), device=_dev(), generator=gen) / K ** 0.5).to(torch.float16)
    rng = np.random.default_rng(2)
    tids = _random_routing(rng, T, topk, E)
    s_ids, e_ids, npost, _ = _tables(tids, E)
    tw = _t(_weights_like(rng, T, topk))
    knob12(0)
    y_new = awq_ext.grouped_gemm_forward(x, qw, sc, qz, tw, s_ids, e_ids, npost, True, 8)
    knob12(FORCED)
    assert torch.equal(y_new, awq_ext.grouped_gemm_forward(x, qw, sc, qz, tw, s_ids, e_ids, npost, True, 8))
    knob12(STAGED)
    y_old = awq_ext.grouped_gemm_forward(x, qw, sc, qz, tw, s_ids, e_ids, npost, True, 8)
    # budget |x| . |W| * w per slot from the dequantised experts, fp32 on the device
    d_tids = _t(tids)
    for e in range(E):
        w_abs = ext.dequantize_weights_cuda(qw[e], sc[e], qz[e]).abs().float()
        t, k = torch.nonzero(d_tids == e, as_tuple=True)
        budget = (x[t, 0].abs().float() @ w_abs) * tw[t, k][:, None]
        a, b = y_new[t, k].float(), y_old[t, k].float()
        assert bool(((a - b).abs() <= 2 * RTOL * b.abs() + 2 * WR * budget + 1e-6).all()), f"expert {e}"
    _workspace_clean()


def test_cuda_graph_replay_follows_rewritten_routing(awq_ext, knob12):
    """One captured call; the routing tables, routing weights and activations are rewritten in place before the
    replay: the kernel builds its tile list on the device, so the replay must equal an eager call on the new routing
    (which moves every expert's run and leaves one expert empty)."""
    T, topk, E, K, N, G = 160, 2, 8, 512, 256, 128
    qw, qz, sc, _ = _experts(E, K, N, G, seed=60)
    d_qw, d_sc, d_qz = _t(qw), _t(sc), _t(qz)
    rng = np.random.default_rng(9)
    tids_a = _random_routing(rng, T, topk, E)
    tids_b = np.array([0, 1, 2, 4, 5, 6, 7], dtype=np.int32)[_random_routing(rng, T, topk, 7)]   # expert 3 unused
    x = torch.randn((T, 1, K), device=_dev()).to(torch.float16)
    s_ids, e_ids, npost, _ = _tables(tids_a, E)
    tw = _t(_weights_like(rng, T, topk))
    knob12(FORCED)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        awq_ext.grouped_gemm_forward(x, d_qw, d_sc, d_qz, tw, s_ids, e_ids, npost, True, 8)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        y_g = awq_ext.grouped_gemm_forward(x, d_qw, d_sc, d_qz, tw, s_ids, e_ids, npost, True, 8)
    g.replay()
    torch.cuda.synchronize()
    y_a = y_g.clone()
    assert torch.equal(y_a, awq_ext.grouped_gemm_forward(x, d_qw, d_sc, d_qz, tw, s_ids, e_ids, npost, True, 8))
    s_b, e_b, n_b, _ = _tables(tids_b, E)
    s_ids.copy_(s_b)
    e_ids.copy_(e_b)
    npost.copy_(n_b)
    tw.copy_(_t(_weights_like(rng, T, topk)))
    x.copy_(torch.randn((T, 1, K), device=_dev()).to(torch.float16))
    g.replay()
    torch.cuda.synchronize()
    y_b = awq_ext.grouped_gemm_forward(x, d_qw, d_sc, d_qz, tw, s_ids, e_ids, npost, True, 8)
    assert torch.equal(y_g, y_b), "the replay did not follow the rewritten routing"
    assert not torch.equal(y_a, y_b)
    _workspace_clean()
