"""GPU tests of the decode-program kernel (csrc/program.cu) through the C ABI (b200awq_program_*): every buffer a
program run leaves behind is checked, op by op, against the CPU oracle applied to the op's ACTUAL input (the
buffer the previous op left on the GPU) - so each recorded op is held to the same bar as the stand-alone entry
points (tests/test_gpu_parity.py) - and against the per-op path run on the same inputs."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O

pytestmark = pytest.mark.gpu

RTOL = 2.0**-10
WR_GEMV = 2.0**-11
EPS = 1e-5


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _close(y, ref64, budget, what):
    y = np.asarray(y, dtype=np.float64)
    tol = RTOL * np.abs(ref64) + WR_GEMV * budget + 1e-6
    bad = np.abs(y - ref64) > tol
    assert not bad.any(), f"{what}: {bad.sum()} / {bad.size} outside tolerance, max err {np.abs(y - ref64).max():.3e}"


class Block:
    """One Llama-style block's quantised linears (random AWQ-packed weights) + its call sequence."""

    def __init__(self, hidden, inter, qkv_out, G, seed):
        self.hidden, self.inter, self.G = hidden, inter, G
        shapes = dict(qkv=(hidden, qkv_out), o=(hidden, hidden), gate_up=(hidden, 2 * inter), down=(inter, hidden))
        self.np, self.w = {}, {}
        rng = np.random.default_rng(seed)
        for i, (name, (K, N)) in enumerate(shapes.items()):
            c = O.make_case(K, N, G, seed=seed * 10 + i)
            # scales sized so activations stay O(1) along the chain
            sc = (c["scales"].astype(np.float32) * (1.0 / (6.1 * 0.0108 * np.sqrt(K)))).astype(np.float16)
            self.np[name] = dict(qweight=c["qweight"], qzeros=c["qzeros"], scales=sc,
                                 w=O.dequantize_gemm(c["qweight"], c["qzeros"], sc, G))
            self.w[name] = (_t(c["qweight"]), _t(sc), _t(c["qzeros"]))
        self.norm1 = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
        self.norm2 = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
        self.norm1_t, self.norm2_t = _t(self.norm1), _t(self.norm2)


def _record(api, blocks, h, M):
    """The bench's / fused block's call sequence against `api` (awq_ext-like).  Returns every buffer by name."""
    bufs = []
    for b in blocks:
        xn = torch.empty((M, b.hidden), dtype=torch.float16, device=_dev())
        api.layernorm_forward_cuda(h, b.norm1_t, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *b.w["qkv"], 8)
        o = api.gemm_forward_cuda(qkv[:, : b.hidden], *b.w["o"], 8)
        xn2 = torch.empty((M, b.hidden), dtype=torch.float16, device=_dev())
        api.layernorm_forward_cuda(o, b.norm2_t, xn2, EPS)
        gu = api.gemm_forward_cuda(xn2, *b.w["gate_up"], 8)
        act = torch.empty((M, b.inter), dtype=torch.float16, device=_dev())
        api.silu_and_mul(act, gu)
        down = api.gemm_forward_cuda(act, *b.w["down"], 8)
        bufs.append(dict(h=h, xn=xn, qkv=qkv, o=o, xn2=xn2, gu=gu, act=act, down=down))
        h = down
    return bufs


def _no_abort(tag=""):
    from autoawq_b200.program import DecodeProgram

    rec = DecodeProgram.abort_record()
    assert rec[3] == 0, f"{tag}: program kernel gave up waiting: code={rec[0]} op={rec[1]} cta={rec[2]}"


def _check_against_oracle(blocks, bufs, tag):
    _no_abort(tag)
    for li, (b, t) in enumerate(zip(blocks, bufs)):
        v = {k: x.float().cpu().numpy().astype(np.float16) for k, x in t.items()}
        np.testing.assert_allclose(v["xn"], O.rmsnorm_f64(v["h"], b.norm1, EPS), rtol=2e-3, atol=2e-3,
                                   err_msg=f"{tag} L{li} norm1")
        np.testing.assert_allclose(v["xn2"], O.rmsnorm_f64(v["o"], b.norm2, EPS), rtol=2e-3, atol=2e-3,
                                   err_msg=f"{tag} L{li} norm2")
        g64 = v["gu"][:, : b.inter].astype(np.float64)
        np.testing.assert_allclose(v["act"], g64 / (1 + np.exp(-g64)) * v["gu"][:, b.inter:].astype(np.float64),
                                   rtol=2e-3, atol=2e-3, err_msg=f"{tag} L{li} silu")
        for name, xin, yout in [("qkv", v["xn"], v["qkv"]), ("o", v["qkv"][:, : b.hidden], v["o"]),
                                ("gate_up", v["xn2"], v["gu"]), ("down", v["act"], v["down"])]:
            w = b.np[name]["w"]
            budget = np.abs(xin.astype(np.float64)) @ np.abs(w.astype(np.float64))
            _close(yout, O.gemm_f64(xin, w), budget, f"{tag} L{li} {name}")


@pytest.fixture(scope="module")
def api():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext

    return ext


@pytest.fixture(scope="module")
def small_blocks():
    return [Block(2048, 4096, 3072, 128, seed=s) for s in (1, 2)]


@pytest.fixture(params=["stream"])
def kind(request, api):
    """The kind a fused program reports: the stream kernel (one-time re-layout, csrc/program_stream.cuh)."""
    return request.param


def _h0(hidden, M, seed=0):
    return _t(np.random.default_rng(seed).standard_normal((M, hidden)).astype(np.float16))


def test_program_matches_oracle_op_by_op(api, small_blocks, kind):
    from autoawq_b200.program import DecodeProgram

    h = _h0(2048, 1)
    prog = DecodeProgram()
    bufs = _record(prog, small_blocks, h, 1)
    prog.build()
    assert prog.fused and prog.kernel_ops == 8 and prog.launches_per_run == 1 and prog.kind == kind
    prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, bufs, "program")
    # the per-op path on the same inputs: same arithmetic up to fp32 summation order
    ref = _record(api, small_blocks, h, 1)
    # (loose: the two paths add their fp32 partial sums in different orders, and the difference of one fp16 ulp
    # propagates down the chain; the op-by-op oracle check above is the parity gate)
    for a, b in zip(bufs, ref):
        for k in a:
            assert torch.allclose(a[k].float(), b[k].float(), rtol=3e-2, atol=3e-2), k
    # identical input -> the rmsnorm prologue reproduces the stand-alone kernel bit for bit (later ops see inputs
    # that differ in the last bit: fp32 atomics order)
    assert torch.equal(bufs[0]["xn"], ref[0]["xn"])


def test_program_replays_and_leaves_scratch_clean(api, small_blocks, kind):
    from autoawq_b200.program import DecodeProgram

    h = _h0(2048, 1, seed=3)
    prog = DecodeProgram()
    bufs = _record(prog, small_blocks, h, 1)
    prog.build()
    assert prog.fused
    prog.run()
    first = {k: v.clone() for k, v in bufs[-1].items()}
    for _ in range(5):
        prog.run()
    torch.cuda.synchronize()
    for k, v in bufs[-1].items():
        assert torch.allclose(v.float(), first[k].float(), rtol=3e-2, atol=3e-2), k
    # new input in place -> new output; then the per-op entry points still find an all-zero workspace
    h.copy_(_h0(2048, 1, seed=4))
    prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, bufs, "program replay")
    ref = _record(api, small_blocks, h, 1)
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, ref, "per-op after program")
    for ws in api._WS.values():
        assert int(ws.count_nonzero()) == 0, "program left the shared workspace dirty"


def test_program_is_bit_reproducible(api, kind):
    """Every output is summed in a fixed order by the CTA that owns it (output-stationary, csrc/program_stream.cuh):
    the result does not depend on the order in which CTAs arrive, so two runs on the same input must agree bit for
    bit - at the Llama-3-8B shapes."""
    from autoawq_b200.program import DecodeProgram

    blocks = [Block(4096, 14336, 6144, 128, seed=21)]
    h = _h0(4096, 1, seed=13)
    prog = DecodeProgram()
    bufs = _record(prog, blocks, h, 1)
    prog.build()
    assert prog.fused
    prog.run()
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in bufs[0].items()}
    for _ in range(4):
        prog.run()
        torch.cuda.synchronize()
        for k, v in bufs[0].items():
            assert torch.equal(v, first[k]), f"{k} differs between two runs of the same program"
    _no_abort("reproducibility")


def test_program_in_cuda_graph(api, small_blocks, kind):
    from autoawq_b200.program import DecodeProgram

    h = _h0(2048, 1, seed=5)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog = DecodeProgram()
        bufs = _record(prog, small_blocks, h, 1)
        prog.build()
        prog.run()  # allocates the stream's workspace outside the capture
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            prog.run()
        h.copy_(_h0(2048, 1, seed=6))
        g.replay()
        s.synchronize()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, bufs, "program graph replay")


def test_program_falls_back_per_op_when_not_fusable(api, small_blocks):
    from autoawq_b200.program import DecodeProgram

    h = _h0(2048, 2, seed=7)  # M = 2: outside the fused kernel's envelope
    prog = DecodeProgram()
    bufs = _record(prog, small_blocks[:1], h, 2)
    prog.build()
    assert not prog.fused and prog.launches_per_run == 7
    prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks[:1], bufs, "program (per-op replay)")


def test_program_rejects_unconsumed_glue_and_aliasing(api, small_blocks):
    from autoawq_b200.program import DecodeProgram

    b = small_blocks[0]
    h = _h0(2048, 1)
    xn = torch.empty_like(h)
    p = DecodeProgram()
    p.layernorm_forward_cuda(h, b.norm1_t, xn, EPS)   # nobody reads xn
    p.gemm_forward_cuda(h, *b.w["qkv"], 8)
    p.build()
    assert not p.fused
    p2 = DecodeProgram()
    p2.layernorm_forward_cuda(h, b.norm1_t, xn, EPS)
    p2.gemm_forward_cuda(xn, *b.w["qkv"], 8)
    p2.gemm_forward_cuda(xn, *b.w["o"], 8)            # second reader of the same norm output: prologue re-applied
    p2.build()
    assert p2.fused and p2.kernel_ops == 2
    p2.run()
    torch.cuda.synchronize()


def test_program_llama8b_layer_shapes(api, kind):
    """BASELINE config 2 shapes (Llama-3-8B, g128): two full-size blocks, program vs oracle op by op."""
    from autoawq_b200.program import DecodeProgram

    blocks = [Block(4096, 14336, 6144, 128, seed=s) for s in (11, 12)]
    h = _h0(4096, 1, seed=9)
    prog = DecodeProgram()
    bufs = _record(prog, blocks, h, 1)
    prog.build()
    assert prog.fused and prog.kernel_ops == 8 and prog.kind == kind
    for _ in range(3):
        prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(blocks, bufs, "program 8B shapes")


def test_program_bias_group64_and_older_source(api, kind):
    """Paths the Llama chain does not touch: linears with a bias (added before the fp16 rounding, as the per-op path
    does), group size 64, and a linear whose source is the output of an op OLDER than its predecessor (read from that
    op's published row, `ext_dep`)."""
    from autoawq_b200.program import DecodeProgram

    H, G = 2048, 64
    rng = np.random.default_rng(5)
    cs = [O.make_case(H, H, G, seed=70 + i) for i in range(3)]
    sc = [(c["scales"].astype(np.float32) / (6.1 * 0.0108 * np.sqrt(H))).astype(np.float16) for c in cs]
    ws = [O.dequantize_gemm(c["qweight"], c["qzeros"], s, G) for c, s in zip(cs, sc)]
    bias = [(rng.standard_normal(H) * 0.25).astype(np.float16) for _ in range(3)]
    x = _h0(H, 1, seed=17)
    prog = DecodeProgram()
    y0 = prog.gemm_forward_cuda(x, _t(cs[0]["qweight"]), _t(sc[0]), _t(cs[0]["qzeros"]), 8, bias=_t(bias[0]))
    y1 = prog.gemm_forward_cuda(y0, _t(cs[1]["qweight"]), _t(sc[1]), _t(cs[1]["qzeros"]), 8, bias=_t(bias[1]))
    y2 = prog.gemm_forward_cuda(y0, _t(cs[2]["qweight"]), _t(sc[2]), _t(cs[2]["qzeros"]), 8, bias=_t(bias[2]))  # older src
    prog.build()
    assert prog.fused and prog.kernel_ops == 3 and prog.kind == kind
    for _ in range(3):
        prog.run()
    torch.cuda.synchronize()
    _no_abort("bias / g64 / ext_dep")
    xin = [x.cpu().numpy(), y0.cpu().numpy(), y0.cpu().numpy()]
    for i, y in enumerate((y0, y1, y2)):
        ref = O.gemm_f64(xin[i], ws[i]) + bias[i].astype(np.float64)
        budget = np.abs(xin[i].astype(np.float64)) @ np.abs(ws[i].astype(np.float64))
        _close(y.cpu().numpy(), ref, budget, f"op {i}")


# ------------------------------------------------------------------------------------- the stream format itself
@pytest.mark.parametrize("K,N,G,mode", [(256, 32, 128, 0), (128, 32, 32, 0), (256, 48, 64, 0), (256, 64, 128, 1),
                                        (512, 32, -1, 0), (4096, 4096, 128, 0), (4096, 28672, 128, 1)])
def test_stream_pack_bit_exact_vs_oracle(api, K, N, G, mode):
    """b200awq_stream_pack (the one-time re-layout, SURVEY 8f #4) against its numpy restatement
    (oracle/stream_format.py, itself pinned to the reference's dequantize_gemm semantics in the CPU tests)."""
    from oracle import stream_format as SF

    c = O.make_case(K, N, G, seed=K + N + mode, raw=True)
    Gs = c["group_size"]
    got = api.stream_pack(_t(c["qweight"]), _t(c["scales"]), _t(c["qzeros"]), mode).cpu().numpy()
    want = SF.pack_stream(c["qweight"], c["qzeros"], c["scales"], Gs, mode)
    assert got.size == SF.stream_bytes(K, N, Gs) == want.size
    assert np.array_equal(got, want)


def test_stream_program_general_groups_and_small_shapes(api):
    """Stream variant outside the Llama shapes: G = 32 / 64 / per-channel (G = K), N not a multiple of 256, a chain of
    plain copies; every op against the oracle."""
    from autoawq_b200.program import DecodeProgram

    api.set_knob(14, 2)
    try:
        rng = np.random.default_rng(3)
        dims = [(512, 1024, 32), (1024, 1936, 64), (1920, 512, 128)]   # op 2 reads columns 16 .. 1935 of op 1's output
        cs, scs, ws = [], [], []
        for K, N, G in dims:
            c = O.make_case(K, N, G, seed=K)
            sc = (c["scales"].astype(np.float32) / (6.1 * 0.0108 * np.sqrt(K))).astype(np.float16)
            cs.append(c); scs.append(sc); ws.append(O.dequantize_gemm(c["qweight"], c["qzeros"], sc, c["group_size"]))
        x = _t(rng.standard_normal((1, 512)).astype(np.float16))
        prog = DecodeProgram()
        y0 = prog.gemm_forward_cuda(x, _t(cs[0]["qweight"]), _t(scs[0]), _t(cs[0]["qzeros"]), 8)
        y1 = prog.gemm_forward_cuda(y0, _t(cs[1]["qweight"]), _t(scs[1]), _t(cs[1]["qzeros"]), 8)
        y2 = prog.gemm_forward_cuda(y1[:, 16:1936], _t(cs[2]["qweight"]), _t(scs[2]), _t(cs[2]["qzeros"]), 8)
        prog.build()
        assert prog.kind == "stream"
        for _ in range(2):
            prog.run()
        torch.cuda.synchronize()
        _no_abort("stream general")
        xin = [x.cpu().numpy(), y0.cpu().numpy(), y1.cpu().numpy()[:, 16:1936]]
        for i, y in enumerate((y0, y1, y2)):
            budget = np.abs(xin[i].astype(np.float64)) @ np.abs(ws[i].astype(np.float64))
            _close(y.cpu().numpy(), O.gemm_f64(xin[i], ws[i]), budget, f"stream general op {i}")
    finally:
        api.set_knob(14, 0)
