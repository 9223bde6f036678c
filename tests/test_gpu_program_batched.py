"""Batched decode programs (csrc/program_batch.cuh, b200awq_program_create_batched): a fused block recorded with
M = 2 .. 8 token rows runs as one persistent kernel.  Every buffer is checked op by op against the fp64 oracle on the
op's actual input (the tolerance of tests/test_gpu_program.py), and every token against an M = 1 stream program run on
that token's row alone: the two must agree bit for bit.  The last test needs no GPU: the argument checks of the new
entry points (the kernels' ptxas budget is in tests/test_build_budget.py)."""
import ctypes

import numpy as np
import pytest

from test_gpu_program import Block, _check_against_oracle, _close, _h0, _no_abort, _record, _t

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext

    return ext


@pytest.fixture(scope="module")
def small_blocks():
    return [Block(2048, 4096, 3072, 128, seed=s) for s in (1, 2)]


def _batched(blocks, M, seed=0, max_tokens=None):
    from autoawq_b200.program import DecodeProgram

    h = _h0(blocks[0].hidden, M, seed=seed)
    prog = DecodeProgram(max_tokens=max_tokens or M)
    bufs = _record(prog, blocks, h, M)
    prog.build()
    return prog, h, bufs


@gpu
@pytest.mark.parametrize("M", [2, 3, 4, 8])
def test_batched_program_matches_oracle(api, small_blocks, M):
    import torch

    prog, _, bufs = _batched(small_blocks, M, seed=M)
    assert prog.fused and prog.kind == "stream" and prog.tokens == M and prog.kernel_ops == 8
    prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, bufs, f"batched M={M}")


@gpu
@pytest.mark.parametrize("M", [3, 8])
def test_batched_tokens_bit_identical_to_single_token_programs(api, small_blocks, M):
    """Token m of a batched run equals an M = 1 stream program (8 consumer warps) on row m alone."""
    import torch

    from autoawq_b200.program import DecodeProgram

    prog, h, bufs = _batched(small_blocks, M, seed=20 + M)
    assert prog.fused
    prog.run()
    torch.cuda.synchronize()
    _no_abort(f"batched M={M}")
    api.set_knob(14, 2)
    try:
        for m in range(M):
            hm = h[m:m + 1].clone()
            p1 = DecodeProgram()
            ref = _record(p1, small_blocks, hm, 1)
            p1.build()
            assert p1.fused and p1.kind == "stream" and p1.tokens == 1
            p1.run()
            torch.cuda.synchronize()
            for li, (a, b) in enumerate(zip(bufs, ref)):
                for k in a:
                    assert torch.equal(a[k][m:m + 1], b[k]), f"token {m} L{li} {k} differs from the M = 1 program"
            p1.close()
    finally:
        api.set_knob(14, 0)


@gpu
@pytest.mark.parametrize("M", [2, 4, 8])
def test_batched_llama8b_layer_shapes(api, M):
    """Llama-3-8B shapes: fused at M <= 4; at M = 8 the activations of down (K = 14336) do not fit shared memory next to
    the ring, and the program replays per op."""
    import torch

    blocks = [Block(4096, 14336, 6144, 128, seed=s) for s in (11, 12)]
    prog, _, bufs = _batched(blocks, M, seed=9)
    if M <= 4:
        assert prog.fused and prog.kind == "stream" and prog.tokens == M
    else:
        assert not prog.fused and prog.kind == "per-op" and prog.launches_per_run == 14
    for _ in range(2):
        prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(blocks, bufs, f"batched 8B shapes M={M}")


@gpu
def test_batched_replay_graph_and_reproducibility(api, small_blocks):
    import torch

    M = 4
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog, h, bufs = _batched(small_blocks, M, seed=31)
        assert prog.fused
        prog.run()
        s.synchronize()
        first = [{k: v.clone() for k, v in b.items()} for b in bufs]
        for _ in range(4):
            prog.run()
            s.synchronize()
            for a, b in zip(bufs, first):
                for k in a:
                    assert torch.equal(a[k], b[k]), f"{k} differs between two runs of the same program"
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            prog.run()
        h.copy_(_h0(2048, M, seed=32))
        g.replay()
        s.synchronize()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, bufs, "batched graph replay")
    assert not torch.equal(bufs[-1]["down"], first[-1]["down"])
    ref = _record(api, small_blocks, h, M)
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks, ref, "per-op after batched program")
    for ws in api._WS.values():
        assert int(ws.count_nonzero()) == 0, "program left the shared workspace dirty"


def _case(K, N, G, seed):
    from oracle import awq_oracle as O

    c = O.make_case(K, N, G, seed=seed)
    sc = (c["scales"].astype(np.float32) / (6.1 * 0.0108 * np.sqrt(K))).astype(np.float16)
    return c, sc, O.dequantize_gemm(c["qweight"], c["qzeros"], sc, c["group_size"])


@gpu
def test_batched_bias_group64_and_older_source(api):
    """At M = 4: linears with a bias, G = 64, and a source that is the output of an op older than its predecessor."""
    import torch

    from autoawq_b200.program import DecodeProgram
    from oracle import awq_oracle as O

    M, H = 4, 2048
    rng = np.random.default_rng(5)
    cs = [_case(H, H, 64, 70 + i) for i in range(3)]
    bias = [(rng.standard_normal(H) * 0.25).astype(np.float16) for _ in range(3)]
    x = _h0(H, M, seed=17)
    prog = DecodeProgram(max_tokens=M)
    args = [(_t(c["qweight"]), _t(sc), _t(c["qzeros"])) for c, sc, _ in cs]
    y0 = prog.gemm_forward_cuda(x, *args[0], 8, bias=_t(bias[0]))
    y1 = prog.gemm_forward_cuda(y0, *args[1], 8, bias=_t(bias[1]))
    y2 = prog.gemm_forward_cuda(y0, *args[2], 8, bias=_t(bias[2]))   # older source (ext_dep)
    prog.build()
    assert prog.fused and prog.kind == "stream" and prog.kernel_ops == 3
    for _ in range(3):
        prog.run()
    torch.cuda.synchronize()
    _no_abort("batched bias / g64 / ext_dep")
    xin = [x.cpu().numpy(), y0.cpu().numpy(), y0.cpu().numpy()]
    for i, y in enumerate((y0, y1, y2)):
        w = cs[i][2]
        ref = O.gemm_f64(xin[i], w) + bias[i].astype(np.float64)
        _close(y.cpu().numpy(), ref, np.abs(xin[i].astype(np.float64)) @ np.abs(w.astype(np.float64)), f"op {i}")


@gpu
def test_batched_general_groups_and_column_slice(api):
    """At M = 4: G = 32, G = 64, per-channel G = K, N not a multiple of 256, and a source that is a column slice of the
    producer's rows (ldx = the producer's N)."""
    import torch

    from autoawq_b200.program import DecodeProgram
    from oracle import awq_oracle as O

    M = 4
    dims = [(512, 1024, 32), (1024, 1936, 64), (1920, 512, -1)]   # op 2 reads columns 16 .. 1935 of op 1's rows
    cs = [_case(K, N, G, seed=K) for K, N, G in dims]
    x = _h0(512, M, seed=3)
    prog = DecodeProgram(max_tokens=M)
    args = [(_t(c["qweight"]), _t(sc), _t(c["qzeros"])) for c, sc, _ in cs]
    y0 = prog.gemm_forward_cuda(x, *args[0], 8)
    y1 = prog.gemm_forward_cuda(y0, *args[1], 8)
    y2 = prog.gemm_forward_cuda(y1[:, 16:1936], *args[2], 8)
    prog.build()
    assert prog.fused and prog.kind == "stream" and prog.tokens == M
    for _ in range(2):
        prog.run()
    torch.cuda.synchronize()
    _no_abort("batched general")
    xin = [x.cpu().numpy(), y0.cpu().numpy(), y1.cpu().numpy()[:, 16:1936]]
    for i, y in enumerate((y0, y1, y2)):
        w = cs[i][2]
        _close(y.cpu().numpy(), O.gemm_f64(xin[i], w), np.abs(xin[i].astype(np.float64)) @ np.abs(w.astype(np.float64)),
               f"batched general op {i}")


@gpu
def test_batched_envelope(api, small_blocks):
    """M > max_tokens, mixed M across ops and knob 14 = 1 (do not fuse) replay per op - still correct."""
    import torch

    from autoawq_b200.program import DecodeProgram
    from oracle import awq_oracle as O

    prog, _, bufs = _batched(small_blocks[:1], 4, seed=41, max_tokens=2)
    assert not prog.fused and prog.tokens == 4
    prog.run()
    torch.cuda.synchronize()
    _check_against_oracle(small_blocks[:1], bufs, "M > max_tokens (per-op)")

    b = small_blocks[0]
    mixed = DecodeProgram(max_tokens=4)
    xs = [_h0(2048, 2, seed=42), _h0(2048, 4, seed=43)]
    ys = [mixed.gemm_forward_cuda(x, *b.w["o"], 8) for x in xs]
    mixed.build()
    assert not mixed.fused
    mixed.run()
    torch.cuda.synchronize()
    w = b.np["o"]["w"]
    for i, (x, y) in enumerate(zip(xs, ys)):
        xin = x.cpu().numpy()
        _close(y.cpu().numpy(), O.gemm_f64(xin, w), np.abs(xin.astype(np.float64)) @ np.abs(w.astype(np.float64)),
               f"mixed M (per-op) op {i}")

    api.set_knob(14, 1)
    try:
        prog, _, bufs = _batched(small_blocks[:1], 4, seed=44)
        assert not prog.fused
        prog.run()
        torch.cuda.synchronize()
        _check_against_oracle(small_blocks[:1], bufs, "knob 14 = 1, M = 4 (per-op)")
    finally:
        api.set_knob(14, 0)


@gpu
@pytest.mark.parametrize("K,warps", [(18944, 8), (14336, 12)])
def test_single_token_stream_program_keeps_its_shared_memory(api, K, warps):
    """An M = 1 stream program reserves one activation row (K x 2 bytes), as before batched programs existed: with 8
    consumer warps K = 18944 (Qwen2-7B's intermediate size) fits only then, and so does K = 14336 with 12 warps (knob 9)."""
    import torch

    from autoawq_b200.program import DecodeProgram
    from oracle import awq_oracle as O

    c, sc, w = _case(K, 4096, 128, seed=K + warps)
    x = _h0(K, 1, seed=50)
    api.set_knob(14, 2)
    api.set_knob(9, warps)
    try:
        prog = DecodeProgram()
        y = prog.gemm_forward_cuda(x, _t(c["qweight"]), _t(sc), _t(c["qzeros"]), 8)
        prog.build()
        assert prog.fused and prog.kind == "stream" and prog.tokens == 1
        prog.run()
        torch.cuda.synchronize()
    finally:
        api.set_knob(9, 0)
        api.set_knob(14, 0)
    _no_abort(f"M = 1, K = {K}, {warps} warps")
    xin = x.cpu().numpy()
    _close(y.cpu().numpy(), O.gemm_f64(xin, w), np.abs(xin.astype(np.float64)) @ np.abs(w.astype(np.float64)),
           f"M = 1 stream, K = {K}, {warps} warps")


# ------------------------------------------------------------------------------------------------- no GPU needed
def test_batched_create_argument_validation_without_gpu():
    import autoawq_b200  # noqa: F401  (builds / locates the library)
    from autoawq_b200 import _cabi

    lib = _cabi.lib
    h = ctypes.c_void_p()
    ops = (_cabi.Op * 1)()
    for bad in (0, 9, -1):
        assert lib.b200awq_program_create_batched(ops, 1, bad, ctypes.byref(h)) == 1 and not h.value
    assert lib.b200awq_program_create_batched(None, 0, 4, ctypes.byref(h)) == 1
    assert lib.b200awq_program_create_batched(ops, 1, 4, None) == 1
    assert lib.b200awq_program_create_batched(ops, 1, 4, ctypes.byref(h)) == 1 and not h.value   # null tensors
    assert lib.b200awq_program_tokens(None) == 0
    from autoawq_b200.program import DecodeProgram

    for bad in (0, 9):
        with pytest.raises(_cabi.B200AwqError):
            DecodeProgram(max_tokens=bad)
    assert DecodeProgram(max_tokens=8).tokens == 0

