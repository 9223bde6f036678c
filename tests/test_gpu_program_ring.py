"""GPU tests of the M = 1 stream kernels' program-sized weight ring and L2 run-ahead (csrc/program.cu: sp_pick_spw,
knobs 8 / 9 / 10).  The ring depth, the run-ahead window and the load gate change only when weight bytes arrive, never
which warp computes what or in which order: every output must stay bit for bit what the default run computes."""
import pytest
import torch

from test_gpu_program import Block, _check_against_oracle, _h0, _no_abort, _record

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext

    return ext


def _run_with(api, prog, bufs, knobs):
    was = {k: api.get_knob(k) for k in knobs}
    try:
        for k, v in knobs.items():
            api.set_knob(k, v)
        prog.run()
        torch.cuda.synchronize()
    finally:
        for k, v in was.items():
            api.set_knob(k, v)
    _no_abort(f"knobs {knobs}")
    return [{k: v.clone() for k, v in b.items()} for b in bufs]


@pytest.mark.parametrize("hidden,inter,qkv_out", [(4096, 14336, 6144), (1024, 2048, 1536)])
def test_ring_and_run_ahead_do_not_change_outputs(api, hidden, inter, qkv_out):
    """Llama-3-8B shapes (5 ring stages per warp) and a small model (6 stages): the default run against the L2
    run-ahead windows, the gated loads and both together, bit for bit; every run also against the oracle."""
    from autoawq_b200.program import DecodeProgram

    blocks = [Block(hidden, inter, qkv_out, 128, seed=s) for s in (31, 32)]
    h = _h0(hidden, 1, seed=3)
    prog = DecodeProgram()
    bufs = _record(prog, blocks, h, 1)
    prog.build()
    assert prog.fused and prog.kind == "stream"
    ref = _run_with(api, prog, bufs, {8: 0, 10: 0})
    _check_against_oracle(blocks, bufs, "default ring")
    for knobs in ({8: 8}, {8: 16}, {8: 32}, {8: 4096}, {10: 2}, {8: 16, 10: 2}):
        got = _run_with(api, prog, bufs, knobs)
        for li, (r, g) in enumerate(zip(ref, got)):
            for k in r:
                assert torch.equal(r[k], g[k]), f"knobs {knobs}: layer {li} {k} differs from the default run"


def test_twelve_warp_ring(api):
    """knob 9 = 12: 12 consumer warps with the ring depth chosen for them at creation, against the oracle."""
    from autoawq_b200.program import DecodeProgram

    blocks = [Block(4096, 14336, 6144, 128, seed=33)]
    h = _h0(4096, 1, seed=4)
    prog = DecodeProgram()
    bufs = _record(prog, blocks, h, 1)
    prog.build()
    assert prog.fused
    _run_with(api, prog, bufs, {9: 12})
    _check_against_oracle(blocks, bufs, "12 warps")
    _run_with(api, prog, bufs, {9: 12, 8: 16})
    _check_against_oracle(blocks, bufs, "12 warps, 16 MB run-ahead")
