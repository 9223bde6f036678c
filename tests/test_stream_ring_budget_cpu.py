"""Register budget of the M = 1 stream entries that run the real-model path (stream_moe_kernel, stream_residual_kernel,
stream_rope_kernel), checked from ptxas without a GPU.  They take their ring depth as a kernel argument
(csrc/program_stream.cuh: sp_fixed_smem); a layout whose offsets depend on the program costs these 9-warp kernels
registers they do not have (a thread is capped at 168), and the spill would sit in the unit loop."""
from _toolchain import entries, needs_nvcc


@needs_nvcc
def test_stream_moe_residual_rope_kernels_do_not_spill():
    found = entries("program.cu", r"stream_(?:moe|residual|rope)_kernel")
    assert len(found) == 3, found
    for name, (regs, stack, st, ld) in found.items():
        assert st == 0 and ld == 0, f"{name}: spills {st} / {ld} bytes"
        assert regs <= 168, f"{name}: {regs} registers (9 warps: at most 168 per thread)"
