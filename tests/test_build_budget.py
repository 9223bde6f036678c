"""Resource budget of the decode-program and tensor-core kernels, checked from ptxas without a GPU (nvcc cross-compiles
sm_90a): one CTA per SM must fit the register file without spilling - a spill in the tile loop, or a register count
that drops the launch to zero resident CTAs, would only show up on the GPU otherwise."""
import re

from _toolchain import entries, needs_nvcc


@needs_nvcc
def test_stream_program_kernel_register_and_spill_budget():
    found = entries("program.cu", r"stream_program_kernel")
    assert len(found) == 2, found          # stream_program_kernel<8|12 warps>
    for name, (regs, stack, st, ld) in found.items():
        # one resident CTA of 32 + 32 NW threads; a few spilled words in the staging phase (off the unit loop) are
        # tolerated, a spilling unit loop is not: keep the total small
        nw = int(re.search(r"kernelILi(\d+)E", name).group(1))
        assert regs * (32 + 32 * nw) <= 65536, f"{name}: {regs} registers x {32 + 32 * nw} threads"
        assert st <= 128 and ld <= 256, f"{name}: spills {st} / {ld} bytes"


@needs_nvcc
def test_batched_kernel_register_and_spill_budget():
    """One resident CTA of 288 threads must fit the register file, and nothing may spill: ptxas does not say where a
    spill would land, and one in the unit loop would cost a local-memory round trip per unit."""
    found = entries("program.cu", r"stream_batch_kernel")
    assert sorted(int(re.search(r"kernelILi(\d+)E", n).group(1)) for n in found) == [2, 4, 8], found
    for name, (regs, stack, st, ld) in found.items():
        assert regs * (32 + 32 * 8) <= 65536, f"{name}: {regs} registers x 288 threads"
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills {st} / {ld} bytes, stack {stack}"


@needs_nvcc
def test_tensor_core_kernels_register_budget():
    """One CTA per SM: gemm_tc_kernel runs 512 threads, gemm_tcq_kernel 576 - registers x threads must fit the 64 K
    register file and nothing may spill (the accumulators live in the consumer warpgroups' registers: a spill there
    would put them in local memory on every k-step)."""
    found = entries("gemm_tc.cu", r"gemm_tcq?_kernel")
    tcq = {n: v for n, v in found.items() if "gemm_tcq_kernel" in n}
    tc = {n: v for n, v in found.items() if "gemm_tcq_kernel" not in n}
    assert len(tcq) == 4 and len(tc) == 12, (len(tcq), len(tc))     # BT in {16, 32, 64, 128}; 3 token tiles x 4 layouts
    for name, (regs, stack, st, ld) in tcq.items():
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills"
        assert regs * 576 <= 65536, f"{name}: {regs} registers x 576 threads"
    for name, (regs, stack, st, ld) in tc.items():
        assert st == 0 and ld == 0, f"{name}: spills"
        assert regs * 512 <= 65536, f"{name}: {regs} registers x 512 threads"
