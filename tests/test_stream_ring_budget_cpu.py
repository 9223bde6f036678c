"""Register budget of the M = 1 stream entries that run the real-model path (stream_moe_kernel, stream_residual_kernel,
stream_rope_kernel), checked from ptxas without a GPU.  They take their ring depth as a kernel argument
(csrc/program_stream.cuh: sp_fixed_smem); a layout whose offsets depend on the program costs these 9-warp kernels
registers they do not have (a thread is capped at 168), and the spill would sit in the unit loop."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_stream_moe_residual_rope_kernels_do_not_spill(tmp_path):
    src = os.path.join(ROOT, "autoawq_b200", "csrc", "program.cu")
    out = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xptxas", "-v", "-c", src,
         "-o", str(tmp_path / "program.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stderr + out.stdout
    entries = re.findall(r"Compiling entry function '(\S*stream_(?:moe|residual|rope)_kernel\S*)'[^\n]*\n[^\n]*\n\s*"
                         r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) "
                         r"registers", log)
    assert len(entries) == 3, log[-1500:]
    for name, stack, st, ld, regs in entries:
        assert int(st) == 0 and int(ld) == 0, f"{name}: spills {st} / {ld} bytes"
        assert int(regs) <= 168, f"{name}: {regs} registers (9 warps: at most 168 per thread)"
