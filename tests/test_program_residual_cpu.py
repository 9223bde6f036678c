"""Host logic of residual adds in decode programs (B200AWQ_OP_ADD), checked without a GPU: argument validation, every
rule that sends a sequence back to the per-op path, the ABI constant, and the register / spill budget of the residual
kernel entries.

The sequences go through b200awq_program_plan: program_create's folding for a 132-SM device, without any CUDA call, so
every test discriminates on any machine.  The recorded pointers are fake (aligned integers): the folding only compares
addresses.  Shapes are Llama-like (4096 columns: 31 sets per SM)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, EUNSUPPORTED = 0, 1, 2
K, N, SMS = 4096, 4096, 132
_next = [0x10000000]


def _buf(nbytes=1 << 16):
    p = _next[0]
    _next[0] += (nbytes + 0xffff) & ~0xffff
    return p


def _lin(x, y=None, k=K, n=N):
    return dict(kind=_cabi.OP_LINEAR_GEMM, M=1, K=k, N=n, group_size=128, ldx=k, x=x, qweight=_buf(), scales=_buf(),
                qzeros=_buf(), y=y or _buf())


def _add(a, b, y=None, k=N):
    return dict(kind=_cabi.OP_ADD, M=1, K=k, x=a, weight=b, y=y or _buf())


def _norm(x, y=None, k=N):
    return dict(kind=_cabi.OP_RMSNORM, M=1, K=k, x=x, weight=_buf(), y=y or _buf(), eps=1e-5)


def _create(ops):
    arr = (_cabi.Op * len(ops))()
    for c, o in zip(arr, ops):
        for f, v in o.items():
            setattr(c, f, v)
    kops = ctypes.c_int()
    return lib.b200awq_program_plan(arr, len(ops), 1, SMS, 0, ctypes.byref(kops))


def test_op_add_matches_header(tmp_path):
    src = tmp_path / "k.c"
    src.write_text('#include <stdio.h>\n#include "b200awq.h"\nint main(void) { printf("%d", B200AWQ_OP_ADD); return 0; }\n')
    exe = tmp_path / "k"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)])) == _cabi.OP_ADD == 5


def test_add_argument_validation():
    x = _buf()
    lin = _lin(x)
    r = _buf()
    assert _create([lin, _add(lin["y"], 0)]) == EINVAL
    assert _create([lin, _add(0, r)]) == EINVAL
    assert _create([lin, dict(_add(lin["y"], r), y=0)]) == EINVAL
    assert _create([lin, _add(lin["y"], r, k=0)]) == EINVAL
    assert _create([lin, _add(lin["y"], r, k=N - 4)]) == EUNSUPPORTED        # K % 8
    assert _create([lin, _add(lin["y"], r + 8)]) == EUNSUPPORTED             # not 16-byte aligned


def test_controls_fold():
    x, r = _buf(), _buf()
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r)]) == OK                        # external residual
    assert _create([lin, _add(r, lin["y"])]) == OK                        # either operand order
    # the segment shape: o + h_in -> h, norm(h) -> gate|up ... down + h (two kernel ops back)
    o = _lin(x)
    h = _add(o["y"], r)
    nm = _norm(h["y"])
    a = _lin(nm["y"], k=N)
    b = _lin(a["y"], k=N)
    assert _create([o, h, nm, a, b, _add(b["y"], h["y"])]) == OK
    # an op reading the add's output resolves to the producer's row
    o2 = _lin(x)
    h2 = _add(o2["y"], r)
    assert _create([o2, h2, _lin(h2["y"], k=N)]) == OK


def test_add_after_glue_op():
    x, r = _buf(), _buf()
    nm = _norm(x)
    assert _create([nm, _add(nm["y"], r), _lin(nm["y"], k=N)]) == EUNSUPPORTED


def test_add_after_add():
    x, r, r2 = _buf(), _buf(), _buf()
    lin = _lin(x)
    a1 = _add(lin["y"], r)
    assert _create([lin, a1, _add(a1["y"], r2)]) == EUNSUPPORTED


def test_add_after_gate_up_read_by_silu():
    x, r = _buf(), _buf()
    gu = _lin(x, n=2 * N)
    act = _buf()
    ops = [gu, _add(gu["y"], r, k=2 * N), dict(kind=_cabi.OP_SILU_AND_MUL, M=1, K=N, x=gu["y"], y=act), _lin(act, k=N)]
    assert _create(ops) == EUNSUPPORTED


def test_add_with_both_operands_external():
    x = _buf()
    lin = _lin(x)
    assert _create([lin, _add(_buf(), _buf())]) == EUNSUPPORTED
    assert _create([lin, _add(lin["y"], lin["y"])]) == EUNSUPPORTED        # y + y: no residual


def test_in_place_add():
    x, r = _buf(), _buf()
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r, y=lin["y"])]) == EUNSUPPORTED
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r, y=r)]) == EUNSUPPORTED


def test_residual_window():
    x = _buf()
    chain = [_lin(x)]
    for _ in range(5):
        chain.append(_lin(chain[-1]["y"], k=N))
    assert _create(chain[:5] + [_add(chain[4]["y"], chain[0]["y"])]) == OK               # four kernel ops back
    assert _create(chain + [_add(chain[5]["y"], chain[0]["y"])]) == EUNSUPPORTED         # five: outside the window


def test_residual_the_program_overwrites():
    x, r = _buf(), _buf()
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r), _lin(_buf(), y=r, k=K)]) == EUNSUPPORTED     # a later linear writes it
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r), _norm(_buf(), y=r), _lin(r, k=N)]) == EUNSUPPORTED   # ... a later glue op


def test_reading_the_raw_output_under_an_add():
    x, r = _buf(), _buf()
    lin = _lin(x)
    assert _create([lin, _add(lin["y"], r), _lin(lin["y"], k=N)]) == EUNSUPPORTED


def test_residual_row_rewritten_without_a_staging_wait():
    """Residual of op 1 = op 0's row; op 4 republishes row 0.  With ops 2..4 reading only external buffers nothing makes
    a CTA wait for op 1's finish before it overwrites row 0 (tests/test_stream_residual_model.py)."""
    x, r = _buf(), _buf()
    l0 = _lin(x, n=N)
    l1 = _lin(l0["y"], k=N)
    tail = [_lin(_buf()) for _ in range(3)]
    assert _create([l0, l1, _add(l1["y"], l0["y"])] + tail) == EUNSUPPORTED


def test_residual_row_rewritten_after_a_staging_wait_folds():
    x = _buf()
    l0 = _lin(x, n=N)
    l1 = _lin(l0["y"], k=N)
    s = _add(l1["y"], l0["y"])
    l2 = _lin(s["y"], k=N)                  # stages from op 1: every CTA finished op 1 before anyone passes it
    tail = [_lin(_buf()) for _ in range(2)]
    assert _create([l0, l1, s, l2] + tail) == OK


def test_residual_row_rewritten_after_a_wait_on_a_slice():
    """The wait that orders the CTAs must be on a whole row: op 2 stages only the first half of op 1's sum, so it waits
    for the CTAs owning those columns, and the others may run on to op 4, which republishes row 0 while a CTA owning the
    second half still reads op 0's row as its residual in op 1's finish."""
    x = _buf()
    l0 = _lin(x)
    l1 = _lin(l0["y"], k=N)
    s = _add(l1["y"], l0["y"])
    l2 = _lin(s["y"], k=N // 2)
    tail = [_lin(_buf(), n=2 * N) for _ in range(2)]
    assert _create([l0, l1, s, l2] + tail) == EUNSUPPORTED
    l2 = _lin(s["y"], k=N)                  # the whole row: folds
    assert _create([l0, l1, s, l2] + tail) == OK


def test_residual_row_rewritten_after_a_wait_on_a_narrow_op():
    x = _buf()
    l0 = _lin(x, n=1024)                    # 64 sets: fewer than one per SM
    l1 = _lin(l0["y"], k=1024, n=1024)
    s = _add(l1["y"], l0["y"], k=1024)
    l2 = _lin(s["y"], k=1024)
    assert _create([l0, l1, s, l2] + [_lin(_buf()) for _ in range(2)]) == EUNSUPPORTED


def test_plan_argument_validation():
    ops = (_cabi.Op * 1)()
    kops = ctypes.c_int()
    assert lib.b200awq_program_plan(ops, 1, 1, 0, 0, ctypes.byref(kops)) == EINVAL
    assert lib.b200awq_program_plan(ops, 1, 9, SMS, 0, ctypes.byref(kops)) == EINVAL
    assert lib.b200awq_program_plan(ops, 1, 1, SMS, 0, None) == EINVAL


def test_external_residual_aliasing_a_moe_buffer():
    """The fused MoE block writes its routing tensors too: none of them may be an external residual."""
    H, I, E, k = 1024, 512, 8, 2
    x, h = _buf(), _buf()
    for field in ("logits", "topk_weights", "topk_ids", "token_expert_indices", "sorted_ids", "expert_ids",
                  "num_tokens_post_pad", "gate_up", "act", "down"):
        d = _cabi.Moe()
        d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, H, I, 16
        d.sorted_len = k + E * 15
        for f, _ in _cabi.Moe._fields_[8:]:
            setattr(d, f, _buf())
        res = _buf()
        setattr(d, field, res)
        nm = _norm(x, k=H)
        moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=H, N=H, x=nm["y"], y=_buf(), weight=ctypes.addressof(d))
        pre = _lin(h, n=H)
        ops = [pre, _add(pre["y"], res, k=H), nm, moe]
        assert _create(ops) == EUNSUPPORTED, field
        ops = [pre, _add(pre["y"], _buf(), k=H), nm, moe]
        assert _create(ops) == OK, field


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_residual_kernels_register_and_spill_budget(tmp_path):
    """One CTA per SM: the residual entries (M = 1: 288 threads; batched: 288 threads) fit the register file and spill
    nothing."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "autoawq_b200", "csrc", "program.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xptxas",
                          "-v", "-c", src, "-o", str(tmp_path / "program.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stderr + out.stdout
    entries = re.findall(r"Compiling entry function '(\S*residual_kernel\S*)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log)
    assert len(entries) == 4, log[-1500:]          # stream_residual_kernel, stream_batch_residual_kernel<2|4|8>
    for name, stack, st, ld, regs in entries:
        assert int(regs) * (32 + 32 * 8) <= 65536, f"{name}: {regs} registers x 288 threads"
        assert int(st) == 0 and int(ld) == 0 and int(stack) == 0, f"{name}: spills {st} / {ld}, stack {stack}"
