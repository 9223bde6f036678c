"""Host logic of residual adds in decode programs (B200AWQ_OP_ADD), checked without a GPU: argument validation, every
rule that sends a sequence back to the per-op path, the ABI constant, and the register / spill budget of the residual
kernel entries.

The sequences go through b200awq_program_plan: program_create's folding for a 132-SM device, without any CUDA call, so
every test discriminates on any machine.  The recorded pointers are fake (aligned integers): the folding only compares
addresses.  Shapes are Llama-like (4096 columns: 31 sets per SM)."""
import ctypes

from _fake_ops import add, buf, linear, plan, rmsnorm, silu
from _toolchain import entries, header_constants, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
K, N, SMS = 4096, 4096, 132


def _create(ops):
    return plan(ops, sms=SMS)[0]


def test_op_add_matches_header():
    assert header_constants("B200AWQ_OP_ADD") == (_cabi.OP_ADD,) == (5,)


def test_add_argument_validation():
    x = buf()
    lin = linear(x, K, N)
    r = buf()
    assert _create([lin, add(lin["y"], 0, N)]) == EINVAL
    assert _create([lin, add(0, r, N)]) == EINVAL
    assert _create([lin, dict(add(lin["y"], r, N), y=0)]) == EINVAL
    assert _create([lin, add(lin["y"], r, 0)]) == EINVAL
    assert _create([lin, add(lin["y"], r, N - 4)]) == EUNSUPPORTED        # K % 8
    assert _create([lin, add(lin["y"], r + 8, N)]) == EUNSUPPORTED             # not 16-byte aligned


def test_controls_fold():
    x, r = buf(), buf()
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N)]) == OK                        # external residual
    assert _create([lin, add(r, lin["y"], N)]) == OK                        # either operand order
    # the segment shape: o + h_in -> h, norm(h) -> gate|up ... down + h (two kernel ops back)
    o = linear(x, K, N)
    h = add(o["y"], r, N)
    nm = rmsnorm(h["y"], N)
    a = linear(nm["y"], N, N)
    b = linear(a["y"], N, N)
    assert _create([o, h, nm, a, b, add(b["y"], h["y"], N)]) == OK
    # an op reading the add's output resolves to the producer's row
    o2 = linear(x, K, N)
    h2 = add(o2["y"], r, N)
    assert _create([o2, h2, linear(h2["y"], N, N)]) == OK


def test_add_after_glue_op():
    x, r = buf(), buf()
    nm = rmsnorm(x, N)
    assert _create([nm, add(nm["y"], r, N), linear(nm["y"], N, N)]) == EUNSUPPORTED


def test_add_after_add():
    x, r, r2 = buf(), buf(), buf()
    lin = linear(x, K, N)
    a1 = add(lin["y"], r, N)
    assert _create([lin, a1, add(a1["y"], r2, N)]) == EUNSUPPORTED


def test_add_after_gate_up_read_by_silu():
    x, r = buf(), buf()
    gu = linear(x, K, 2 * N)
    act = buf()
    ops = [gu, add(gu["y"], r, 2 * N), silu(gu["y"], N, y=act), linear(act, N, N)]
    assert _create(ops) == EUNSUPPORTED


def test_add_with_both_operands_external():
    x = buf()
    lin = linear(x, K, N)
    assert _create([lin, add(buf(), buf(), N)]) == EUNSUPPORTED
    assert _create([lin, add(lin["y"], lin["y"], N)]) == EUNSUPPORTED        # y + y: no residual


def test_in_place_add():
    x, r = buf(), buf()
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N, y=lin["y"])]) == EUNSUPPORTED
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N, y=r)]) == EUNSUPPORTED


def test_residual_window():
    x = buf()
    chain = [linear(x, K, N)]
    for _ in range(5):
        chain.append(linear(chain[-1]["y"], N, N))
    assert _create(chain[:5] + [add(chain[4]["y"], chain[0]["y"], N)]) == OK               # four kernel ops back
    assert _create(chain + [add(chain[5]["y"], chain[0]["y"], N)]) == EUNSUPPORTED         # five: outside the window


def test_residual_the_program_overwrites():
    x, r = buf(), buf()
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N), linear(buf(), K, N, y=r)]) == EUNSUPPORTED     # a later linear writes it
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N), rmsnorm(buf(), N, y=r), linear(r, N, N)]) == EUNSUPPORTED   # ... a later glue op


def test_reading_the_raw_output_under_an_add():
    x, r = buf(), buf()
    lin = linear(x, K, N)
    assert _create([lin, add(lin["y"], r, N), linear(lin["y"], N, N)]) == EUNSUPPORTED


def test_residual_row_rewritten_without_a_staging_wait():
    """Residual of op 1 = op 0's row; op 4 republishes row 0.  With ops 2..4 reading only external buffers nothing makes
    a CTA wait for op 1's finish before it overwrites row 0 (tests/test_stream_residual_model.py)."""
    x, r = buf(), buf()
    l0 = linear(x, K, N)
    l1 = linear(l0["y"], N, N)
    tail = [linear(buf(), K, N) for _ in range(3)]
    assert _create([l0, l1, add(l1["y"], l0["y"], N)] + tail) == EUNSUPPORTED


def test_residual_row_rewritten_after_a_staging_wait_folds():
    x = buf()
    l0 = linear(x, K, N)
    l1 = linear(l0["y"], N, N)
    s = add(l1["y"], l0["y"], N)
    l2 = linear(s["y"], N, N)                  # stages from op 1: every CTA finished op 1 before anyone passes it
    tail = [linear(buf(), K, N) for _ in range(2)]
    assert _create([l0, l1, s, l2] + tail) == OK


def test_residual_row_rewritten_after_a_wait_on_a_slice():
    """The wait that orders the CTAs must be on a whole row: op 2 stages only the first half of op 1's sum, so it waits
    for the CTAs owning those columns, and the others may run on to op 4, which republishes row 0 while a CTA owning the
    second half still reads op 0's row as its residual in op 1's finish."""
    x = buf()
    l0 = linear(x, K, N)
    l1 = linear(l0["y"], N, N)
    s = add(l1["y"], l0["y"], N)
    l2 = linear(s["y"], N // 2, N)
    tail = [linear(buf(), K, 2 * N) for _ in range(2)]
    assert _create([l0, l1, s, l2] + tail) == EUNSUPPORTED
    l2 = linear(s["y"], N, N)                  # the whole row: folds
    assert _create([l0, l1, s, l2] + tail) == OK


def test_residual_row_rewritten_after_a_wait_on_a_narrow_op():
    x = buf()
    l0 = linear(x, K, 1024)                    # 64 sets: fewer than one per SM
    l1 = linear(l0["y"], 1024, 1024)
    s = add(l1["y"], l0["y"], 1024)
    l2 = linear(s["y"], 1024, N)
    assert _create([l0, l1, s, l2] + [linear(buf(), K, N) for _ in range(2)]) == EUNSUPPORTED


def test_plan_argument_validation():
    ops = (_cabi.Op * 1)()
    kops = ctypes.c_int()
    assert lib.b200awq_program_plan(ops, 1, 1, 0, 0, ctypes.byref(kops)) == EINVAL
    assert lib.b200awq_program_plan(ops, 1, 9, SMS, 0, ctypes.byref(kops)) == EINVAL
    assert lib.b200awq_program_plan(ops, 1, 1, SMS, 0, None) == EINVAL


def test_external_residual_aliasing_a_moe_buffer():
    """The fused MoE block writes its routing tensors too: none of them may be an external residual."""
    H, I, E, k = 1024, 512, 8, 2
    x, h = buf(), buf()
    for field in ("logits", "topk_weights", "topk_ids", "token_expert_indices", "sorted_ids", "expert_ids",
                  "num_tokens_post_pad", "gate_up", "act", "down"):
        d = _cabi.Moe()
        d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, H, I, 16
        d.sorted_len = k + E * 15
        for f, _ in _cabi.Moe._fields_[8:]:
            setattr(d, f, buf())
        res = buf()
        setattr(d, field, res)
        nm = rmsnorm(x, H)
        moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=H, N=H, x=nm["y"], y=buf(), weight=ctypes.addressof(d))
        pre = linear(h, K, H)
        ops = [pre, add(pre["y"], res, H), nm, moe]
        assert _create(ops) == EUNSUPPORTED, field
        ops = [pre, add(pre["y"], buf(), H), nm, moe]
        assert _create(ops) == OK, field


@needs_nvcc
def test_residual_kernels_register_and_spill_budget():
    """One CTA per SM: the residual entries (M = 1: 288 threads; batched: 288 threads) fit the register file and spill
    nothing."""
    found = entries("program.cu", r"residual_kernel")
    assert len(found) == 4, found          # stream_residual_kernel, stream_batch_residual_kernel<2|4|8>
    for name, (regs, stack, st, ld) in found.items():
        assert regs * (32 + 32 * 8) <= 65536, f"{name}: {regs} registers x 288 threads"
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills {st} / {ld}, stack {stack}"
