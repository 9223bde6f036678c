"""Host logic of sparse-MoE blocks in stream decode programs, checked without a GPU: the envelope and partition that
b200awq_moe_plan reports (the function program creation uses), the unit -> (slot, expert unit) translation the producer
and the consumers share (restated here as the device code walks it: every unit of every selected expert is streamed
exactly once and no bulk copy crosses a slot), the per-expert stream-slice sizes against oracle/stream_format.py, the
ctypes mirror of b200awq_moe_t, and the register / spill budget of the MoE kernel instantiation."""
import ctypes

import pytest

from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from oracle import stream_format as SF

UPS = {128: 4, 64: 7, 32: 14}       # units per 4288-byte ring stage (kSpStageBytes / unit bytes)


def _plan(E, k, H, I, G, sms=132):
    out = (ctypes.c_int * 8)()
    rc = lib.b200awq_moe_plan(E, k, H, I, G, sms, out)
    return rc, list(out)


def test_plan_mixtral_on_h100():
    rc, p = _plan(8, 2, 4096, 14336, 128)
    assert rc == 0
    assert p[:7] == [2, 2 * 28672 // 16, (28672 // 16) * 32, 28, 2 * 14336 // 128, 14336 // 128, 2 * 2]
    assert p[7] <= 227 * 1024


@pytest.mark.parametrize("args,rc", [((65, 2, 4096, 14336, 128), 2), ((16, 9, 1024, 512, 128), 2),
                                     ((8, 8, 256, 4352, 128), 2),          # 33 gate|up sets per CTA > 32
                                     ((8, 2, 4096, 14336 + 64, 128), 2),   # I % 128: not in the stream format
                                     ((8, 2, 4096, 65536, 128), 2),        # K' = 2 x 65536: activations > smem
                                     ((0, 1, 1024, 512, 128), 1), ((4, 5, 1024, 512, 128), 1),
                                     ((64, 8, 512, 256, 32), 0), ((64, 6, 512, 256, 128), 0)])
def test_plan_envelope(args, rc):
    assert _plan(*args)[0] == rc


def _units(total, grid, nw, per_set, seg, ups):
    """(cta, warp, first unit, n) of every bulk copy: the CTA partition (whole sets), the warps' even split, chunks of
    at most `ups` units cut at slot-segment boundaries (the producer's mchunk and the consumers' loop)."""
    S = total // per_set
    for c in range(grid):
        u0, u1 = (S * c // grid) * per_set, (S * (c + 1) // grid) * per_set
        for w in range(nw):
            u, ub = u0 + (u1 - u0) * w // nw, u0 + (u1 - u0) * (w + 1) // nw
            while u < ub:
                n = min(ub - u, ups, seg - u % seg)
                yield c, w, u, n
                u += n


@pytest.mark.parametrize("E,k,H,I,G", [(8, 2, 4096, 14336, 128), (4, 1, 1024, 512, 128), (64, 6, 512, 256, 128),
                                       (8, 2, 1024, 768, 64), (16, 4, 2048, 1408 + 128, 128)])
def test_expert_units_streamed_once_and_never_across_a_slot(E, k, H, I, G):
    rc, p = _plan(E, k, H, I, G)
    assert rc == 0
    UK = min(G, 128)
    for kind in (1, 2):
        if kind == 1:   # gate|up: sets of the top_k slots side by side, H / UK units per set
            per_set, seg, total = H // UK, p[2], p[1] * (H // UK)
        else:           # down: K' = top_k I, one set = top_k segments of I / UK units
            per_set, seg, total = p[4], p[5], (H // 16) * p[4]
        seen = {}
        rows = {}
        for c, w, u, n in _units(total, 132, 8, per_set, seg, UPS[UK]):
            q, r = divmod(u, seg)
            slot, local = q % k, (q // k) * seg + r
            assert r + n <= seg, "a bulk copy crosses a slot segment"
            for i in range(n):
                key = (slot, local + i)
                assert key not in seen, f"unit {key} streamed twice"
                seen[key] = c
            if kind == 2:
                rows.setdefault(c, set()).update((u + i) // seg for i in range(n))
        per_slot_units = (2 * I // 16) * (H // UK) if kind == 1 else (H // 16) * (I // UK)
        assert len(seen) == k * per_slot_units
        for s in range(k):
            assert {lu for (sl, lu) in seen if sl == s} == set(range(per_slot_units))
        if kind == 2:   # the (set, slot) partial rows one CTA keeps fit the plan's bound
            assert max(len(v) for v in rows.values()) <= p[6] <= 32


@pytest.mark.parametrize("H,I,G", [(4096, 14336, 128), (1024, 768, 64), (512, 256, 32)])
def test_expert_slices_match_stream_format(H, I, G):
    """One stream copy per expert slice: its size is the oracle's stream_bytes of that expert's linear."""
    assert lib.b200awq_stream_bytes(H, 2 * I, G) == SF.stream_bytes(H, 2 * I, G)
    assert lib.b200awq_stream_bytes(I, H, G) == SF.stream_bytes(I, H, G)
    assert SF.unit_bytes(G) * (2 * I // 16) * (H // SF.unit_k(G)) == SF.stream_bytes(H, 2 * I, G)


def test_moe_struct_matches_header():
    assert header_layout(_cabi.Moe, "b200awq_moe_t") == mirror_layout(_cabi.Moe)
    assert header_constants("B200AWQ_OP_SPARSE_MOE") == (_cabi.OP_SPARSE_MOE,)


def test_moe_op_argument_validation_without_gpu():
    ops = (_cabi.Op * 1)()
    ops[0].kind, ops[0].M, ops[0].K = _cabi.OP_SPARSE_MOE, 1, 1024
    h = ctypes.c_void_p()
    assert lib.b200awq_program_create(ops, 1, ctypes.byref(h)) == 1 and not h.value      # no descriptor
    d = _cabi.Moe()
    ops[0].weight = ctypes.addressof(d)
    assert lib.b200awq_program_create(ops, 1, ctypes.byref(h)) == 1 and not h.value      # null tensors
    assert lib.b200awq_moe_plan(8, 2, 4096, 14336, 128, 132, None) == 1


@needs_nvcc
def test_moe_kernel_register_and_spill_budget():
    """The MoE instantiation (288 threads, one CTA per SM) fits the register file and spills nothing."""
    found = entries("program.cu", r"stream_moe_kernel")
    assert len(found) == 1, found
    (regs, stack, st, ld), = found.values()
    assert regs * (32 + 32 * 8) <= 65536, f"{regs} registers x 288 threads"
    assert st == 0 and ld == 0 and stack == 0, f"spills {st} / {ld} bytes, stack {stack}"
