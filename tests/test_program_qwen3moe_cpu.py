"""Host logic of QWEN3_MOE blocks in stream decode programs, checked without a GPU: b200awq_qwen3_moe_plan at Qwen3-MoE
shapes and its envelope, the folding of a trailing residual add (b200awq_program_plan), the op constant against the
header, the register / spill budget of the MoE kernel entries, the SASS of the other entries against a given revision,
a model of the grid-wide router-logit exchange (program_stream.cuh: kSpQwenEMax) and the stacked-expert loader.
The exchange model checks the protocol's design (one writer per word and run, tags that never pass a stale word); it
does not run the kernel code, which tests/test_gpu_program_qwen3moe.py covers on the GPU."""
import ctypes
import random

import pytest

from _fake_ops import add, buf, plan
from _toolchain import entries, header_constants, needs_nvcc, sass_compare
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib


def _plan(E, k, H, I, G, sms=132):
    out = (ctypes.c_int * 8)()
    return lib.b200awq_qwen3_moe_plan(E, k, H, I, G, sms, out), list(out)


@pytest.mark.parametrize("H,I", [(2048, 768), (4096, 1536)])     # Qwen3-30B-A3B, Qwen3-235B-A22B
def test_plan_qwen3_moe_shapes(H, I):
    rc, p = _plan(128, 8, H, I, 128)
    assert rc == 0
    sets_a = 8 * 2 * I // 16
    assert p[:7] == [2, sets_a, (2 * I // 16) * (H // 128), -(-sets_a // 132), 8 * I // 128, I // 128,
                     -(-(H // 16) // 132) * 8]
    assert p[7] <= 227 * 1024


@pytest.mark.parametrize("args,rc", [((129, 8, 2048, 768, 128), 2), ((128, 9, 2048, 768, 128), 2),
                                     ((128, 8, 2048, 768 + 64, 128), 2),      # I % 128 != 0
                                     ((128, 8, 2048, 16384, 128), 2),         # K' = 8 x 16384: activations > smem
                                     ((0, 1, 2048, 768, 128), 1), ((4, 5, 2048, 768, 128), 1),
                                     ((128, 8, 2048, 768, 64), 0), ((65, 4, 1024, 512, 128), 0)])
def test_plan_envelope(args, rc):
    assert _plan(*args)[0] == rc


def test_sparse_moe_envelope_unchanged():
    out = (ctypes.c_int * 8)()
    assert lib.b200awq_moe_plan(65, 2, 4096, 14336, 128, 132, out) == 2
    assert lib.b200awq_moe_plan(64, 8, 512, 256, 32, 132, out) == 0


def _moe_ops(with_add, kind=None):
    """[QWEN3_MOE (+ ADD of its output and an external residual)] with placeholder addresses (the plan makes no CUDA
    call and reads no tensor)."""
    H, I, E, k = 2048, 768, 128, 8
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, H, I, 16
    d.sorted_len = k + E * 15
    d.gate_weight = buf(E * H * 2)
    d.w1_qweight, d.w1_scales, d.w1_qzeros = buf(E * H * 2 * I // 2), buf(E * H // 128 * 2 * I * 2), buf(E * 2 * I)
    d.w2_qweight, d.w2_scales, d.w2_qzeros = buf(E * I * H // 2), buf(E * I // 128 * H * 2), buf(E * H)
    for f, n in (("logits", E * 2), ("topk_weights", k * 4), ("topk_ids", k * 4), ("token_expert_indices", k * 4),
                 ("sorted_ids", d.sorted_len * 4), ("expert_ids", (k + E) * 4), ("num_tokens_post_pad", 4),
                 ("gate_up", k * 2 * I * 2), ("act", k * I * 2), ("down", k * H * 2)):
        setattr(d, f, buf(n))
    ops = [dict(kind=kind or _cabi.OP_QWEN3_MOE, M=1, K=H, N=H, x=buf(H * 2), y=buf(H * 2), weight=ctypes.addressof(d))]
    if with_add:
        ops.append(add(ops[0]["y"], buf(H * 2), H))
    return ops, d


@pytest.mark.parametrize("with_add", [False, True])
def test_trailing_add_folds_into_down(with_add):
    ops, _keep = _moe_ops(with_add)
    assert plan(ops) == (0, 2)               # gate|up with the routing, down (+ the add in its finish)


def test_op_constant_matches_header():
    assert header_constants("B200AWQ_OP_QWEN3_MOE", "B200AWQ_OP_SPARSE_MOE") == (_cabi.OP_QWEN3_MOE, _cabi.OP_SPARSE_MOE)


@needs_nvcc
def test_moe_entries_register_and_spill_budget():
    """Every MoE-instantiated M = 1 entry (288 threads, one CTA per SM) fits the register file and spills nothing."""
    names = ("stream_moe_kernel", "stream_residual_kernel", "stream_rope_kernel", "stream_qknorm_kernel",
             "stream_qwen3moe_kernel")
    for name in names:
        found = entries("program.cu", name)
        assert found, name
        regs, stack, st, ld = next(iter(found.values()))
        assert regs * (32 + 32 * 8) <= 65536 and st == 0 and ld == 0 and stack == 0, (name, regs, st, ld, stack)


@needs_nvcc
def test_plain_entries_sass_unchanged():
    """With B200AWQ_SASS_BASE set to a git revision (e.g. the commit before a change to the MoE kernels), the SASS of the
    plain and batched stream entries and the pack kernels equals that revision's (tools/sass_unchanged.py).  Unset, the
    test is skipped: which entries a change may touch is the change's own claim, not a property of the tree."""
    res = sass_compare(["stream_program_kernel", "stream_batch_", "stream_pack_kernel", "stream_pack_rotary_kernel"])
    assert res, "no entry to compare"
    assert all(res.values()), [n for n, same in res.items() if not same]


def _exchange_run(words, base, n_ops, op, E, grid, rng, value):
    """One run of one QWEN3_MOE op: CTA c publishes the logits e = c mod grid (tag << 32 | value) before it polls; the
    CTAs' steps interleave at random.  Returns what every CTA read for each expert."""
    tag = (base + op) % 65535 + 1
    pending = {c: [e for e in range(c, E, grid)] for c in range(grid)}
    seen = {c: {} for c in range(grid)}
    writers = {}
    while any(pending.values()) or any(len(s) < E for s in seen.values()):
        c = rng.randrange(grid)
        if pending[c]:                                  # publish first
            e = pending[c].pop()
            assert (e, tag) not in writers, "a word written twice in one run"
            writers[e, tag] = c
            words[op][e] = (tag, value(e))
        else:                                           # then poll one word it has not seen yet
            missing = [e for e in range(E) if e not in seen[c]]
            if not missing:
                continue
            e = rng.choice(missing)
            t, v = words[op][e]
            if t == tag:
                seen[c][e] = v
    return seen, tag


@pytest.mark.parametrize("E,grid,n_ops", [(128, 132, 2), (128, 7, 4), (96, 132, 6), (64, 16, 3)])
def test_logit_exchange_model(E, grid, n_ops):
    rng = random.Random(E * grid + n_ops)
    ops = [o for o in range(0, n_ops, 2)]               # the gate|up ops of the program's MoE blocks
    words = {o: [(0, None)] * E for o in ops}           # zero tags: never a run's (tags are >= 1)
    base, last = 0, {}
    for run in range(6):
        for o in ops:
            seen, tag = _exchange_run(words, base, n_ops, o, E, grid, rng, lambda e: (run, o, e))
            assert last.get(o) != tag, "an op's tag repeats in the next run: last run's words would pass"
            last[o] = tag
            for c in range(grid):
                assert seen[c] == {e: (run, o, e) for e in range(E)}, "a CTA read a logit of another run or op"
        assert len({(base + o) % 65535 + 1 for o in ops}) == len(ops), "two ops of one run share a tag"
        base = (base + n_ops) % 65535


def test_load_stacked_experts_matches_stack_experts(tmp_path):
    """A two-shard checkpoint of a 5-expert block: the loader's stacked tensors equal packing.stack_experts on the same
    modules."""
    import json
    import types

    import torch
    from safetensors.torch import save_file

    from autoawq_b200 import packing
    from autoawq_b200.loader import load_stacked_experts

    E, H, I, G = 5, 256, 128, 64
    gen = torch.Generator().manual_seed(0)

    def lin(K, N):
        return types.SimpleNamespace(
            qweight=torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, generator=gen),
            scales=torch.rand((K // G, N), generator=gen).half(),
            qzeros=torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, generator=gen))

    experts = [types.SimpleNamespace(gate_proj=lin(H, I), up_proj=lin(H, I), down_proj=lin(I, H)) for _ in range(E)]
    block = types.SimpleNamespace(gate=types.SimpleNamespace(weight=torch.randn(E, H).half()), experts=experts,
                                  top_k=2, norm_topk_prob=True)
    prefix = "model.layers.3.mlp"
    shards, wmap = [{}, {}], {}
    for e, ex in enumerate(experts):
        for proj in ("gate_proj", "up_proj", "down_proj"):
            for t in ("qweight", "scales", "qzeros"):
                name = f"{prefix}.experts.{e}.{proj}.{t}"
                k = (e + len(proj)) % 2                       # experts' tensors spread over both shards
                shards[k][name] = getattr(getattr(ex, proj), t)
                wmap[name] = f"model-{k}.safetensors"
    for k in range(2):
        save_file(shards[k], str(tmp_path / f"model-{k}.safetensors"))
    (tmp_path / "model.safetensors.index.json").write_text(json.dumps({"weight_map": wmap}))
    w1, w2 = load_stacked_experts(str(tmp_path), prefix, E, "cpu")
    _, r1, r2, k, norm = packing.stack_experts(block)
    assert k == 2 and norm
    for a, b in zip(w1 + w2, r1 + r2):
        assert a.dtype == b.dtype and torch.equal(a, b)
    with pytest.raises(KeyError):
        load_stacked_experts(str(tmp_path), prefix, E + 1, "cpu")
