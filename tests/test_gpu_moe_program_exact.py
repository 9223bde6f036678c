"""Exact-arithmetic probes of the MoE decode-program ops (DecodeProgram.sparse_moe, .qwen3_moe, .deepseek_moe) and of
their per-op replays (oracle/exact_probe.py: make_exact_moe_case; DESIGN.md section 4).

The test chooses the routing (one-hot router rows), every gate is 0, +32 or -64 so that SiLU * mul is exact, and the
weights and activations are integers times powers of two sized so that gate|up, act, every per-slot down output and
the shared expert's are fp16 values.  Over the runs of a plan every expert is selected, every (expert, k-row) pair of
gate|up and of down meets a non-zero activation, and expert 0 / E - 1 take the first / last slot.  Every buffer of every
run is compared for equality with the exact reference (moe_expected): the recorded routing, gate|up and act slot by
slot through the recorded ids, the per-slot c, out and y_s.  A wrong expert address, a dropped or repeated k-row of
either expert op, a swapped slot or a shared row read as a routed one changes at least one compared value; the failure
names the run, the slot and the columns.

Each case runs fused when the plan allows it (asserted, with no abort record) and again as the per-op replay (knob 14 =
1), which must be exact too and equal to the fused buffers; M = 2 runs the per-op replay on two tokens per step."""
import ctypes

import numpy as np
import pytest
import torch

from autoawq_b200 import ext
from autoawq_b200._cabi import lib
from autoawq_b200.program import DecodeProgram
from oracle import exact_probe as X
from test_gpu_program import _no_abort

pytestmark = pytest.mark.gpu

SEED = 11
BATCH = 4096          # runs per reference batch

MIXTRAL = dict(op="sparse", E=8, top_k=2, H=4096, I=14336, G=128)
V3_GROUPS = dict(op="deepseek", E=128, top_k=8, H=2048, I=768, G=128, I_s=768, scoring="sigmoid", n_group=8,
                 topk_group=4, rsf=2.5)
# id -> (plan arguments, fused: True / False / "plan" (whatever b200awq_qwen3_moe_plan says on this device))
CASES = {
    "mixtral-8x7b": (dict(MIXTRAL, renormalize=True), True),
    "mixtral-8x7b-no-renorm": (dict(MIXTRAL, renormalize=False), True),
    "sparse-E64": (dict(op="sparse", E=64, top_k=8, H=1024, I=512, G=128), True),
    "qwen3-30b-a3b": (dict(op="qwen3", E=128, top_k=8, H=2048, I=768, G=128), True),
    "qwen3-235b-a22b": (dict(op="qwen3", E=128, top_k=8, H=4096, I=1536, G=128), "plan"),
    "qwen3-E96": (dict(op="qwen3", E=96, top_k=8, H=2048, I=768, G=128), True),
    "qwen3-G64": (dict(op="qwen3", E=64, top_k=4, H=1024, I=512, G=64), True),
    "deepseek-v2-lite": (dict(op="deepseek", E=64, top_k=6, H=2048, I=1408, G=128, I_s=2816, renormalize=False), True),
    "deepseek-v3-style-E128": (dict(V3_GROUPS, renormalize=True), True),
    "deepseek-v3-style-E128-descending": (dict(V3_GROUPS, renormalize=True, order="descending"), True),
    "deepseek-v3": (dict(op="deepseek", E=256, top_k=8, H=7168, I=2048, G=128, I_s=2048, scoring="sigmoid",
                         n_group=8, topk_group=4, rsf=2.5, renormalize=True), False),
}
M2_CASES = ["sparse-E64", "qwen3-G64", "deepseek-v3-style-E128"]


def _dev():
    return torch.device("cuda:0")


_W = {}


def _case(name):
    """The plan and the block's tensors.  The weights depend only on the sizes, the seed and the reserved coordinates,
    so the cases that differ in renormalisation, scaling or slot order share them (one block is kept at a time)."""
    kw, fused = CASES[name]
    c = X.make_exact_moe_case(seed=SEED, **kw)
    key = tuple(c[k] for k in ("op", "E", "top_k", "H", "I", "G", "I_s", "n_group", "topk_group"))
    if key not in _W:
        _W.clear()
        torch.cuda.empty_cache()
        _W[key] = X.moe_weights(c, _dev())
    W = dict(_W[key], bias=torch.as_tensor(c["bias"], device=_dev()))
    if fused == "plan":
        plan = (ctypes.c_int * 8)()
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        fused = lib.b200awq_qwen3_moe_plan(c["E"], c["top_k"], c["H"], c["I"], c["G"], sms, plan) == 0
    return c, W, fused


def _record(prog, c, W, x):
    op = c["op"]
    if op == "sparse":
        return prog.sparse_moe(x, W["gate"], W["w1"], W["w2"], c["top_k"], c["renormalize"])
    if op == "qwen3":
        return prog.qwen3_moe(x, W["gate"], W["w1"], W["w2"], c["top_k"], c["renormalize"])
    return prog.deepseek_moe(x, W["gate"], W["w1"], W["w2"], c["top_k"], (W["ws1"], W["ws2"]), c["scoring"],
                             e_score_correction_bias=W["bias"] if c["scoring"] == "sigmoid" else None,
                             n_group=c["n_group"], topk_group=c["topk_group"], norm_topk_prob=c["renormalize"],
                             routed_scaling_factor=c["rsf"])


NAMES = ("logits", "topk_weights", "topk_ids", "gate_up", "act", "down", "out")


def _run_plan(c, W, M, replay):
    """Every run of the plan through one program (M tokens per step: runs r, r + 1, ...), the buffers of each step
    stacked by run.  Returns (program, {name: [R, ...]})."""
    prev = ext.get_knob(14)
    ext.set_knob(14, 1 if replay else 0)
    try:
        prog = DecodeProgram()
        xb = torch.zeros((M, c["H"]), dtype=torch.float16, device=_dev())
        _record(prog, c, W, xb)
        prog.build()
    finally:
        ext.set_knob(14, prev)
    R = c["runs"]
    order = np.concatenate([np.arange(R), np.arange((-R) % M)])           # the last step is filled up with run 0, ..
    xs = torch.as_tensor(c["x_units"], device=_dev()).half()
    b = prog.moe_buffers(0)
    names = NAMES + (("shared_out",) if c["I_s"] else ())
    rec = {n: torch.empty((R,) + tuple(b[n].shape[1:]), dtype=b[n].dtype, device=_dev()) for n in names}
    for s in range(0, R, M):
        xb.copy_(xs[torch.as_tensor(order[s:s + M], device=_dev())])
        prog.run()
        n_real = min(M, R - s)
        for n in names:
            rec[n][s:s + n_real].copy_(b[n][:n_real])
    torch.cuda.synchronize()
    return prog, rec


def _compare(got, want, c, what, run0):
    if got.dtype == torch.int32:
        ok = torch.equal(got, want)
    else:
        ok = bool((got.double() == want.double()).all())
    if ok:
        return
    g, w = got.double().cpu().numpy(), want.double().cpu().numpy()
    if g.ndim == 3:         # [runs, slots, N]: one report row per (run, slot)
        rows = np.argwhere((g != w).any(axis=2))[:4]
        where = ", ".join(f"run {run0 + r} slot {s} (expert {c['ids'][run0 + r, s]})" for r, s in rows)
        g, w = g.reshape(-1, g.shape[2]), w.reshape(-1, w.shape[2])
        raise AssertionError(f"{what}: {where}; (row = run * top_k + slot) "
                             + X.mismatch_report(g, w, 1.0))
    g, w = g.reshape(g.shape[0], -1), w.reshape(w.shape[0], -1)
    span = f" (slot = column // {2 * c['I'] if 'gate' in what else c['I']} for the routed columns)" \
        if c["op"] == "deepseek" and ("gate_up" in what or "act" in what) else ""
    raise AssertionError(f"{what}: rows are runs from {run0}{span}: " + X.mismatch_report(g, w, 1.0))


def _check_exact(c, W, rec, tag, ordered):
    """Every stacked buffer against moe_expected, in reference batches.  ordered: the op's documented slot order
    (ties to the lower id, or the bias order) is asserted; otherwise the recorded ids must be the designed selection
    in any order, and the reference follows them."""
    R = c["runs"]
    ids = rec["topk_ids"].cpu().numpy()
    if ordered:
        _compare(rec["topk_ids"], torch.as_tensor(c["ids"], device=_dev()), c, f"{tag}: topk_ids", 0)
        cc = c
    else:
        assert (np.sort(ids, axis=1) == np.sort(c["ids"], axis=1)).all(), f"{tag}: routed experts differ from the plan"
        cc = dict(c, ids=ids)
    for r0 in range(0, R, BATCH):
        runs = np.arange(r0, min(R, r0 + BATCH))
        want = X.moe_expected(cc, W, runs=runs)
        for n in rec:
            if n == "topk_ids":
                continue
            _compare(rec[n][runs[0]:runs[-1] + 1], want[n], cc, f"{tag}: {n}", r0)
        del want


@pytest.mark.parametrize("name", list(CASES))
def test_moe_program_exact(name):
    c, W, fused = _case(name)
    tag = f"{name} ({c['runs']} runs)"
    if fused:
        prog, rec = _run_plan(c, W, 1, replay=False)
        assert prog.fused and prog.kernel_ops == 2, f"{tag}: fused={prog.fused} kernel_ops={prog.kernel_ops}"
        _no_abort(tag)
        _check_exact(c, W, rec, tag + " fused", ordered=True)
    rep, rrec = _run_plan(c, W, 1, replay=True)
    assert not rep.fused and rep.kernel_ops == 0
    # topk_softmax (sparse / qwen3 replays) breaks ties to the lower id; torch.topk (deepseek) documents no order
    _check_exact(c, W, rrec, tag + " per-op replay", ordered=c["op"] != "deepseek")
    if fused:
        for n in rec:
            if c["op"] == "deepseek" and n in ("topk_ids", "gate_up", "act", "down"):
                continue        # slot order may differ; both were held to the reference slot by slot above
            assert torch.equal(rec[n], rrec[n]), f"{tag}: fused and per-op replay differ in {n}"
    rep.close()
    if fused:
        prog.close()


@pytest.mark.parametrize("name", M2_CASES)
def test_moe_program_exact_two_tokens(name):
    c, W, _ = _case(name)
    rep, rec = _run_plan(c, W, 2, replay=False)         # max_tokens = 1: two rows replay per op
    assert not rep.fused
    _check_exact(c, W, rec, f"{name} M=2 per-op", ordered=c["op"] != "deepseek")
    rep.close()
