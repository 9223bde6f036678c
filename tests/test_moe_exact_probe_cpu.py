"""The exact MoE probes (oracle/exact_probe.py: make_exact_moe_case, moe_weights, moe_expected) checked without a GPU:
the plan's limits and coverage for every case of tests/test_gpu_moe_program_exact.py, the designed routing against the
routing oracles the other MoE tests hold the kernels to, the SiLU arithmetic the construction relies on, and a fault
table: every injected index fault changes a buffer the exact check compares."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import exact_probe as X
from test_gpu_moe_program_exact import CASES, M2_CASES, SEED
from test_gpu_program_qwen3moe import _routing_oracle
from test_program_deepseek_moe_cpu import route_oracle


@pytest.mark.parametrize("name", list(CASES))
def test_limits_and_coverage_of_every_gpu_case(name):
    kw, _ = CASES[name]
    c = X.make_exact_moe_case(seed=SEED, **kw)          # asserts the plan's limits and coverage itself
    E, k = c["E"], c["top_k"]
    assert c["cov_gu"].all() and c["cov_dn"].all()
    assert (c["slot_hits"].sum(axis=1) > 0).all(), "an expert is never selected"
    first, last = (E - 1, 0) if c["order"] == "descending" else (0, E - 1)
    assert c["slot_hits"][first, 0] > 0 and c["slot_hits"][last, k - 1] > 0
    # every down run turns on one class; every up run turns none on
    ctl_x = c["x_units"][:, c["ctl_rows"]]
    assert (ctl_x[c["kind"] == 0] == 0).all() and (ctl_x[c["kind"] == 1].sum(axis=1) == 1).all()
    assert c["runs"] < 20000
    if name in M2_CASES:
        assert c["runs"] >= 2


def _routing_cases():
    for name in ("mixtral-8x7b", "mixtral-8x7b-no-renorm", "sparse-E64", "qwen3-30b-a3b", "qwen3-E96", "qwen3-G64",
                 "deepseek-v2-lite", "deepseek-v3-style-E128", "deepseek-v3-style-E128-descending", "deepseek-v3"):
        yield name


@pytest.mark.parametrize("name", list(_routing_cases()))
def test_designed_routing_is_what_the_oracles_pick(name):
    kw, _ = CASES[name]
    c = X.make_exact_moe_case(seed=SEED, **kw)
    rng = np.random.default_rng(0)
    runs = np.concatenate([np.flatnonzero(c["kind"] == 0)[:3], np.flatnonzero(c["kind"] == 1)[:3],
                           rng.choice(c["runs"], size=6, replace=False)])
    k = c["top_k"]
    for r in runs:
        logits = (X.MOE_LOGIT * c["x_units"][r, c["route_rows"]]).astype(np.float32)
        want_ids = c["ids"][r]
        if c["op"] == "sparse":
            w, ids, _ = O.topk_softmax(logits.astype(np.float16).astype(np.float32)[None], k)
            w = w[0]
            if c["renormalize"]:
                w = (w.astype(np.float64) / w.astype(np.float64).sum()).astype(np.float32)
            ids = ids[0]
        elif c["op"] == "qwen3":
            ids, w = _routing_oracle(torch.from_numpy(logits.astype(np.float16)), k, c["renormalize"])
        else:
            ids, w = route_oracle(logits, k, c["scoring"], c["bias"], c["n_group"], c["topk_group"], c["renormalize"],
                                  c["rsf"])
        assert np.array_equal(np.asarray(ids), want_ids), (name, r, ids, want_ids)
        assert (np.asarray(w, dtype=np.float64) == c["weight"]).all(), (name, r, w, c["weight"])


def test_silu_of_the_gate_values_under_the_kernels_formulas():
    f32 = np.float32
    g = f32(X.GATE_ON)
    # aux.cu / stream kernels: g / (1 + exp(-g)); torch: g * sigmoid(g); Qwen3: fp16 of that, then the product
    assert g / (f32(1) + np.exp(-g)) == g
    assert g * (f32(1) / (f32(1) + np.exp(-g))) == g
    assert np.float16(g / (f32(1) + np.exp(-g))) == np.float16(32)
    assert f32(0) / (f32(1) + np.exp(f32(0))) == 0                 # the up runs' gates
    off = f32(X.GATE_OFF)
    s_off = off / (f32(1) + np.exp(-off))
    assert s_off < 0 and np.float16(s_off) == 0
    # the largest |u| a down run makes: (top_k + 1) units; the products round to +-0 in fp16
    for k in (2, 4, 6, 8):
        u = f32((k + 1) * 2.0**-6)
        assert abs(float(s_off) * float(u)) < 2.0**-25 and np.float16(s_off * u) == 0
    assert np.float16(X.GATE_SCALE * (12 - X.GATE_ZERO)) == X.GATE_ON
    assert np.float16(X.GATE_SCALE * (0 - X.GATE_ZERO)) == X.GATE_OFF


# ------------------------------------------------------------------------------------------------ fault table
SMALL = {
    "sparse": dict(op="sparse", E=8, top_k=2, H=512, I=256, G=64),
    "qwen3": dict(op="qwen3", E=16, top_k=4, H=512, I=256, G=64),
    "deepseek": dict(op="deepseek", E=32, top_k=4, H=1024, I=256, G=64, I_s=256, scoring="sigmoid", n_group=4,
                     topk_group=2, rsf=2.5),
}
SLOT_BUFFERS = ("gate_up", "act", "down")


def _faults(c, W):
    """name -> the buffers a kernel with that fault would leave (the reference with the fault applied)."""
    E, k, H, I = c["E"], c["top_k"], c["H"], c["I"]
    e = E - 1

    def deq_with(which, ee, fn):
        def deq(w, x):
            t = X.moe_dequant(W, w, x)
            return fn(t.clone()) if (w, x) == (which, ee) else t
        return deq

    def zero_row(r):
        def fn(t):
            t[r] = 0
            return t
        return fn

    out = {
        "gate|up: last k-row dropped": dict(deq=deq_with("w1", e, zero_row(H - 1))),
        "gate|up: routing k-row dropped": dict(deq=deq_with("w1", e, zero_row(int(c["route_rows"][0])))),
        "gate|up: control k-row dropped": dict(deq=deq_with("w1", e, zero_row(int(c["ctl_rows"][-1])))),
        "down: last k-row dropped": dict(deq=deq_with("w2", e, zero_row(I - 1))),
        "down: first k-row dropped": dict(deq=deq_with("w2", 0, zero_row(0))),
        "last slot reads expert (e + 1) % E": dict(read=np.concatenate(
            [c["ids"][:, :-1], (c["ids"][:, -1:] + 1) % E], axis=1)),
        "two slots swapped": "swap",
    }
    if c["I_s"]:
        ws2 = X.moe_dequant(W, "ws2", None)

        def shared_row(t):
            t[I - 1] = ws2[I - 1]
            return t
        out["a shared-expert down row read as a routed one"] = dict(deq=deq_with("w2", e, shared_row))
    return out


def _apply(c, W, ref, f):
    if f == "swap":
        got = dict(ref)
        for n in SLOT_BUFFERS:
            t = ref[n]
            if c["op"] == "deepseek" and n != "down":
                per = (2 if n == "gate_up" else 1) * c["I"]
                t = t.clone()
                t[:, :per], t[:, per:2 * per] = ref[n][:, per:2 * per], ref[n][:, :per]
            else:
                t = t[:, [1, 0] + list(range(2, c["top_k"]))]
            got[n] = t
        return got
    return X.moe_expected(c, W, **f)


def _tolerance_sees(c, W, ref, got):
    """The bar of the tolerance-based MoE tests: per stage 2^-10 |ref| + 2^-11 (|x| . |W|) (+ 1e-6), and on the block
    output 0.02 rms + 2e-3 (tests/test_gpu_program_moe.py)."""
    x = torch.as_tensor(c["x_units"]).double()
    k, I = c["top_k"], c["I"]
    ids = torch.as_tensor(c["ids"].astype(np.int64))
    act = ref["act"].double()
    if c["op"] == "deepseek":
        act = act[:, :k * I].reshape(-1, k, I)
    seen = False
    for n in ("gate_up", "down"):
        a, b = got[n].double(), ref[n].double()
        if c["op"] == "deepseek" and n == "gate_up":
            a, b = a[:, :k * 2 * I].reshape(-1, k, 2 * I), b[:, :k * 2 * I].reshape(-1, k, 2 * I)
        budget = torch.zeros_like(b)
        for e in range(c["E"]):
            rr, ss = torch.nonzero(ids == e, as_tuple=True)
            if n == "gate_up":
                budget[rr, ss] = x[rr].abs() @ X.moe_dequant(W, "w1", e).abs()
            else:
                budget[rr, ss] = act[rr, ss].abs() @ X.moe_dequant(W, "w2", e).abs() * abs(c["weight"])
        seen |= bool(((a - b).abs() > 2.0**-10 * b.abs() + 2.0**-11 * budget + 1e-6).any())
    o, r = got["out"].double(), ref["out"].double()
    rms = r.pow(2).mean(dim=-1, keepdim=True).sqrt()
    seen |= bool(((o - r).abs() > 0.02 * rms + 2e-3).any())
    return seen


@pytest.mark.parametrize("op", list(SMALL))
def test_exact_check_flags_every_injected_fault(op):
    c = X.make_exact_moe_case(seed=5, **SMALL[op])
    W = X.moe_weights(c, "cpu")
    ref = X.moe_expected(c, W)
    missed_by_tolerance = []
    for name, f in _faults(c, W).items():
        got = _apply(c, W, ref, f)
        differs = [n for n in ref if not torch.equal(got[n].double(), ref[n].double())]
        assert differs, f"{op}: '{name}' goes unnoticed by the exact check"
        if not _tolerance_sees(c, W, ref, got):
            missed_by_tolerance.append(name)
    # a wrong expert or swapped slots move whole rows: the tolerance bars see them too.  Which single-k-row faults they
    # let through depends on the data (on the probe's sparse integers they happen to show; on the random rows of the
    # tolerance tests a k-row moves outputs by far less than 2^-11 |x| . |W|, tests/test_exact_probe_cpu.py)
    assert "last slot reads expert (e + 1) % E" not in missed_by_tolerance
    assert "two slots swapped" not in missed_by_tolerance


def test_packing_matches_the_oracle_and_the_design():
    c = X.make_exact_moe_case(seed=2, **SMALL["deepseek"])
    W = X.moe_weights(c, "cpu")
    q, s, z = (t[3] for t in W["w1"])
    iw = X.unpack_words_torch(q).numpy().astype(np.uint8)
    iz = X.unpack_words_torch(z).numpy().astype(np.uint8)
    qq, zz = O.pack_gemm(iw, iz)
    assert np.array_equal(qq, q.numpy()) and np.array_equal(zz, z.numpy())
    w = X.moe_dequant(W, "w1", 3)
    I = c["I"]
    gate = w[:, :I]
    ctl = torch.as_tensor(c["ctl_rows"])
    assert (gate[ctl] != 0).all() and gate.abs().sum() == gate[ctl].abs().sum()        # zero off the control rows
    on = torch.as_tensor(c["classes"])[None, :] == torch.arange(c["m"])[:, None]
    assert torch.equal(gate[ctl], torch.where(on, X.GATE_ON, X.GATE_OFF).double())
    assert torch.equal(w[ctl, I:].abs() / c["unit"], torch.ones((ctl.numel(), I), dtype=torch.float64))
    route = w[torch.as_tensor(c["route_rows"]), I:].abs() / c["unit"]
    rc = torch.as_tensor(c["route_cols"])
    assert (route[:, rc] == 1).all() and route.sum() == route[:, rc].sum()
    # distinct experts
    assert not torch.equal(X.moe_dequant(W, "w1", 0), X.moe_dequant(W, "w1", 1))
    assert not torch.equal(X.moe_dequant(W, "w2", 0), X.moe_dequant(W, "w2", 1))
