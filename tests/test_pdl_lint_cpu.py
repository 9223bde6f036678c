"""Static check (no GPU): every kernel that may be launched with the programmatic-dependent-launch attribute (everything
that goes through launch_kernel(), kernels.h) must execute griddepcontrol.wait - pdl_wait() - in its body, and the grouped
(MoE) persistent GEMV must do so BEFORE it reads the routing tables.  The GPU tests never set knob 4, so a kernel that
forgets the wait passes them and only misbehaves in the bench (that is how the grouped GEMV's race was found: round 2)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autoawq_b200", "csrc")
# launched with <<<>>> or the cooperative attribute only (plain stream order), never with the PDL attribute
EXEMPT = {"stream_pack_kernel", "oneshot_allreduce_kernel", "ll_allreduce_kernel", "stream_program_kernel"}


def _kernels(path):
    src = open(path).read()
    out = {}
    for m in re.finditer(r"__global__\s+void\s+", src):
        p = m.end()
        if src.startswith("__launch_bounds__", p):       # skip the (possibly nested) argument list
            p = src.index("(", p)
            depth = 1
            p += 1
            while depth:
                depth += {"(": 1, ")": -1}.get(src[p], 0)
                p += 1
        nm = re.match(r"\s*(\w+)\s*\(", src[p:])
        if nm is None:
            continue
        name, i = nm.group(1), src.index("{", p + nm.end())
        depth, j = 1, i + 1
        while depth:
            depth += {"{": 1, "}": -1}.get(src[j], 0)
            j += 1
        out[name] = src[i:j]
    return out


def test_every_pdl_launchable_kernel_waits():
    seen = 0
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cu", ".cuh")):
            continue
        for name, body in _kernels(os.path.join(CSRC, f)).items():
            if name in EXEMPT:
                continue
            seen += 1
            assert "pdl_wait()" in body, f"{f}: {name} can be launched with the PDL attribute but never waits"
    assert seen >= 10, "kernel parser found too few kernels"


def test_grouped_gemv_waits_before_reading_routing_tables():
    body = _kernels(os.path.join(CSRC, "gemv.cu"))["gemv_v3_kernel"]
    first_wait = body.index("pdl_wait()")
    for field in ("moe.num_post_pad", "moe.sorted_ids", "moe.expert_ids"):
        assert first_wait < body.index(field), f"gemv_v3_kernel reads {field} before griddepcontrol.wait"


def test_moe_kernels_wait_first():
    k = _kernels(os.path.join(CSRC, "moe.cu"))
    for name in ("topk_softmax_kernel", "moe_align_kernel", "moe_grouped_kernel"):
        body = k[name]
        w = body.index("pdl_wait()")
        # nothing but declarations / index arithmetic before the wait: no global-memory read (no '[' dereference of a
        # kernel pointer argument) in front of it
        assert "__ldg" not in body[:w] and "ld_" not in body[:w], f"{name} loads before the wait"
