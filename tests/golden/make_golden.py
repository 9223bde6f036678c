"""Generate the golden fixtures in this directory FROM THE REAL REFERENCE.

Run where an upstream checkout of the reference exists (AWQ_REFERENCE_DIR, see oracle/reference.py):

    python tests/golden/make_golden.py

It imports the unmodified reference modules (casper-hansen/AutoAWQ @ 88e4c76) with an
`accelerate` stub (the reference imports accelerate at package import; it is not installed and
not on the hot path), forces the naive CPU branch of WQLinearMMFunction (gemm.py:71-77), runs the
reference code on seeded inputs and stores inputs + reference outputs as small .npz files.
Nothing here is product code; the committed vectors are what tests/test_oracle_golden.py and the
GPU parity tests compare against.
"""
import contextlib
import hashlib
import importlib.machinery
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("AWQ_REFERENCE_DIR", "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # repo root, for oracle.*

warnings.filterwarnings("ignore")


def _import_reference():
    import transformers  # noqa: F401  (must precede the stub)

    def stub(name, **kw):
        m = types.ModuleType(name)
        m.__spec__ = importlib.machinery.ModuleSpec(name, None)
        m.__path__ = []
        m.__dict__.update(kw)
        sys.modules[name] = m
        return m

    stub(
        "accelerate",
        big_modeling=stub(
            "accelerate.big_modeling",
            init_empty_weights=contextlib.nullcontext,
            load_checkpoint_and_dispatch=lambda *a, **k: None,
        ),
    )
    # The repo root is on sys.path (for oracle.*) and holds THIS repo's `awq_ext` / `awq_v2_ext` drop-in packages:
    # the reference would bind them at import (awq/utils/module.py:4-9) and its forward would then run on our CUDA
    # extension instead of its own naive CPU branch.  Goldens must come from the reference alone: mask both names
    # (a None entry makes the import raise, try_import returns None).
    sys.modules["awq_ext"] = None
    sys.modules["awq_v2_ext"] = None
    sys.path.insert(0, REF)
    import awq  # noqa: F401
    import awq.modules.linear.gemm as G
    import awq.modules.linear.gemv as V
    import awq.modules.linear.gemv_fast as F
    import awq.utils.packing_utils as P
    from awq.quantize.quantizer import AwqQuantizer

    G.TRITON_AVAILABLE = False  # CPU: reach the naive branch (gemm.py:71-77)
    G.get_best_device = lambda: "cpu"
    return G, V, F, P, AwqQuantizer


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    G, V, F, P, AwqQuantizer = _import_reference()
    from oracle import awq_oracle as O

    # ---- (1) dequantize_gemm on small cases, canonical and raw recipes --------------------
    out = {}
    cases = [(256, 64, 128), (256, 64, 64), (128, 32, 32), (256, 40, -1), (384, 72, 128)]
    meta = []
    for ci, (K, N, Gs) in enumerate(cases):
        for raw in (False, True):
            c = O.make_case(K, N, Gs, seed=100 + ci, raw=raw)
            w = P.dequantize_gemm(
                torch.from_numpy(c["qweight"]), torch.from_numpy(c["qzeros"]), torch.from_numpy(c["scales"]), 4,
                c["group_size"],
            )
            assert w.dtype == torch.float16
            tag = f"c{ci}_{'raw' if raw else 'can'}"
            out[f"{tag}_qweight"] = c["qweight"]
            out[f"{tag}_qzeros"] = c["qzeros"]
            out[f"{tag}_scales"] = c["scales"]
            out[f"{tag}_w"] = w.numpy()
            meta.append((tag, K, N, c["group_size"]))
    out["meta"] = np.array([f"{t},{k},{n},{g}" for t, k, n, g in meta])
    # known-answer word (SURVEY 8c(2)): 0x76543210 -> columns decode to 0,4,1,5,2,6,3,7
    qw = torch.full((8, 2), 0x76543210, dtype=torch.int32)
    ka = P.dequantize_gemm(qw, torch.zeros((1, 2), dtype=torch.int32), torch.ones((1, 16), dtype=torch.float16), 4, 8)
    out["known_answer_w"] = ka.numpy()
    np.savez_compressed(os.path.join(HERE, "dequant_small.npz"), **out)

    # ---- (2) the reference test's own shape (tests/test_dequantization.py), digest + rows ----
    big = {}
    for N in (1792, 4096):
        c = O.make_case(4096, N, 128, seed=0, raw=True)
        w = P.dequantize_gemm(
            torch.from_numpy(c["qweight"]), torch.from_numpy(c["qzeros"]), torch.from_numpy(c["scales"]), 4, 128
        ).numpy()
        rows = np.array([0, 1, 127, 128, 2049, 4095])
        big[f"n{N}_sha256"] = np.array(sha(w))
        big[f"n{N}_rows"] = rows
        big[f"n{N}_w_rows"] = w[rows]
        c2 = O.make_case(4096, N, 128, seed=1, raw=False)
        w2 = P.dequantize_gemm(
            torch.from_numpy(c2["qweight"]), torch.from_numpy(c2["qzeros"]), torch.from_numpy(c2["scales"]), 4, 128
        ).numpy()
        big[f"n{N}_can_sha256"] = np.array(sha(w2))
    np.savez_compressed(os.path.join(HERE, "dequant_ref_shape.npz"), **big)

    # ---- (3) packers: from_linear of the three module classes on a pseudo-quantised Linear ----
    pk = {}
    torch.manual_seed(7)
    for tag, (K, N, Gs) in {"a": (256, 64, 64), "b": (1024, 32, 128), "c": (128, 96, 32)}.items():
        lin = torch.nn.Linear(K, N, bias=True)
        w = lin.weight.data.clone()
        # reference pseudo-quantiser (quantizer.py:74-109); instance not needed for this method
        q = AwqQuantizer.__new__(AwqQuantizer)
        q.w_bit, q.group_size, q.zero_point = 4, Gs, True
        wq, s, z = q.pseudo_quantize_tensor(w)
        lin.weight.data = wq.half()
        s_gn, z_gn = s.t().contiguous(), z.t().contiguous()  # [K/G, N] for GEMM (quantizer.py:236-240)
        m = G.WQLinear_GEMM.from_linear(lin, 4, Gs, False, s_gn, z_gn)
        pk[f"{tag}_weight"] = lin.weight.data.numpy()
        pk[f"{tag}_bias"] = lin.bias.data.half().numpy()
        pk[f"{tag}_scales_ng"] = s.half().numpy()
        pk[f"{tag}_zeros_ng"] = z.numpy().astype(np.uint8)
        pk[f"{tag}_gemm_qweight"] = m.qweight.numpy()
        pk[f"{tag}_gemm_qzeros"] = m.qzeros.numpy()
        pk[f"{tag}_gemm_scales"] = m.scales.numpy()
        mv = V.WQLinear_GEMV.from_linear(lin, 4, Gs, False, s, z)
        pk[f"{tag}_gemv_qweight"] = mv.qweight.numpy()
        pk[f"{tag}_gemv_qzeros"] = mv.qzeros.numpy()
        pk[f"{tag}_gemv_scales"] = mv.scales.numpy()
        if K % 64 == 0:
            mf = F.WQLinear_GEMVFast.from_linear(lin, 4, Gs, False, s, z)
            pk[f"{tag}_fast_qweight"] = mf.qweight.numpy()
            pk[f"{tag}_fast_qzeros"] = mf.qzeros.numpy()
            pk[f"{tag}_fast_scales"] = mf.scales.numpy()
        # forward through the reference module (naive CPU branch), incl. bias and 2-D/3-D inputs
        g = torch.Generator().manual_seed(11)
        for xi, shp in enumerate([(1, 1, K), (2, 3, K), (5, K)]):
            x = torch.randn(shp, generator=g, dtype=torch.float16)
            y = m(x)
            pk[f"{tag}_x{xi}"] = x.numpy()
            pk[f"{tag}_y{xi}"] = y.numpy()
        pk[f"{tag}_meta"] = np.array([K, N, Gs])
    # zeros-width table (gemv.py:12-24)
    zw_in = [(4096, 128), (14336, 128), (8192, 128), (28672, 128), (4096, 64), (4096, 32), (256, 32), (11008, 128), (5120, 64)]
    pk["zw_in"] = np.array(zw_in)
    pk["zw_out"] = np.array([V.calculate_zeros_width(k, g) for k, g in zw_in])
    np.savez_compressed(os.path.join(HERE, "packers.npz"), **pk)

    # ---- (4) fuse_qkv-style concatenation along N (fused_utils.py:87-96) is format preserving --
    # (property checked in tests from the oracle; nothing to store)
    print("golden fixtures written:", [f for f in os.listdir(HERE) if f.endswith(".npz")])


if __name__ == "__main__":
    main()
