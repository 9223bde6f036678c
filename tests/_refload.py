"""Test-only loader of the UNMODIFIED reference package (casper-hansen/AutoAWQ @ 88e4c76).

Where it comes from: `oracle/_ref/awq` - a copy of the upstream package made by `__graft_entry__.build()`
(`oracle/reference.py`; git-ignored, it travels with the built tree like the compiled libraries).  Nothing of it is
in the repository's history and no product code imports this.

Two modes:
  * `load_reference(shim=True)`  - the repo root goes on sys.path FIRST, so the reference's
    `try_import("awq_ext")` (awq/utils/module.py:4-9, bound at awq/modules/linear/gemm.py:11,
    gemv.py:6, gemv_fast.py:5, fused/norm.py:5) binds THIS repo's `awq_ext` / `awq_v2_ext`: the
    reference's own module classes then run on this repository's kernels - the drop-in, exercised for real.
  * `load_reference(shim=False)` - `awq_ext` / `awq_v2_ext` are masked (sys.modules[name] = None makes
    the import raise, try_import returns None): the reference falls back to its Triton kernels on a
    GPU (gemm.py:60-69) or, with TRITON_AVAILABLE forced off, to its naive CPU branch (gemm.py:71-77).
    This is the "kernel to beat" leg and the golden-vector generator's mode.
The two modes cannot coexist in one interpreter (the binding happens at import): tests that need the
other mode run in a subprocess.

`accelerate` is not installed in this image and is imported at package import time
(awq/utils/utils.py:4, awq/models/base.py:42-45); it is not on the hot path, so a stub stands in.
"""
import contextlib
import importlib
import importlib.machinery
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CANDIDATES = [os.path.join(ROOT, "oracle", "_ref")]


def reference_root():
    for c in CANDIDATES:
        if os.path.isfile(os.path.join(c, "awq", "modules", "linear", "gemm.py")):
            return c
    return None


def _stub(name, **kw):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__path__ = []
    m.__dict__.update(kw)
    sys.modules[name] = m
    return m


def stub_accelerate(dispatch=None):
    """A stand-in for `accelerate` with the two names the reference's loader uses
    (awq/models/base.py:497,527): `init_empty_weights` and `load_checkpoint_and_dispatch`."""
    import transformers  # noqa: F401  (its availability probes must run before the stub exists)

    if "accelerate" in sys.modules and getattr(sys.modules["accelerate"], "__b200_stub__", False):
        if dispatch is not None:
            sys.modules["accelerate.big_modeling"].load_checkpoint_and_dispatch = dispatch
        return
    try:
        import accelerate  # noqa: F401  (a real install wins)
        return
    except Exception:  # noqa: BLE001
        pass

    @contextlib.contextmanager
    def init_empty_weights(include_buffers=False):
        import torch

        with torch.device("meta"):
            yield

    big = _stub("accelerate.big_modeling", init_empty_weights=init_empty_weights,
                load_checkpoint_and_dispatch=dispatch or (lambda *a, **k: None))
    acc = _stub("accelerate", big_modeling=big, init_empty_weights=init_empty_weights)
    acc.__b200_stub__ = True
    _stub("accelerate.utils", get_balanced_memory=lambda *a, **k: None)


def load_reference(shim=True):
    """Imports the reference package and returns it (None when no copy of the reference is reachable)."""
    ref = reference_root()
    if ref is None:
        return None
    if "awq" in sys.modules:
        return sys.modules["awq"]
    stub_accelerate()
    if shim:
        if ROOT not in sys.path:
            sys.path.insert(0, ROOT)
        import awq_ext  # noqa: F401  (this repo's; must be importable before the reference binds it)
        import awq_v2_ext  # noqa: F401
    else:
        sys.modules["awq_ext"] = None
        sys.modules["awq_v2_ext"] = None
    if ref not in sys.path:
        sys.path.append(ref)          # after the repo root: the repo's awq_ext wins, `awq` exists only there
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        awq = importlib.import_module("awq")
    return awq
