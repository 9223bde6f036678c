"""Test / bench infrastructure: a copy of the unmodified upstream AutoAWQ package under oracle/_ref/.

The drop-in tests (tests/test_gpu_reference_dropin.py) run the reference's own module classes on top of this
repository's `awq_ext`, and bench.py times the reference's Triton kernels on the same tensors; both read
oracle/_ref/awq and nothing else of the upstream tree.  The reference is pure Python, so the copy is the whole
"build": `install()` copies the `awq` package of an upstream checkout (AWQ_REFERENCE_DIR, default /root/reference)
when one is present.  oracle/_ref/ is git-ignored; the product never imports it.
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
MARKER = os.path.join("awq", "modules", "linear", "gemm.py")


def source_dir():
    return os.environ.get("AWQ_REFERENCE_DIR", "/root/reference")


def install() -> str:
    """Copies the upstream `awq` package to oracle/_ref/awq once; returns oracle/_ref, or "" without a copy."""
    if os.path.isfile(os.path.join(DST, MARKER)):
        return DST
    src = source_dir()
    if not os.path.isfile(os.path.join(src, MARKER)):
        return ""
    tmp = DST + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(os.path.join(src, "awq"), os.path.join(tmp, "awq"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    for root, dirs, files in os.walk(tmp):   # the upstream tree may be read-only; the copy must stay removable
        for n in dirs + files:
            os.chmod(os.path.join(root, n), 0o755 if n in dirs else 0o644)
    os.replace(tmp, DST)
    return DST
