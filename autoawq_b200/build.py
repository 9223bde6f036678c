"""In-tree build of libb200awq.so (nvcc, sm_90a only) and of the C oracle (gcc).  No JIT cache:
the .so lands in autoawq_b200/lib/ so it travels to the GPU box with the snapshot."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libb200awq.so")
SOURCES = ["cabi.cu", "dequant.cu", "gemv.cu", "gemm_tc.cu", "aux.cu", "program.cu", "moe.cu", "comm.cu"]
HEADERS = ["common.cuh", "gemv_tile.cuh", "program_stream.cuh", "program_stream_body.inc", "program_batch.cuh", "program_batch_body.inc", "rope.cuh", "layernorm.cuh", "kernels.h", os.path.join(ROOT, "include", "b200awq.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _digest(paths, extra: str = "") -> str:
    """Content hash of the sources + flags: the rebuild decision does not depend on file times (a checkout or a
    copy to another box resets them)."""
    import hashlib

    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build_lib(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    stamp = LIB + ".sha256"
    want = _digest(deps, " ".join(NVCC_FLAGS))
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == want:
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        if os.path.exists(LIB):   # a box without the toolkit (never this image): keep the shipped library
            return LIB
        raise RuntimeError("nvcc not found: cannot build libb200awq.so (and there is no fallback path)")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + srcs
    subprocess.run(cmd, check=True, cwd=CSRC)
    with open(stamp, "w") as f:
        f.write(want)
    return LIB


def build_oracle(force: bool = False) -> str:
    odir = os.path.join(ROOT, "oracle")
    out = os.path.join(odir, "_build", "libawqoracle.so")
    src = os.path.join(odir, "awq_oracle.c")
    if force or _newer(out, [src]):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["gcc", "-O2", "-fopenmp", "-fPIC", "-shared", "-o", out, src, "-lm"], check=True)
    return out


if __name__ == "__main__":
    print(build_lib(force=True, verbose=False))
    print(build_oracle(force=True))
