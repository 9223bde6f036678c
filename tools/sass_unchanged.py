#!/usr/bin/env python
"""Compare the SASS of program.cu's kernel entries (encodings included) between the working tree and a git revision.

Compiles csrc/program.cu of both trees for sm_90a with the library's flags (into a temporary directory), disassembles
them with `cuobjdump -sass` and compares every kernel entry present in both, or the entries whose mangled names contain
one of --only.  Prints one line per entry and exits 1 if any compared entry differs.

    python tools/sass_unchanged.py [--base HEAD~] [--only stream_program_kernel stream_batch ...]
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo"]
SOURCES = ["autoawq_b200/csrc", "include"]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found")
    return nvcc


def _functions(obj):
    """mangled name -> SASS text (instructions with encodings, addresses and line comments stripped, runs of blanks
    collapsed: cuobjdump pads every line to the widest instruction of the whole object, so a new kernel elsewhere in
    program.cu would otherwise change the text of every entry)"""
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name is not None:
                funcs[name] = "\n".join(body)
            name, body = m.group(1), []
        elif name is not None:
            body.append(" ".join(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split()))
    if name is not None:
        funcs[name] = "\n".join(body)
    return funcs


def compare(base="HEAD~", only=None):
    """{mangled entry name: True when its SASS is identical} for the entries both trees have (filtered by `only`)."""
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory() as tmp:
        btree = os.path.join(tmp, "base")
        os.makedirs(btree)
        arch = subprocess.run(["git", "-C", ROOT, "archive", base] + SOURCES, capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", btree], input=arch, check=True)
        jobs = [subprocess.Popen([nvcc] + FLAGS + ["-c", os.path.join(tree, "autoawq_b200/csrc/program.cu"), "-o",
                                                   os.path.join(tmp, f"{tag}.o")], stderr=subprocess.PIPE)
                for tag, tree in (("base", btree), ("cur", ROOT))]
        for j in jobs:
            _, err = j.communicate()
            if j.returncode != 0:
                raise RuntimeError(err.decode()[-2000:])
        a, b = _functions(os.path.join(tmp, "base.o")), _functions(os.path.join(tmp, "cur.o"))
    names = sorted(n for n in a if n in b and (not only or any(s in n for s in only)))
    return {n: a[n] == b[n] for n in names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD~")
    ap.add_argument("--only", nargs="*", default=None)
    a = ap.parse_args()
    res = compare(a.base, a.only)
    for n, same in res.items():
        print(("unchanged " if same else "CHANGED   ") + n)
    sys.exit(0 if res and all(res.values()) else 1)


if __name__ == "__main__":
    main()
