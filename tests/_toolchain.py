"""Compiler-side checks the CPU tests share, without a GPU: each kernel source is compiled once per process with the
library's own flags (ptxas report, SASS), and include/b200awq.h is read through gcc (struct layouts, constants).

Every result is cached for the process, so a session compiles program.cu once however many budget tests read it."""
import ctypes
import functools
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from autoawq_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")

_HOST_ONLY = ("-Xcompiler", "-fPIC", "-shared")     # flags of the shared-library link, not of the device code
_TMP = tempfile.TemporaryDirectory(prefix="b200awq-tests-")      # removed at interpreter exit


@functools.lru_cache(maxsize=None)
def ptxas_report(source):
    """Compiles autoawq_b200/csrc/<source> to an object with the library's flags and `-Xptxas -v`.  Returns
    ({mangled entry name: (registers, stack frame, spill stores, spill loads)}, object path)."""
    obj = os.path.join(_TMP.name, os.path.splitext(source)[0] + ".o")
    flags = [f for f in build.NVCC_FLAGS if f not in _HOST_ONLY]
    out = subprocess.run([NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, source), "-o", obj],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    frames, regs, entry, props = {}, {}, None, None
    for line in (out.stderr + out.stdout).splitlines():
        if m := re.search(r"Compiling entry function '(\S+)'", line):
            entry = m.group(1)
        elif m := re.search(r"Function properties for (\S+)", line):
            props = m.group(1)
        elif m := re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line):
            frames[props] = tuple(int(v) for v in m.groups())
        elif (m := re.search(r"Used (\d+) registers", line)) and entry is not None:
            regs[entry] = int(m.group(1))
            entry = None
    return {name: (r,) + frames[name] for name, r in regs.items()}, obj


def entries(source, pattern):
    """ptxas_report's entries of `source` whose mangled name matches the regex `pattern`."""
    return {name: v for name, v in ptxas_report(source)[0].items() if re.search(pattern, name)}


@functools.lru_cache(maxsize=None)
def _sass_functions(source):
    from tools.sass_unchanged import _functions

    return _functions(ptxas_report(source)[1])


def sass(source, entry):
    """The SASS of the one kernel of `source` whose mangled name contains `entry` (tools/sass_unchanged.py's text)."""
    found = [body for name, body in _sass_functions(source).items() if entry in name]
    assert len(found) == 1, (entry, len(found))
    return found[0]


@functools.lru_cache(maxsize=None)
def _compare(base):
    from tools.sass_unchanged import compare

    return compare(base)


def sass_compare(only=None):
    """tools/sass_unchanged.compare against the revision in B200AWQ_SASS_BASE (computed once per revision), restricted
    to the entries whose names contain one of `only`.  Skips when the variable is unset or names no commit here."""
    base = os.environ.get("B200AWQ_SASS_BASE")
    if not base:
        pytest.skip("set B200AWQ_SASS_BASE to a git revision to compare against")
    if shutil.which("git") is None or subprocess.run(["git", "-C", ROOT, "cat-file", "-e", base + "^{commit}"],
                                                     capture_output=True).returncode != 0:
        pytest.skip(f"{base} is not a commit of this checkout")
    return {n: same for n, same in _compare(base).items() if not only or any(s in n for s in only)}


def _gcc_print(body):
    """Compiles and runs a C program printing integers from include/b200awq.h; returns them."""
    d = tempfile.mkdtemp(dir=_TMP.name)
    src, exe = os.path.join(d, "probe.c"), os.path.join(d, "probe")
    with open(src, "w") as f:
        f.write('#include <stdio.h>\n#include <stddef.h>\n#include "b200awq.h"\nint main(void) {\n' + body +
                "  return 0;\n}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
    return [int(v) for v in subprocess.check_output([exe]).split()]


def mirror_layout(ctype):
    """{"sizeof": size, field: offset} of a ctypes structure, every field."""
    return {"sizeof": ctypes.sizeof(ctype), **{f: getattr(ctype, f).offset for f, _ in ctype._fields_}}


@functools.lru_cache(maxsize=None)
def header_layout(ctype, c_name):
    """gcc's {"sizeof": size, field: offset} of the C struct `c_name`, for every field of its ctypes mirror `ctype`."""
    fields = [f for f, _ in ctype._fields_]
    got = _gcc_print(f'  printf("%zu\\n", sizeof({c_name}));\n' +
                     "".join(f'  printf("%zu\\n", offsetof({c_name}, {f}));\n' for f in fields))
    return dict(zip(["sizeof"] + fields, got))


@functools.lru_cache(maxsize=None)
def header_constants(*names):
    """The values of integer constants of include/b200awq.h (enumerators, macros), in the order named."""
    return tuple(_gcc_print("".join(f'  printf("%lld\\n", (long long)({n}));\n' for n in names)))
