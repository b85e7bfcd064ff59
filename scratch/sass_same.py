#!/usr/bin/env python
"""Is the SASS of the serve kernels the same as at a git ref?   python scratch/sass_same.py [REF] [tu.cu ...]

"This feature must not touch that kernel" as a check that needs no GPU: the named translation units are compiled from the
working tree and from REF (default HEAD) with the build's flags, and their `cuobjdump -sass` instruction streams (opcodes,
registers, immediates — addresses and encodings stripped) are compared.
"""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gofr_b200 import _build  # noqa: E402


def sass(src_root: str, tu: str, out: str):
    obj = out + ".o"
    subprocess.check_call(["nvcc"] + _build.NVCC_FLAGS + ["-c", "-o", obj, os.path.join(src_root, "gofr_b200", "csrc", tu)], stderr=subprocess.DEVNULL)
    text = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    ins = []
    for ln in text.splitlines():
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
        if m:
            ins.append(m.group(1).strip())
    return ins


def main():
    args = sys.argv[1:]
    ref = args[0] if args and not args[0].endswith(".cu") else "HEAD"
    tus = [a for a in args if a.endswith(".cu")] or ["serve_slots_kernel.cu", "serve_slots_wide_kernel.cu", "serve_kernel.cu"]
    rc = 0
    with tempfile.TemporaryDirectory() as td:
        old = os.path.join(td, "ref")
        os.makedirs(old)
        subprocess.check_call("git archive %s gofr_b200/csrc include | tar -x -C %s" % (ref, old), shell=True, cwd=ROOT)
        for tu in tus:
            a, b = sass(old, tu, os.path.join(td, "a_" + tu)), sass(ROOT, tu, os.path.join(td, "b_" + tu))
            same = a == b
            diff = sum(x != y for x, y in zip(a, b)) + abs(len(a) - len(b))
            print(f"{tu}: {'IDENTICAL' if same else 'DIFFERENT'} ({len(a)} vs {len(b)} instructions" + ("" if same else f", {diff} differ") + f") against {ref}")
            rc |= not same
    return rc


if __name__ == "__main__":
    sys.exit(main())
