#!/usr/bin/env python3
"""Checks that every kernel of an older libgsb200.so is still in a newer one, instruction for instruction.

    python tools/sass_diff.py OLD/libgsb200.so NEW/libgsb200.so

Runs `cuobjdump -sass` on both and compares each function's instructions and encodings (addresses are function-relative,
so a kernel that kept its code compares equal wherever it now lies).  A kernel that gained a defaulted template parameter
has a new mangled name; it is matched by demangled name with the trailing default arguments removed, and otherwise by an
identical body.  Prints one line per old kernel that has no identical counterpart and exits 1 if there is any.  Needs no GPU.
"""
from __future__ import annotations

import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def functions(lib):
    """{mangled name: tuple of instruction lines (text and encodings, addresses dropped)}"""
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = tuple(body)
            name, body = m.group(1), []
            continue
        if name is None:
            continue
        if "/* 0x" not in line:  # labels, directives and the next section's header
            continue
        line = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip()  # the instruction's address
        body.append(line)
    if name:
        funcs[name] = tuple(body)
    return funcs


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, r.stdout.splitlines()))


def canonical(d):
    """The demangled name without trailing `, false` template arguments and without the parameter list."""
    d = d.replace("(anonymous namespace)", "").split("(")[0]
    while True:
        e = re.sub(r", false>$", ">", d)
        if e == d:
            return d
        d = e


def main(old_lib, new_lib):
    old, new = functions(old_lib), functions(new_lib)
    dm = demangle(list(old) + list(new))
    by_name = {}
    for k in new:
        by_name.setdefault(canonical(dm[k]), []).append(k)
    bodies = {}
    for k, b in new.items():
        bodies.setdefault(b, []).append(k)
    bad = 0
    for k, b in old.items():
        cands = by_name.get(canonical(dm[k]), [])
        if any(new[c] == b for c in cands):
            continue
        if b in bodies:
            print(f"moved name : {dm[k]} -> {dm[bodies[b][0]]}")
            continue
        bad += 1
        print(f"CHANGED    : {dm[k]}")
    print(f"{len(old)} kernels in {old_lib}, {len(new)} in {new_lib}: {len(old) - bad} identical, {bad} changed")
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
