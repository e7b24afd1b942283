"""Translate a GLSL 4.50 compute shader into C++ that runs on glsl_shim.hpp (test infrastructure only).

    python glsl_to_cpp.py <shader.comp> <namespace> <out.inc>

A generic source-to-source rewrite, run at build time on the shader files as they are; it carries no shader text of
its own.  It:
  - drops comments, `#version` and `#extension`, and inlines `#include "..."` (relative to the including file);
  - turns `layout(...) buffer` blocks into glsl::Buffer<T> globals (a runtime array; `.length()` is the bound count)
    and `layout(...) uniform` blocks and push constants into plain globals, which the driver sets;
  - turns `layout(...) uniform image2D` into a glsl::Image2D global, `layout(local_size_*) in;` into LOCAL_SIZE,
    and `shared T[N] x;` / `shared T x[N];` into a workgroup-shared global;
  - maps `in` / `out` / `inout` parameters to by-value / reference parameters;
  - adds an `f` suffix to unsuffixed floating literals (fp32 in GLSL, fp64 in C++) and drops `lf`;
  - spells the int(...) / uint(...) constructors to_int / to_uint, swizzles `.xyz` as `.swizzle<0,1,2>()`, and main
    as glsl_main;
and wraps the result in `namespace glsl::<namespace>`, #undef-ing the macros the shader defined at the end.  Anything
it does not recognise is left alone, so an unsupported construct fails at compile time rather than silently.
"""
from __future__ import annotations

import re
import sys
from pathlib import Path


def strip_comments(src: str) -> str:
    out, i, n = [], 0, len(src)
    while i < n:
        c = src[i]
        if c == '"':
            j = i + 1
            while j < n and src[j] != '"':
                j += 2 if src[j] == "\\" else 1
            out.append(src[i:j + 1])
            i = j + 1
        elif src.startswith("//", i):
            j = src.find("\n", i)
            i = n if j < 0 else j
        elif src.startswith("/*", i):
            j = src.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append("\n" * src.count("\n", i, j))
            i = j
        else:
            out.append(c)
            i += 1
    return "".join(out)


def resolve(path: Path, seen=()) -> str:
    if path in seen:
        raise ValueError(f"recursive #include of {path}")
    lines = []
    for line in strip_comments(path.read_text()).splitlines():
        m = re.match(r'\s*#\s*include\s+"([^"]+)"', line)
        if m:
            lines.append(resolve((path.parent / m.group(1)).resolve(), seen + (path,)))
        elif re.match(r"\s*#\s*(version|extension)\b", line):
            lines.append("")
        else:
            lines.append(line)
    return "\n".join(lines)


def _members(body: str):
    """`T a; T b[];` -> [(type, name, array_suffix)]"""
    out = []
    for decl in body.split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        m = re.fullmatch(r"(.+?)\s*(\w+)\s*(\[[^\]]*\])?", decl)
        if not m:
            raise ValueError(f"cannot parse block member {decl!r}")
        out.append((m.group(1).strip(), m.group(2), m.group(3) or ""))
    return out


def _block(m: re.Match) -> str:
    kind, name, body, inst = m.group(3), m.group(4), m.group(5), m.group(6)
    if inst:
        raise NotImplementedError(f"named block instance {name} {inst}")
    out = [f"/* {kind} block {name} */"]
    for typ, member, arr in _members(body):
        if arr == "[]":
            if kind != "buffer":
                raise ValueError(f"runtime array in a {kind} block")
            out.append(f"Buffer<{typ}> {member};")
        else:
            out.append(f"{typ} {member}{arr};")
    return " ".join(out)


def _local_size(m: re.Match) -> str:
    sizes = {"x": "1", "y": "1", "z": "1"}
    for key, val in re.findall(r"local_size_([xyz])\s*=\s*([^,]+)", m.group(1)):
        sizes[key] = val.strip()
    return f"static const uvec3 LOCAL_SIZE = uvec3({sizes['x']}, {sizes['y']}, {sizes['z']});"


SWZ = {c: i for i, c in enumerate("xyzw")} | {c: i for i, c in enumerate("rgba")} | {c: i for i, c in enumerate("stpq")}


def translate(src: str, namespace: str) -> str:
    macros = re.findall(r"^\s*#\s*define\s+(\w+)", src, re.M)
    s = src
    # resource declarations
    s = re.sub(r"layout\s*\(([^)]*)\)\s*((?:readonly|writeonly|restrict|coherent|volatile|\s)*)"
               r"(buffer|uniform)\s+(\w+)\s*\{(.*?)\}\s*(\w*)\s*;", _block, s, flags=re.S)
    s = re.sub(r"layout\s*\(([^)]*)\)\s*(?:(?:readonly|writeonly|restrict|coherent|volatile|uniform)\s+)+image2D\s+(\w+)\s*;",
               lambda m: f"Image2D {m.group(2)};", s)
    s = re.sub(r"layout\s*\(([^)]*local_size[^)]*)\)\s*in\s*;", _local_size, s)
    s = re.sub(r"\bshared\s+([\w:]+)\s*\[([^\]]+)\]\s*(\w+)\s*;", r"\1 \3[\2];", s)
    s = re.sub(r"\bshared\s+", "", s)
    # parameters
    s = re.sub(r"(?<=[(,])(\s*)(?:const\s+)?(inout|out)\s+(\w+)\s+(\w+)", r"\1\3 &\4", s)
    s = re.sub(r"(?<=[(,])(\s*)(?:const\s+)?in\s+(\w+)\s+(\w+)", r"\1\2 \3", s)
    # literals: unsuffixed floats are fp32 in GLSL; `lf` is double
    s = re.sub(r"(?<![\w.])((?:\d+\.\d*|\.\d+)(?:[eE][+-]?\d+)?|\d+[eE][+-]?\d+)(lf|LF|[fF])?(?![\w.])",
               lambda m: m.group(1) + ("" if m.group(2) in ("lf", "LF") else "f"), s)
    # scalar constructors whose C++ cast is undefined out of range, swizzles, entry point
    s = re.sub(r"(?<![\w.])int\s*\(", "to_int(", s)
    s = re.sub(r"(?<![\w.])uint\s*\(", "to_uint(", s)
    # a member name of a struct or block the shader declares (`aabb`) is not a swizzle
    members = set()
    for body in re.findall(r"\bstruct\s+\w+\s*\{(.*?)\}", s, re.S):
        members |= {name for _, name, _ in _members(body)}
    members |= set(re.findall(r"/\* (?:buffer|uniform) block \w+ \*/.*?\b(\w+)(?:\[[^\]]*\])?;", s))
    s = re.sub(r"(?<=[\w\])])\.([xyzw]{2,4}|[rgba]{2,4}|[stpq]{2,4})\b(?!\s*\()",
               lambda m: m.group(0) if m.group(1) in members else
               ".swizzle<" + ",".join(str(SWZ[c]) for c in m.group(1)) + ">()", s)
    s = re.sub(r"\bvoid\s+main\s*\(", "void glsl_main(", s)
    undef = "".join(f"#undef {name}\n" for name in dict.fromkeys(macros))
    return (f"/* generated by glsl_to_cpp.py: do not edit */\nnamespace glsl {{\nnamespace {namespace} {{\n"
            f"{s}\n}} // namespace {namespace}\n}} // namespace glsl\n{undef}")


def main(argv):
    shader, namespace, out = Path(argv[1]), argv[2], Path(argv[3])
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(translate(resolve(shader.resolve()), namespace))


if __name__ == "__main__":
    main(sys.argv)
