"""Checks the #[repr(C)] structs of ffi/llmlb-b200-sys/src/lib.rs against include/llmlb_b200.h without
a Rust toolchain: the Rust text is parsed (field names, order, primitive types), a gcc-compiled probe
prints sizeof / offsetof of every field of the C structs, and the Rust layout is computed with the C
rules `repr(C)` guarantees (natural alignment, declaration order).  Also checks the integer constants
and that every `extern "C"` function exists in the header with the same number of parameters."""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RS = os.path.join(ROOT, "ffi", "llmlb-b200-sys", "src", "lib.rs")
HDR = os.path.join(ROOT, "include", "llmlb_b200.h")

PRIM = {"u8": (1, 1), "i8": (1, 1), "c_char": (1, 1), "u32": (4, 4), "i32": (4, 4), "f32": (4, 4), "c_int": (4, 4),
        "u64": (8, 8), "i64": (8, 8), "f64": (8, 8)}


def rust_structs(text):
    out = {}
    for m in re.finditer(r"#\[repr\(C\)\][^{]*?pub struct (\w+)\s*\{(.*?)\n\}", text, re.S):
        name, body = m.group(1), m.group(2)
        fields = []
        for fm in re.finditer(r"pub (\w+):\s*([^,\n]+),", body):
            fields.append((fm.group(1), fm.group(2).strip()))
        out[name] = fields
    return out


def layout(ty, structs):
    """(size, align) of a Rust type under repr(C)"""
    ty = ty.strip()
    if ty.startswith("*"):
        return 8, 8
    m = re.match(r"\[(.+);\s*(\d+)\]", ty)
    if m:
        s, a = layout(m.group(1), structs)
        return s * int(m.group(2)), a
    if ty in PRIM:
        return PRIM[ty]
    if ty in structs:
        off, al = 0, 1
        for _, fty in structs[ty]:
            s, a = layout(fty, structs)
            off = (off + a - 1) // a * a + s
            al = max(al, a)
        return (off + al - 1) // al * al, al
    raise ValueError("unknown Rust type " + ty)


def rust_offsets(name, structs):
    off, al, res = 0, 1, []
    for fname, fty in structs[name]:
        s, a = layout(fty, structs)
        off = (off + a - 1) // a * a
        res.append((fname, off, s))
        off += s
        al = max(al, a)
    return res, (off + al - 1) // al * al


def c_offsets(structs):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "llmlb_b200.h"', "int main(void){"]
    for name, fields in structs.items():
        if not fields:
            continue
        lines.append('printf("S %s %%zu\\n", sizeof(%s));' % (name, name))
        for f, _ in fields:
            lines.append('printf("F %s %s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (name, f, name, f, name, f))
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        txt = subprocess.check_output([exe], text=True)
    sizes, offs = {}, {}
    for ln in txt.splitlines():
        p = ln.split()
        if p[0] == "S":
            sizes[p[1]] = int(p[2])
        else:
            offs[(p[1], p[2])] = (int(p[3]), int(p[4]))
    return sizes, offs


def check():
    text = open(RS).read()
    hdr = open(HDR).read()
    structs = rust_structs(text)
    problems = []
    want = ["llmlb_model_config", "llmlb_engine_config", "llmlb_model_info", "llmlb_health", "llmlb_sampling", "llmlb_token_event",
            "llmlb_prefix_cache_stats"]
    for w in want:
        if w not in structs:
            problems.append("struct %s missing from lib.rs" % w)
    sizes, offs = c_offsets({k: v for k, v in structs.items() if k in want})
    for name in want:
        if name not in structs:
            continue
        ro, rsize = rust_offsets(name, structs)
        if rsize != sizes[name]:
            problems.append("%s: size %d in Rust, %d in C" % (name, rsize, sizes[name]))
        for fname, off, sz in ro:
            if (name, fname) not in offs:
                problems.append("%s.%s is not a field of the C struct" % (name, fname))
            elif offs[(name, fname)] != (off, sz):
                problems.append("%s.%s: offset/size %s in Rust, %s in C" % (name, fname, (off, sz), offs[(name, fname)]))
        # every C field must be bound: count the fields in the header's struct body
        cm = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S)
        c_fields = re.findall(r"\b(\w+)(?:\[\w+\])?;", re.sub(r"/\*.*?\*/", "", cm.group(1), flags=re.S))
        if [f for f, _ in structs[name]] != c_fields:
            problems.append("%s: field lists differ: Rust %s vs C %s" % (name, [f for f, _ in structs[name]], c_fields))
    # constants
    for m in re.finditer(r"pub const (LLMLB_\w+): \w+ = (-?\d+);", text):
        cname, val = m.group(1), int(m.group(2))
        hm = re.search(r"\b%s\s*=\s*(-?\d+)" % cname, hdr) or re.search(r"#define %s\s+(-?\d+)" % cname, hdr)
        if not hm:
            problems.append("constant %s not found in the header" % cname)
        elif int(hm.group(1)) != val:
            problems.append("constant %s: %d in Rust, %s in C" % (cname, val, hm.group(1)))
    # functions
    for m in re.finditer(r"pub fn (llmlb_\w+)\((.*?)\)", text, re.S):
        fname, params = m.group(1), m.group(2)
        hm = re.search(r"^[\w \*]+\b%s\s*\(([^;{]*?)\)\s*;" % fname, hdr, re.S | re.M)
        if not hm:
            problems.append("function %s is not declared in the header" % fname)
            continue
        n_rust = 0 if not params.strip() else len([p for p in params.split(",") if p.strip()])
        c_params = hm.group(1).strip()
        n_c = 0 if c_params in ("", "void") else len([p for p in re.sub(r"/\*.*?\*/", "", c_params, flags=re.S).split(",") if p.strip()])
        if n_rust != n_c:
            problems.append("function %s: %d parameters in Rust, %d in C" % (fname, n_rust, n_c))
    return problems


if __name__ == "__main__":
    p = check()
    for x in p:
        print("MISMATCH:", x)
    print("ok" if not p else "%d problems" % len(p))
    sys.exit(1 if p else 0)
