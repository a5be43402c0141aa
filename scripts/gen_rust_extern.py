"""Prints a Rust `extern "C"` block for EVERY function declared in include/sdbgpu.h (the appendix of INTEGRATION.md).
Opaque handles become `*mut Sdb…`, enums and sdb_status `i32`; double-pointer const-ness is approximated."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
h = open(os.path.join(ROOT, "include", "sdbgpu.h")).read()
h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
protos = re.findall(r"^\s*((?:const\s+)?[A-Za-z_][A-Za-z0-9_]*\s*\**)\s*(sdb_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", h, flags=re.M)
HANDLES = {"sdb_ctx": "SdbCtx", "sdb_corpus": "SdbCorpus", "sdb_hnsw": "SdbHnsw", "sdb_graph": "SdbGraph"}
PRIM = {"uint64_t": "u64", "uint32_t": "u32", "uint16_t": "u16", "uint8_t": "u8", "int8_t": "i8", "int64_t": "i64", "int32_t": "i32", "double": "f64",
        "float": "f32", "int": "i32", "size_t": "usize", "char": "c_char", "void": "c_void", "sdb_status": "i32",
        "sdb_metric": "i32", "sdb_order": "i32", "sdb_dtype": "i32", "sdb_vector_type": "i32", "sdb_screen": "i32", "sdb_knn_stats": "SdbKnnStats", "sdb_hop_filter": "SdbHopFilter"}


def conv(t):
    t = t.replace("volatile", "").strip()
    stars = t.count("*")
    toks = t.replace("*", " ").split()
    is_const = "const" in toks
    toks = [x for x in toks if x != "const"]
    base = toks[0] if toks else "void"
    handle = base in HANDLES
    r = HANDLES.get(base, PRIM.get(base, base))
    for i in range(stars):
        inner_handle_ptr = handle and i == 0 and stars > 1  # `sdb_x* const*`: an array of (mutable) handles
        r = ("*mut " if inner_handle_ptr or not is_const else "*const ") + r
    return r


print('extern "C" {')
for ret, name, args in protos:
    args = " ".join(args.split())
    alist = [] if args.strip() in ("", "void") else [x.strip() for x in args.split(",")]
    out = []
    for i, x in enumerate(alist):
        if re.search(r"[\*\s]([A-Za-z_][A-Za-z0-9_]*)$", x) and not x.rstrip().endswith("*"):
            nm = re.search(r"([A-Za-z_][A-Za-z0-9_]*)$", x).group(1)
            ty = x[: x.rfind(nm)]
            if not ty.strip():
                ty, nm = nm, f"a{i}"
        else:
            ty, nm = x, f"a{i}"
        if nm in ("type", "fn", "ref", "in", "box", "match"):
            nm += "_"
        out.append(f"{nm}: {conv(ty)}")
    r = conv(ret)
    print(f"    pub fn {name}({', '.join(out)})" + ("" if r == "c_void" else f" -> {r}") + ";")
print("}")
