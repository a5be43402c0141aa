"""Check that kernels' machine code is unchanged apart from names between two builds.

    python scripts/sass_compare.py OLD.o NEW.o screen_tc_kernel screen_simt_kernel ...

For every kernel whose demangled name starts with one of the given names, the SASS of each instantiation in OLD.o
(`cuobjdump -sass`) must equal the SASS of some instantiation in NEW.o after symbol names, which encode the template
arguments, are blanked out.  New instantiations (a new template argument) are listed, not required to match.  Exit
status 1 when an old instantiation has no identical body in the new build.
"""
import re
import subprocess
import sys
from collections import defaultdict


def functions(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            name, body = m.group(1), []
            continue
        if name is None:
            continue
        code = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)  # instruction addresses
        code = re.sub(r"\b_Z\w+", "SYM", code)  # mangled names (relocations, calls)
        code = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", code).strip()  # encodings (they embed relocated offsets)
        if code:
            body.append(code)
    if name:
        funcs[name] = body
    return funcs


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), check=True, capture_output=True, text=True).stdout
    return dict(zip(names, out.splitlines()))


def main():
    old_obj, new_obj, prefixes = sys.argv[1], sys.argv[2], sys.argv[3:]
    old, new = functions(old_obj), functions(new_obj)
    dem = demangle(sorted(set(old) | set(new)))

    def family(n):
        base = re.sub(r"^.*::", "", dem[n].split("<")[0].split("(")[0])
        return next((p for p in prefixes if base == p), None)

    new_bodies = defaultdict(list)
    for n, b in new.items():
        if family(n):
            new_bodies[family(n)].append(("\n".join(b), n))
    bad = 0
    for n, b in sorted(old.items()):
        f = family(n)
        if not f:
            continue
        body = "\n".join(b)
        hit = [m for bb, m in new_bodies[f] if bb == body]
        print(("same   " if hit else "CHANGED"), dem[n])
        bad += 0 if hit else 1
    old_bodies = {"\n".join(b) for n, b in old.items() if family(n)}
    for f, lst in new_bodies.items():
        for bb, m in lst:
            if bb not in old_bodies:
                print("new    ", dem[m])
    print(f"{bad} old instantiation(s) changed")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
