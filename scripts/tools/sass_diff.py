"""Compare the SASS of two builds of libjfgpu.so, kernel by kernel (CPU only).

    python scripts/tools/sass_diff.py OLD/lib/libjfgpu.so NEW/lib/libjfgpu.so [--show NAME]

Each library is disassembled with `cuobjdump -sass` and split at its `Function :` lines.  Only the `/*0040*/` address
comments are dropped, so opcodes, registers and encodings are compared.  The `ptxas.log` beside each library (the
Makefile writes it) gives the registers, stack/spill bytes and shared memory of every function; those lines are compared
too.  Prints the functions whose SASS changed with their instruction counts, then `same N changed M`; `--show NAME`
(a substring of the mangled name) prints the differing lines of the matching functions.
"""
import argparse
import difflib
import os
import re
import subprocess

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
ADDR = re.compile(r"/\*[0-9a-f]{4,}\*/")


def sass(lib):
    out = subprocess.run([CUOBJDUMP, "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :")[1].strip()
            funcs[name] = []
        elif name is not None and line.strip().startswith(".........."):
            name = None
        elif name is not None and line.strip():
            funcs[name].append(ADDR.sub("", line).strip())
    return funcs


def resources(lib):
    """{function: sorted list of its ptxas resource lines} from the ptxas.log next to the library"""
    res, name = {}, None
    path = os.path.join(os.path.dirname(os.path.abspath(lib)), "ptxas.log")
    with open(path) as f:
        for line in f:
            m = re.search(r"Function properties for (\S+)", line)
            if m:
                name = m.group(1)
                res.setdefault(name, [])
            elif name and ("bytes stack frame" in line or line.startswith("ptxas info    : Used")):
                res[name].append(line.split(":", 1)[-1].strip())
    return {k: sorted(v) for k, v in res.items()}


def n_instr(lines):
    return sum(1 for l in lines if not l.startswith(("/*", ".")))     # (the rest are encoding halves and headers)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--show", metavar="NAME", help="print the differing lines of the functions whose name contains NAME")
    a = ap.parse_args()
    old, new = sass(a.old), sass(a.new)
    same = changed = 0
    for name in sorted(set(old) | set(new)):
        o, n = old.get(name), new.get(name)
        if o == n:
            same += 1
            continue
        changed += 1
        print("changed %-90s %s -> %s instructions" % (name, n_instr(o) if o else "absent", n_instr(n) if n else "absent"))
        if a.show and a.show in name:
            for d in difflib.unified_diff(o or [], n or [], "old", "new", n=0, lineterm=""):
                print("    " + d)
    ro, rn = resources(a.old), resources(a.new)
    res_changed = 0
    for name in sorted(set(ro) | set(rn)):
        if ro.get(name) != rn.get(name):
            res_changed += 1
            print("resources %s\n    old %s\n    new %s" % (name, ro.get(name), rn.get(name)))
    print("same %d changed %d  (resource lines changed: %d)" % (same, changed, res_changed))


if __name__ == "__main__":
    main()
