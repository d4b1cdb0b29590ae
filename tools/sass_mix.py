"""Static instruction report of one kernel of the built library: no GPU needed.

  python tools/sass_mix.py idct_color_420 [--lib dali_b200/lib/libdali_b200.so] [--top 12]

Runs `cuobjdump -sass` on the library, picks the kernel whose (mangled) name contains the given string, and prints its total
instruction count, then every loop (a backward branch to an earlier offset) with its instruction count and opcode mix, innermost
loops listed inside the ones that contain them.  Opcodes are counted without their modifiers (IMAD.WIDE -> IMAD).  These are static
counts: how often a loop runs, and how many lanes are active, is up to the shapes.  The compiler may place a branch's code after
the loop that contains it (idct_color_420's halo path), and then that loop looks shorter and an outer range appears beside it."""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)([.A-Z0-9_]*)\s*(.*?);")


def kernel_sass(lib, name):
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            m = INSN.match(line)
            if m:
                funcs[cur].append((int(m.group(1), 16), m.group(3), m.group(5)))
    hits = [f for f in funcs if name in f]
    if len(hits) != 1:
        sys.exit(f"{len(hits)} kernels match {name!r}: {hits[:8]}")
    return hits[0], funcs[hits[0]]


def loops(ins):
    """(start, end) offsets of every backward branch's body, outermost first"""
    out = set()
    for off, op, args in ins:
        if op == "BRA":
            t = re.search(r"0x([0-9a-f]+)", args)
            if t and int(t.group(1), 16) <= off:
                out.add((int(t.group(1), 16), off))
    return sorted(out, key=lambda r: (r[0], -r[1]))


def mix(ins, a, b):
    return collections.Counter(op for off, op, _ in ins if a <= off <= b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("kernel")
    ap.add_argument("--lib", default=os.path.join(ROOT, "dali_b200", "lib", "libdali_b200.so"))
    ap.add_argument("--top", type=int, default=12)
    a = ap.parse_args()
    fname, ins = kernel_sass(a.lib, a.kernel)
    print(f"{fname}: {len(ins)} instructions")
    ls = loops(ins)
    for s, e in ls:
        depth = sum(1 for s2, e2 in ls if (s2, e2) != (s, e) and s2 <= s and e <= e2)
        c = mix(ins, s, e)
        pad = "  " * (depth + 1)
        print(f"{pad}loop {s:#06x}-{e:#06x}: {sum(c.values())} instructions")
        print(pad + "  " + ", ".join(f"{op} {n}" for op, n in c.most_common(a.top)))


if __name__ == "__main__":
    main()
