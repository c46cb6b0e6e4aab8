#!/usr/bin/env python
"""Instruction mix of a kernel in an sm_90a object file, read from `cuobjdump -sass` (nothing runs on a GPU).

  python tools/sass_mix.py build/obj/msm.o                       # k_msm_accumulate<128, 2>
  python tools/sass_mix.py build/obj/msm.o --kernel heavy_chunks

Prints the registers per thread and the stack frame (`cuobjdump -res-usage`), the opcode mix of the kernel
(out-of-line functions it calls, listed after its EXIT, counted apart), and the mix of its bucket loop: the
span of the backward branch that loads from global memory (the next point) and encloses the most
IMAD.WIDE.U32 instructions.  "common path" is that span
without the forward-branch region that holds a CALL (the call site of the rare case, with its saves and
restores).  A rare case inlined into the loop stays in the span; --skip START:END (hex addresses, end
exclusive, repeatable) takes such a region out of the common path.
"""
import argparse
import collections
import re
import subprocess

INS = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);")
TARGET = re.compile(r"(0x[0-9a-f]+)\s*$")


def functions(sass):
    name, body = None, []
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                yield name, body
            name, body = m.group(1), []
        elif name:
            body.append(line)
    if name:
        yield name, body


def parse(body):
    """[(address, opcode, branch or call target address or None)]"""
    ins = []
    for line in body:
        m = INS.search(line)
        if m:
            op = m.group(2)
            t = TARGET.search(m.group(3)) if op.startswith(("BRA", "CALL")) else None
            ins.append((int(m.group(1), 16), op, int(t.group(1), 16) if t else None))
    return ins


def bucket(op):
    if op.startswith("IMAD.WIDE.U32"):
        return op
    if op.startswith("IMAD"):
        return "IMAD (other)"
    if op.startswith("HFMA2.MMA") or op.startswith("MOV"):
        return "MOV + HFMA2.MMA"
    return op.split(".")[0]


def show(title, ins):
    c = collections.Counter(bucket(op) for _, op, _ in ins)
    print(f"{title}: {len(ins)} instructions")
    for k, v in c.most_common():
        print(f"  {k:<22} {v:>7}")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("obj")
    ap.add_argument("--kernel", default="k_msm_accumulateILi128ELi2E", help="substring of the mangled kernel name")
    ap.add_argument("--skip", action="append", default=[], help="START:END hex address range left out of the common path")
    args = ap.parse_args()
    sass = subprocess.run(["cuobjdump", "-sass", args.obj], check=True, capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", args.obj], check=True, capture_output=True, text=True).stdout
    found = [(n, b) for n, b in functions(sass) if args.kernel in n]
    if not found:
        raise SystemExit(f"no function matching {args.kernel!r} in {args.obj}")
    for name, body in found:
        print(name)
        lines = res.splitlines()
        for i, line in enumerate(lines):
            if name in line and i + 1 < len(lines):
                print("  " + lines[i + 1].strip())
        ins = parse(body)
        callees = [t for _, op, t in ins if op.startswith("CALL") and t is not None]
        end = min(callees) if callees else ins[-1][0] + 1
        kernel = [i for i in ins if i[0] < end]
        show("kernel", kernel)
        if callees:
            show("out-of-line callees", [i for i in ins if i[0] >= end])
        best = None
        for j, (a, op, t) in enumerate(kernel):
            if op.startswith("BRA") and t is not None and t <= a:
                span = [i for i in kernel if t <= i[0] <= a]
                if not any(o.startswith("LDG") for _, o, _ in span):
                    continue
                n = sum(1 for _, o, _ in span if o.startswith("IMAD.WIDE.U32"))
                if best is None or n > best[0]:
                    best = (n, span)
        if best:
            span = best[1]
            show("bucket loop (one iteration)", span)
            calls = [a for a, op, _ in span if op.startswith("CALL")]
            skips = [(a, t) for a, op, t in span if op.startswith("BRA") and t is not None and t > a
                     and any(a < c < t for c in calls)]
            out = [tuple(int(x, 16) for x in r.split(":")) for r in args.skip]
            if skips:
                a0, t0 = min(skips, key=lambda r: r[1] - r[0])
                out.append((a0 + 1, t0))
            if out:
                show("bucket loop, common path", [i for i in span if not any(a <= i[0] < b for a, b in out)])
        print()


if __name__ == "__main__":
    main()
