"""SASS opcode census of the built library (which instructions the kernels really issue).

    python tools/sass_census.py [path/to/lib.so|cubin] [--kernel SUBSTR] [--loops] [--lines OPC[,OPC...]]
    python tools/sass_census.py [path/to/lib.so|cubin] --same-as OTHER.so

For every kernel: static instruction count, opcode histogram, pipe summary (IMAD.WIDE-class on the fmaheavy pipe,
narrow IMAD, ALU, FP64, memory).  --loops also prints one census per natural loop (backward branch -> its target),
innermost first, which is what the round loop / S-box loop of the Hades kernel execute dynamically.
--lines prints the first SASS lines of the given opcodes (e.g. LDG.E.128.CONSTANT,STG.E.128,DFMA) per kernel.
--same-as OTHER.so compares every kernel's instruction text with OTHER's (addresses and encodings stripped), prints the
kernels that differ or exist on one side only, and exits 1 if there are any.
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT = os.path.join(ROOT, "poseidon252_b200", "lib", "libposeidon252_b200.so")

INS = re.compile(r"^\s+/\*([0-9a-f]{4,6})\*/\s+(?:@!?U?P[0-9T]+\s+)?([A-Z0-9_.]+)(.*?);")


def parse(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], stdout=subprocess.PIPE, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for ln in txt.splitlines():
        if "Function :" in ln:
            cur = ln.split("Function :")[1].strip()
            kernels[cur] = []
            continue
        m = INS.match(ln)
        if m and cur is not None:
            kernels[cur].append((int(m.group(1), 16), m.group(2), m.group(3).strip(), ln.strip()))
    return kernels


def demangle(name):
    try:
        return subprocess.run(["c++filt", name], stdout=subprocess.PIPE, text=True).stdout.strip() or name
    except Exception:
        return name


def klass(op):
    if op.startswith("IMAD.WIDE") or op.startswith("IMAD.HI"):
        return "imad_wide(fmaheavy,4cyc)"
    if op.startswith("IMAD") or op.startswith("UIMAD"):
        return "imad_narrow(fma,2cyc)"
    if op.startswith(("DFMA", "DADD", "DMUL", "I2F.F64", "F2I.F64", "DSETP")):
        return "fp64"
    if op.startswith(("IADD3", "LOP3", "SHF", "SEL", "MOV", "ISETP", "LEA", "VIADD", "PRMT", "CS2R", "P2R", "R2P", "IABS",
                      "VIMNMX", "IMNMX", "UIADD3", "UMOV", "USEL", "ULEA", "UISETP", "USHF", "ULOP3", "S2R", "S2UR")):
        return "alu"
    if op.startswith(("LDG", "STG", "LDS", "STS", "LDC", "LDCU", "LDL", "STL", "ATOM", "RED", "UBLKCP", "SYNCS")):
        return "memory"
    return "other"


def census(ins):
    h = collections.Counter(op for _, op, _, _ in ins)
    c = collections.Counter()
    for op, n in h.items():
        c[klass(op)] += n
    return h, c


def fmt(h, c, indent="  "):
    tot = sum(h.values())
    out = ["%s%d instructions: %s" % (indent, tot, ", ".join("%s=%d" % kv for kv in sorted(c.items(), key=lambda kv: -kv[1])))]
    out.append(indent + "  " + "  ".join("%s:%d" % kv for kv in h.most_common(28)))
    return "\n".join(out)


def loops(ins):
    addr_index = {a: i for i, (a, _, _, _) in enumerate(ins)}
    found = []
    for i, (a, op, rest, _) in enumerate(ins):
        if op.startswith("BRA"):
            m = re.search(r"0x([0-9a-f]+)", rest)
            if m:
                t = int(m.group(1), 16)
                if t <= a and t in addr_index:
                    found.append((addr_index[t], i))
    return sorted(found, key=lambda lo_hi: lo_hi[1] - lo_hi[0])


def text(ins):
    # instruction text only: the /*addr*/ prefix and the /* 0x... */ encoding comment removed
    return [" ".join(re.sub(r"/\*[^*]*\*/", " ", ln).split()) for _, _, _, ln in ins]


def same_as(path, other):
    a, b = parse(path), parse(other)
    names = list(a) + [k for k in b if k not in a]
    bad = 0
    for name in names:
        if name not in a or name not in b:
            print("only in %s: %s" % (path if name in a else other, demangle(name)))
            bad += 1
        elif text(a[name]) != text(b[name]):
            print("differs: %s" % demangle(name))
            bad += 1
    print("%d kernels, %d identical" % (len(names), len(names) - bad))
    return 1 if bad else 0


def main():
    args = sys.argv[1:]
    path, want, show_loops, lines, other = DEFAULT, None, False, [], None
    while args:
        a = args.pop(0)
        if a == "--kernel":
            want = args.pop(0)
        elif a == "--loops":
            show_loops = True
        elif a == "--lines":
            lines = args.pop(0).split(",")
        elif a == "--same-as":
            other = args.pop(0)
        else:
            path = a
    if other:
        sys.exit(same_as(path, other))
    for name, ins in parse(path).items():
        dn = demangle(name)
        if want and want not in dn and want not in name:
            continue
        print("== %s" % dn)
        h, c = census(ins)
        print(fmt(h, c))
        if show_loops:
            for lo, hi in loops(ins):
                h2, c2 = census(ins[lo:hi + 1])
                print("  loop /*%04x*/../*%04x*/" % (ins[lo][0], ins[hi][0]))
                print(fmt(h2, c2, "    "))
        for opc in lines:
            hits = [ln for _, op, _, ln in ins if op.startswith(opc)]
            print("  -- %s: %d" % (opc, len(hits)))
            for ln in hits[:4]:
                print("     " + ln)


if __name__ == "__main__":
    main()
