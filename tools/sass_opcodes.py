"""SASS opcode histogram per kernel of the shipped library (cuobjdump -sass) (printed to stdout).

    python tools/sass_opcodes.py parseable_b200/libparseable_b200.so > profiles/sass_opcodes_r2.txt
"""
import collections
import re
import subprocess
import sys

FAMILIES = ["UBLKCP", "SYNCS", "ATOMS", "ATOMG", "ATOM", "REDG", "RED", "REDUX", "VOTE", "SHFL", "LDS", "STS", "LDG", "LD", "STG", "ST", "SHF", "LOP3",
            "NANOSLEEP", "BAR"]
DETAIL = ("UBLKCP", "SYNCS", "ATOMS", "ATOM.", "ATOMG")


def demangle_short(name: str) -> str:
    m = re.match(r"_ZN3pqb(\d+)", name)
    if m:
        n = int(m.group(1))
        s = name[len(m.group(0)):len(m.group(0)) + n]
        t = re.search(r"I(L[bi]\d+E)+E", name[len(m.group(0)) + n:len(m.group(0)) + n + 12])
        return s + (f"<{t.group(0)[1:-1]}>" if t else "")
    m = re.match(r"_Z(\d+)", name)
    if m:
        n = int(m.group(1))
        return name[len(m.group(0)):len(m.group(0)) + n]
    return name


def main():
    lib = sys.argv[1]
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    kern, ops = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            kern = demangle_short(m.group(1))
            ops[kern] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", line)
        if m and kern:
            ops[kern][m.group(1)] += 1
    print(f"# SASS opcode histogram of {lib} (cuobjdump -sass, sm_90a cubins only; tools/sass_opcodes.py)")
    print("# UBLKCP = cp.async.bulk (TMA 1-D bulk copy), SYNCS.* = mbarrier ops (ARRIVE.TRANS64, PHASECHK.TRANS64.TRYWAIT), REDUX = warp reduce,")
    print("# ATOMS = shared-memory atomics, RED/REDG/ATOMG/ATOM = global reductions / atomics, LD/ST = generic loads / stores\n")
    for k, c in ops.items():
        total = sum(c.values())
        fam = []
        for f in FAMILIES:
            n = sum(v for o, v in c.items() if o == f or o.startswith(f + "."))
            if n:
                fam.append(f"{f} {n}")
        print(f"{k}: {total} instructions; " + ", ".join(fam))
        det = sorted((o, v) for o, v in c.items() if o.startswith(DETAIL))
        if det:
            print("    " + ", ".join(f"{o} x{v}" for o, v in det))


if __name__ == "__main__":
    main()
