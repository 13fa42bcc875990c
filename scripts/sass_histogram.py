#!/usr/bin/env python
"""Opcode histogram per kernel from the built objects (cuobjdump -sass): the evidence that the sm_90a instructions the design
relies on are really in the binaries (bulk async copy UBLKCP + mbarrier SYNCS, VOTE, ...).
Usage: python scripts/sass_histogram.py [build/obj/*.o]
       python scripts/sass_histogram.py --pipes --kernel k_allocILb0 [--range 0x1a40:0x1c90] build/obj/tsdf.o
--pipes adds the split by execution pipe (PIPES below: which sm_90 pipe issues each opcode); --kernel keeps the kernels whose
mangled name contains the string; --range keeps the instructions at addresses lo <= a < hi (an inner loop: take the
addresses from scripts/sass_kernel.sh)."""
import argparse
import collections
import glob
import re
import subprocess

WATCH = ["UBLKCP", "SYNCS", "MUFU", "F2I", "I2F", "I2FP", "LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "RED", "VOTE", "SHFL", "BAR",
         "IMAD", "FFMA", "LDL", "STL", "LDC", "BRA"]

# Execution pipe by opcode on sm_90.  FMA: the two 16-lane FP32 pipes (FFMA / FMUL / FADD, and IMAD); ALU: the one 16-lane
# integer / logic pipe, which also takes FP32 compare, select and min / max; XU: the 4-lane special-function unit and
# conversions; LSU: memory (LDC goes through the constant cache, counted here); CTRL: branches, barriers, reconvergence;
# UNI: the uniform datapath (opcodes starting with U).  Opcodes not listed are reported as OTHER.
PIPES = {
    "FMA": ["FFMA", "FMUL", "FADD", "IMAD", "HFMA2", "HADD2", "HMUL2"],
    "ALU": ["FSETP", "FSEL", "SEL", "FMNMX", "ISETP", "LOP3", "IADD3", "LEA", "SHF", "PRMT", "MOV", "IMNMX", "PLOP3", "IABS", "I2FP",
            "FSET", "VOTE", "VOTEU", "P2R", "R2P", "CS2R", "SGXT", "BMSK", "IADD", "FCHK", "VABSDIFF", "IDP", "LOP", "SHL", "SHR", "VIADD", "VIMNMX"],
    "XU": ["MUFU", "F2I", "I2F", "F2F", "POPC", "FLO", "BREV", "I2I", "F2IP", "FRND", "S2R", "S2UR"],
    "LSU": ["LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "ATOM", "RED", "LDL", "STL", "LD", "ST", "LDC", "LDSM", "SHFL", "MATCH", "REDUX",
            "MEMBAR", "CCTL", "ERRBAR", "LDGSTS", "LDGDEPBAR", "UBLKCP", "SYNCS", "FENCE"],
    "CTRL": ["BRA", "BSSY", "BSYNC", "EXIT", "CALL", "RET", "WARPSYNC", "BAR", "NOP", "YIELD", "BRX", "JMP", "DEPBAR", "BREAK", "BMOV", "BPT",
             "NANOSLEEP", "KILL", "RPCMOV", "ACQBULK", "ENDCOLLECTIVE"],
}
PIPE_OF = {op: pipe for pipe, ops in PIPES.items() for op in ops}


def pipe_of(op):
    return PIPE_OF.get(op) or ("UNI" if op.startswith("U") else "OTHER")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--pipes", action="store_true")
    ap.add_argument("--kernel", default="")
    ap.add_argument("--range", default="")
    ap.add_argument("objs", nargs="*")
    a = ap.parse_args()
    lo, hi = (int(x, 16) for x in a.range.split(":")) if a.range else (0, 1 << 62)
    objs = a.objs or sorted(glob.glob("build/obj/*.o"))
    print("# SASS opcode histogram per kernel (static instruction counts; cuobjdump -sass of the shipped objects, sm_90a)")
    for o in objs:
        try:
            txt = subprocess.run(["cuobjdump", "-sass", o], capture_output=True, text=True).stdout
        except FileNotFoundError:
            print("cuobjdump not found"); return
        kern = None; hist = {}
        for ln in txt.splitlines():
            m = re.search(r"Function : (\S+)", ln)
            if m:
                kern = m.group(1) if a.kernel in m.group(1) else None
                if kern: hist[kern] = collections.Counter()
                continue
            m = re.match(r"\s+/\*([0-9a-f]{4,6})\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
            if m and kern and lo <= int(m.group(1), 16) < hi:
                hist[kern][m.group(2)] += 1
        if not hist:
            continue
        print(f"\n## {o}")
        for k, h in hist.items():
            short = subprocess.run(["c++filt", k], capture_output=True, text=True).stdout.strip()
            short = re.sub(r"\(anonymous namespace\)::|_GLOBAL__N__\w+::", "", short)
            short = re.sub(r"^void ", "", short)
            depth = 0; cut = len(short)
            for i, ch in enumerate(short):                      # drop the argument list, keep template arguments
                if ch == "<": depth += 1
                elif ch == ">": depth -= 1
                elif ch == "(" and depth == 0: cut = i; break
            short = short[:cut]
            tot = sum(h.values())
            keys = [w for w in WATCH if h.get(w)]
            print(f"{short:70s} total {tot:5d}  " + " ".join(f"{w}={h[w]}" for w in keys))
            if a.pipes:
                by = collections.defaultdict(collections.Counter)
                for op, n in h.items():
                    by[pipe_of(op)][op] += n
                for pipe in list(PIPES) + ["UNI", "OTHER"]:
                    if by[pipe]:
                        n = sum(by[pipe].values())
                        print(f"    {pipe:5s} {n:5d} ({100.0 * n / tot:4.1f} %)  " + " ".join(f"{op}={c}" for op, c in by[pipe].most_common()))


if __name__ == "__main__":
    main()
