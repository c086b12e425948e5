"""Instruction mix of the k_viterbi column loop, read from the SASS (no GPU needed).

usage: python tools/sass_mix.py [--compile] [--lib PATH] [--all] [--filter SUBSTR]

For every k_viterbi<R,LOCAL,SS,CELLOFF> instantiation in the library it finds the column loop (see column_loop)
and prints its static instructions per row visit (one row of one column for the 32 lanes of a warp) by opcode, the
MOVs, LDS (query rows and operand ring) and LDGSTS (cp.async into the ring) per column, registers, the size of the running-maximum rare path inside the loop and, with --compile, the
spill bytes ptxas reports.  It also splits the instructions per row visit between the FP32 pipe and the ALU pipe
(PIPES below), and sums the stall counts ptxas encodes in each instruction's control bits over one pass of the loop
(cycles per column before latency and dependency waits), with how many instructions stall for 2 cycles, the count
ptxas gives back-to-back ALU-pipe instructions, which issue at half the FP32 rate.  --compile builds the library with the flags of build.py into a
temporary directory; otherwise --lib (default hh-suite_b200/libhhg.so) is read.
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "hh-suite_b200"))
import build  # noqa: E402

CUDA_BIN = os.path.dirname(build.NVCC)
MANGLED = re.compile(r"_ZN3hhg9k_viterbiILi(\d+)ELb(\d)ELb(\d)ELb(\d)EEEvNS_9VitParamsE")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)([^;]*);")
HEX = re.compile(r"/\*\s*0x([0-9a-f]{16})\s*\*/\s*$")
# the pipe each opcode issues to on sm_90 (the rest: memory, moves, branches, uniform datapath)
PIPES = {"FP32": {"FADD", "FMUL", "FFMA", "IMAD", "HFMA2"},
         "ALU": {"FMNMX", "FSETP", "FSEL", "SEL", "ISETP", "IADD3", "LOP3", "LEA", "SHF", "PRMT", "PLOP3", "IMNMX"}}


def name_of(m: re.Match) -> str:
    return f"k_viterbi<{m.group(1)},{m.group(2)},{m.group(3)},{m.group(4)}>"


def compile_lib(tmp: str) -> tuple[str, dict]:
    out = os.path.join(tmp, "libhhg.so")
    res = subprocess.run([build.NVCC] + build.FLAGS + ["-Xptxas", "-v", "-o", out, build.SRC],
                         capture_output=True, text=True, check=True)
    spills, cur = {}, None
    for line in res.stderr.splitlines():
        m = MANGLED.search(line)
        if m and "Compiling entry function" in line:
            cur = name_of(m)
        s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if s and cur:
            spills[cur] = (int(s.group(1)), int(s.group(2)))
            cur = None
    return out, spills


def functions(lib: str) -> tuple[dict[str, list[tuple[int, str, str]]], dict[str, dict[int, int]]]:
    """Per instantiation its instructions (address, opcode, operands) and the stall count of each address: bits 41-44
    of the second 64-bit word of the 128-bit encoding, which cuobjdump prints on the line after the instruction."""
    sass = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", lib], capture_output=True, text=True,
                          check=True).stdout
    funcs, stalls, cur, last = {}, {}, None, None
    for line in sass.splitlines():
        if "Function :" in line:
            m = MANGLED.search(line)
            cur = name_of(m) if m else None
            if cur:
                funcs[cur], stalls[cur] = [], {}
            last = None
            continue
        if cur:
            m = INSN.search(line)
            if m:
                last = int(m.group(1), 16)
                funcs[cur].append((last, m.group(3), m.group(4)))
            elif last is not None:
                h = HEX.search(line)
                if h:
                    stalls[cur][last] = (int(h.group(1), 16) >> 41) & 0xF
                last = None
    return funcs, stalls


def registers(lib: str) -> dict[str, tuple[int, int]]:
    txt = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-res-usage", lib], capture_output=True, text=True,
                         check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = MANGLED.search(line)
        if m:
            cur = name_of(m)
            continue
        r = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if r and cur:
            out[cur] = (int(r.group(1)), int(r.group(2)))
            cur = None
    return out


def column_loop(insns: list[tuple[int, str, str]], R: int) -> list[tuple[int, str, str]]:
    """The narrowest backward-branch range [target, branch] that holds at least the 7 R LDS.128 of the R query
    rows, no atomic (work queue) and no SYNCS (mbarrier wait), and that no other backward branch
    crosses: a cold block placed after the loop that jumps back into it spans the loop's back edge, whose target
    lies before the cold block's target."""
    lds = [a for a, op, _ in insns if op == "LDS"]
    bad = [a for a, op, _ in insns if op.startswith("ATOM") or op.startswith("SYNCS")]
    back = []
    for a, op, rest in insns:
        t = re.search(r"0x([0-9a-f]+)", rest) if op == "BRA" else None
        if t and int(t.group(1), 16) < a:
            back.append((int(t.group(1), 16), a))
    best = None
    for lo, hi in back:
        if sum(lo <= x <= hi for x in lds) < 7 * R or any(lo <= x <= hi for x in bad):
            continue
        if any(lo < a2 < hi and lo2 < lo for lo2, a2 in back):
            continue
        if best is None or hi - lo < best[1] - best[0]:
            best = (lo, hi)
    if best is None:
        raise RuntimeError("column loop not found")
    return [i for i in insns if best[0] <= i[0] <= best[1]]


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=build.OUT)
    ap.add_argument("--compile", action="store_true", help="build the library with build.py's flags first")
    ap.add_argument("--all", action="store_true", help="every instantiation (default: the <16,1,0,0> headline)")
    ap.add_argument("--filter", default="", help="only instantiations whose name contains this")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        spills = {}
        lib = args.lib
        if args.compile:
            lib, spills = compile_lib(tmp)
        funcs, stalls = functions(lib)
        regs = registers(lib)
    names = sorted(funcs, key=lambda n: [int(x) for x in re.findall(r"\d+", n)], reverse=True)
    if not args.all:
        names = [n for n in names if n == "k_viterbi<16,1,0,0>"]
    names = [n for n in names if args.filter in n]
    for n in names:
        R = int(re.search(r"<(\d+)", n).group(1))
        loop = column_loop(funcs[n], R)
        mix = collections.Counter(op for _, op, _ in loop)
        reg, stack = regs.get(n, (0, 0))
        sp = spills.get(n)
        # the widest block inside the loop that a forward branch skips: the running-maximum rare path, which the
        # common path jumps over (counted above, since it sits between the loop's first and last instruction)
        cold = 0
        for a, op, rest in loop:
            t = re.search(r"0x([0-9a-f]+)", rest) if op == "BRA" else None
            if t and a < int(t.group(1), 16) <= loop[-1][0]:
                cold = max(cold, sum(a < x < int(t.group(1), 16) for x, _, _ in loop))
        print(f"{n}: {len(loop)} instructions per column = {len(loop) / R:.1f} per row visit; "
              f"MOV {mix['MOV']}, LDS {mix['LDS']}, LDGSTS {mix['LDGSTS']} per column; {reg} registers, stack {stack} B"
              + (f", spill stores {sp[0]} B / loads {sp[1]} B" if sp else "")
              + f"; widest skipped block {cold} ({(len(loop) - cold) / R:.1f} per row visit without it)")
        pipe = {k: sum(c for op, c in mix.items() if op in v) for k, v in PIPES.items()}
        st = [stalls[n][a] for a, _, _ in loop]
        print(f"   per row visit: FP32 pipe {pipe['FP32'] / R:.1f}, ALU pipe {pipe['ALU'] / R:.1f}, other "
              f"{(len(loop) - sum(pipe.values())) / R:.1f}; ptxas stall cycles {sum(st)} per column, "
              f"{st.count(2)} instructions with stall 2")
        print("   " + "  ".join(f"{op} {c / R:.2f}" for op, c in mix.most_common()))


if __name__ == "__main__":
    main()
