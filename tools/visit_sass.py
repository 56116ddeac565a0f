#!/usr/bin/env python
"""Instruction mix of one visit of the shared-memory top walk (walk_top_kernel), read from the SASS; no GPU needed.

usage: tools/visit_sass.py [--source bvh_b200/csrc/traverse.cu] [--kernel '<false, false, 5>'] [--all]

Compiles traverse.cu to a cubin with the library's nvcc flags (bvh_b200/build.py), prints each walk_top_kernel instance's
registers, stack, spills and shared memory from ptxas, and splits the warp-step loop (VPC visits, then the vote on idle
lanes) into its instructions:
  * the loop is the innermost backward branch whose body holds the LDS.128 record loads;
  * the common path leaves out every region a forward branch in the loop jumps over and that contains a store (the leaf
    report: taken by 10 000 of 73 M visits in the benchmark);
  * "one visit" is the common path from the first LDS.128 of visit 2 to the first LDS.128 of visit 3 (VPC >= 3; otherwise the
    whole loop / VPC), i.e. a steady-state visit without the per-step vote.
Pipes on sm_90 (per SM sub-partition: 32 FP32 lanes, 16 INT32 lanes): FMA = FADD/FMUL/FFMA/IMAD*/VIADD (FP32 pipe); ALU =
FMNMX/FSETP/ISETP/SEL/LOP3/PLOP3/IADD3/LEA/SHF/MOV (2 issue cycles per warp instruction); MIO = loads, stores, constant loads,
votes, shuffles; BRANCH = BRA/BSSY/BSYNC/WARPSYNC.  These are the published SM layout, not a measurement.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from bvh_b200 import build as B  # noqa: E402

CUOBJDUMP = os.path.join(os.path.dirname(B.NVCC), "cuobjdump")
FMA = {"FADD", "FMUL", "FFMA", "IMAD", "IMUL", "VIADD", "IADD", "FSWZADD"}
ALU = {"FMNMX", "FSETP", "FSEL", "FSET", "ISETP", "SEL", "LOP3", "PLOP3", "IADD3", "LEA", "SHF", "MOV", "P2R", "R2P", "IMNMX",
       "VIMNMX", "IABS", "FLO", "PRMT", "CSET", "CSETP"}
MIO = {"LDS", "STS", "LDG", "STG", "LD", "ST", "LDC", "VOTE", "SHFL", "REDUX", "ATOM", "ATOMG", "ATOMS", "RED", "S2R", "CS2R", "BAR",
       "MEMBAR", "MATCH", "POPC", "NANOSLEEP", "LDL", "STL"}
BRANCH = {"BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT", "CALL", "RET", "BREAK", "BMOV", "YIELD", "JMP", "BRX"}
LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")


def pipe(op: str) -> str:
    base = op.split(".")[0]
    if base.startswith("U") and base not in ("UNKNOWN",):
        return "UNIFORM"
    for name, ops in (("FMA", FMA), ("ALU", ALU), ("MIO", MIO), ("BRANCH", BRANCH)):
        if base in ops:
            return name
    return "OTHER"


def compile_cubin(src: str, out: str) -> str:
    flags = [f for f in B.FLAGS if f != "-lineinfo"]
    cmd = [B.NVCC] + flags + ["-Xptxas", "-v", "-cubin", src, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(r.stdout + r.stderr)
    return r.stdout + r.stderr


def ptxas_info(log: str) -> dict:
    info, cur = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", ln)
        if m:
            cur = m.group(1)
            info[cur] = ln
            continue
        if cur and ("registers" in ln or "spill" in ln or "smem" in ln):
            info[cur] += "\n" + ln
    return info


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else list(names)


def functions(cubin: str) -> dict:
    out = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for ln in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = LINE.search(ln)
        if cur and m:
            pred = (m.group(2) or "").strip()
            funcs[cur].append((int(m.group(1), 16), pred, m.group(3), m.group(4).strip()))
    return funcs


def target(ins) -> int | None:
    m = re.match(r"(?:!?U?P\w+,\s*)?(0x[0-9a-f]+)", ins[3])
    return int(m.group(1), 16) if ins[2].startswith("BRA") and m else None


def step_loop(code):
    """(lo, hi) addresses of the innermost backward branch loop that contains LDS.128."""
    best = None
    for ins in code:
        t = target(ins)
        if t is None or t >= ins[0]:
            continue
        body = [i for i in code if t <= i[0] <= ins[0]]
        if any(i[2].startswith("LDS.128") for i in body) and (best is None or ins[0] - t < best[1] - best[0]):
            best = (t, ins[0])
    return best


def rare_regions(body):
    """Address ranges a forward conditional branch inside the body jumps over and that hold a store but no record load (leaf
    reports; a region around the whole visit, such as an idle-lane guard, holds the LDS.128 and stays on the common path)."""
    regions = []
    for ins in body:
        t = target(ins)
        if t is None or t <= ins[0] or not ins[1]:
            continue
        skipped = [i for i in body if ins[0] < i[0] < t]
        if any(i[2].startswith("STG") for i in skipped) and not any(i[2].startswith("LDS") for i in skipped):
            regions.append((ins[0] + 1, t - 1))
    return regions


def mix(instrs) -> Counter:
    return Counter(pipe(i[2]) for i in instrs)


def fmt(c: Counter) -> str:
    return "  ".join(f"{k} {c.get(k, 0):g}" for k in ("FMA", "ALU", "MIO", "BRANCH", "UNIFORM", "OTHER") if c.get(k, 0))


def report(name: str, pretty: str, code, vpc: int, ptx: str, verbose: bool):
    print(pretty)
    for ln in ptx.splitlines()[1:]:
        print("   ", ln.strip())
    loop = step_loop(code)
    if loop is None:
        print("    no warp-step loop with LDS.128 found")
        return
    body = [i for i in code if loop[0] <= i[0] <= loop[1]]
    rare = rare_regions(body)
    common = [i for i in body if not any(a <= i[0] <= b for a, b in rare)]
    print(f"    warp-step loop {loop[0]:#x}..{loop[1]:#x}: {len(body)} instructions, {len(common)} on the common path, "
          f"{len(rare)} leaf-report region(s) left out ({sum(1 for i in body if any(a <= i[0] <= b for a, b in rare))} instructions)")
    print(f"    step common path:  {fmt(mix(common))}")
    lds = [k for k, i in enumerate(common) if i[2].startswith("LDS.128")]
    firsts = lds[0::2]                                     # a visit loads its record with two LDS.128
    if vpc >= 3 and len(firsts) >= 3:
        visit = common[firsts[1]:firsts[2]]
        label = "one visit (visit 2 to visit 3)"
    else:
        visit = common
        label = f"one visit (step / {vpc})"
    c = mix(visit)
    if visit is common and vpc > 1:
        c = Counter({k: v / vpc for k, v in c.items()})
    total = sum(c.values())
    print(f"    {label}: {total:g} instructions: {fmt(c)}")
    ops = Counter(i[2].split(".")[0] for i in visit)
    print("    ops:", ", ".join(f"{k} {v}" for k, v in sorted(ops.items(), key=lambda kv: (-kv[1], kv[0]))))
    bssy = sum(1 for i in visit if i[2].startswith("BSSY"))
    bra = sum(1 for i in visit if i[2].startswith("BRA"))
    print(f"    convergence regions (BSSY) in the visit: {bssy}, branches: {bra}")
    if verbose:
        for i in visit:
            print(f"      {i[0]:#06x} {pipe(i[2]):7s} {i[1]:6s} {i[2]} {i[3]}")
    print()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--source", default=os.path.join(ROOT, "bvh_b200", "csrc", "traverse.cu"))
    ap.add_argument("--kernel", default="<false, false, 5>", help="template arguments of the instance to list (substring)")
    ap.add_argument("--all", action="store_true", help="every walk_top_kernel instance")
    ap.add_argument("-v", "--verbose", action="store_true", help="print the visit's instructions")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "traverse.cubin")
        ptx = ptxas_info(compile_cubin(os.path.abspath(a.source), cubin))
        funcs = functions(cubin)
    names = sorted(n for n in funcs if "walk_top_kernel" in n)
    for name, pretty in zip(names, demangle(names)):
        if not a.all and a.kernel not in pretty:
            continue
        m = re.search(r"walk_top_kernel<\w+, \w+, (\d+)>", pretty)
        vpc = int(m.group(1)) if m else 1
        report(name, pretty.split("(")[0], funcs[name], vpc, ptx.get(name, ""), a.verbose)


if __name__ == "__main__":
    main()
