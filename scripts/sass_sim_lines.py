#!/usr/bin/env python
"""Control-flow and convergence instructions of one fused-search instantiation, per CUDA source line, from the SASS alone.

Disassembles a library or cubin built with -lineinfo (nvdisasm -gi: every instruction carries its chain of inlined
source locations) and counts, for one function (default: the headline CartPole instantiation
fc_search_kernel<16, false, CartPoleShape, 1>), per source line:
    ENDC   ENDCOLLECTIVE      the end of a divergent-collective fallback (ptxas could not prove the warp converged)
    WSYNC  WARPSYNC           (WARPSYNC.COLLECTIVE included)
    BDIV   BRA.DIV            the run-time "is the warp diverged?" test in front of such a collective
    BSSY   BSSY / BSYNC       reconvergence points of a divergent branch (counted once per pair, BSSY)
    BRA    BRA                every branch, BRA.DIV included
    AIMAD  IMAD (not .MOV) whose result is an address: its register is read inside the [...] of a load, store or atomic
           before it is overwritten, within the same basic block
The source line is the innermost location in the project's own files (CUDA headers skipped), and each instruction falls
into a region by its location in fc_search.cu's kernel body: setup (before the game loop), root, simulation loop,
write-out.  Runs on a CPU.

    python scripts/sass_sim_lines.py [LIB_OR_CUBIN] [--function SUBSTRING] [--region sim] [--top 40] [--json OUT]
"""
import argparse
import collections
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADLINE = "fc_search_kernelILi16ELb0ENS_12FcFixedShapeILi8ELi16ELi10ELi2EEELi1EEE"
KERNEL_FILE = "fc_search.cu"
COUNTS = ("ENDC", "WSYNC", "BDIV", "BSSY", "BRA", "AIMAD")
MEM_OPS = ("LD", "ST", "LDS", "STS", "LDG", "STG", "ATOM", "ATOMS", "RED", "LDL", "STL", "LDSM")


def _tool(name):
    cuda_bin = "/usr/local/cuda/bin"
    try:
        from muzero_general_b200 import build as b
        cuda_bin = os.path.dirname(b.NVCC)
    except ImportError:
        pass
    exe = os.path.join(cuda_bin, name)
    return exe if os.path.exists(exe) else shutil.which(name)


def kernel_regions(src):
    """{region: (first line, last line)} of fc_search_kernel's game loop, from the comment rulers in its body."""
    lines = open(src).read().splitlines()
    start = next(i for i, l in enumerate(lines) if "__global__" in l and "fc_search_kernel(" in l) + 1
    end = next(i for i in range(start, len(lines)) if lines[i].startswith("}")) + 1
    mark = {}
    for i in range(start, end):
        for name, tag in (("root", "-- root"), ("sim", "-- simulations"), ("out", "-- results")):
            if tag in lines[i]:
                mark[name] = i + 1
        if "for (int g0 =" in lines[i] and "loop" not in mark:
            mark["loop"] = i + 1
    return {"setup": (start, mark["loop"]), "root": (mark["loop"] + 1, mark["sim"] - 1),
            "sim": (mark["sim"], mark["out"] - 1), "out": (mark["out"], end)}


def disassemble(path):
    """[(mangled function, [(offset, opcode text, [(file, line) innermost first])])] of every kernel in the binary."""
    if path.endswith(".cubin"):
        cubins = [path]
        tmp = None
    else:
        import tempfile
        tmp = tempfile.mkdtemp()
        subprocess.run([_tool("cuobjdump"), "-xelf", "all", os.path.abspath(path)], cwd=tmp, check=True,
                       capture_output=True)
        cubins = [os.path.join(tmp, f) for f in sorted(os.listdir(tmp)) if f.endswith(".cubin")]
    out = []
    for cb in cubins:
        dis = subprocess.run([_tool("nvdisasm"), "-gi", cb], capture_output=True, text=True, check=True).stdout
        fn, insts, chain, fresh = None, None, [], True
        for ln in dis.splitlines():
            if ln.startswith(".text."):
                fn = ln[len(".text."):].rstrip(":")
                insts = []
                out.append((fn, insts))
                continue
            if fn is None:
                continue
            m = re.match(r'\s*//## File "([^"]+)", line (\d+)', ln)
            if m:
                if fresh:
                    chain, fresh = [], False
                chain.append((os.path.basename(m.group(1)), int(m.group(2))))
                continue
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(\S.*?)\s*;", ln)
            if m:
                insts.append((int(m.group(1), 16), m.group(2), list(chain)))
                fresh = True
    if tmp:
        shutil.rmtree(tmp, ignore_errors=True)
    return out


def _opcode(text):
    t = re.sub(r"^@!?U?P[T0-9]\s+", "", text)
    return t.split()[0] if t.split() else ""


def _address_imads(insts):
    """indices of the IMADs whose destination is next read inside a memory operand's brackets (same basic block)"""
    hits = set()
    for i, (_, text, _) in enumerate(insts):
        op = _opcode(text)
        if not op.startswith("IMAD") or op.startswith("IMAD.MOV"):
            continue
        parts = re.sub(r"^@!?U?P[T0-9]\s+", "", text).split(None, 1)
        if len(parts) < 2:
            continue
        dst = parts[1].split(",")[0].strip()
        if not re.fullmatch(r"R\d+", dst):
            continue
        pat = re.compile(r"\b" + dst + r"\b")
        for j in range(i + 1, min(i + 64, len(insts))):
            tj = insts[j][1]
            if tj.startswith(".L_") or _opcode(tj) in ("BRA", "EXIT", "RET", "BSYNC", "BSSY"):
                break
            opj = _opcode(tj).split(".")[0]
            brackets = re.findall(r"\[([^\]]*)\]", tj)
            if opj in MEM_OPS and any(pat.search(b) for b in brackets):
                hits.add(i)
                break
            if pat.search(tj):              # read as data first, or overwritten
                break
    return hits


def classify(text):
    op = _opcode(text)
    c = []
    if op == "ENDCOLLECTIVE":
        c.append("ENDC")
    if op.startswith("WARPSYNC"):
        c.append("WSYNC")
    if op == "BSSY":
        c.append("BSSY")
    if op.startswith("BRA"):
        c.append("BRA")
        if op.startswith("BRA.DIV"):
            c.append("BDIV")
    return c


def count(path, function=HEADLINE, src=None):
    src = src or os.path.join(ROOT, "muzero_general_b200", "csrc", KERNEL_FILE)
    regions = kernel_regions(src)
    fns = [(f, ins) for f, ins in disassemble(path) if function in f]
    if len(fns) != 1:
        raise SystemExit(f"{len(fns)} functions match {function!r}")
    fn, insts = fns[0]
    aimad = _address_imads(insts)
    per_line = collections.defaultdict(collections.Counter)
    per_region = collections.defaultdict(collections.Counter)
    for i, (_, text, chain) in enumerate(insts):
        kinds = classify(text) + (["AIMAD"] if i in aimad else [])
        own = [loc for loc in chain if not loc[0].endswith(".hpp") and not loc[0].endswith(".h")]
        inner = own[0] if own else (chain[0] if chain else ("?", 0))
        outer = [loc for loc in chain if loc[0] == KERNEL_FILE]
        kline = outer[-1][1] if outer else 0
        region = next((r for r, (a, b) in regions.items() if a <= kline <= b), "other")
        per_region[region]["inst"] += 1
        for k in kinds:
            per_line[(region, inner)][k] += 1
            per_region[region][k] += 1
    return fn, len(insts), per_region, per_line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("binary", nargs="?", default=None, help="library or cubin (default: the built libmzb200.so)")
    ap.add_argument("--function", default=HEADLINE)
    ap.add_argument("--region", default="sim", help="region whose per-line table is printed (setup, root, sim, out)")
    ap.add_argument("--top", type=int, default=60)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    path = args.binary
    if path is None:
        sys.path.insert(0, ROOT)
        from muzero_general_b200 import build as b
        path = b.LIB
    fn, n, per_region, per_line = count(path, args.function)
    print(f"{fn}: {n} instructions")
    print(f"{'region':8s} {'inst':>6s} " + " ".join(f"{k:>6s}" for k in COUNTS))
    for r in ("setup", "root", "sim", "out", "other"):
        if r in per_region:
            print(f"{r:8s} {per_region[r]['inst']:6d} " + " ".join(f"{per_region[r][k]:6d}" for k in COUNTS))
    rows = [(loc, c) for (r, loc), c in per_line.items() if r == args.region]
    rows.sort(key=lambda x: (-sum(x[1].values()), x[0]))
    print(f"\nregion {args.region}, per source line (innermost location in the project's files):")
    print(f"| {'source line':28s} | " + " | ".join(f"{k:>5s}" for k in COUNTS) + " |")
    print("|" + "---|" * (len(COUNTS) + 1))
    for loc, c in rows[:args.top]:
        print(f"| {loc[0] + ':' + str(loc[1]):28s} | " + " | ".join(f"{c[k]:5d}" for k in COUNTS) + " |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"function": fn, "instructions": n,
                       "regions": {r: dict(c) for r, c in per_region.items()},
                       "lines": [{"region": r, "file": loc[0], "line": loc[1], **dict(c)}
                                 for (r, loc), c in sorted(per_line.items())]}, f, indent=1)


if __name__ == "__main__":
    main()
