"""Per-epilogue SASS instruction budget of the fused SRA chain (csrc/sra_chain2.cu), on the CPU.

Compiles sra_chain2.cu with the library's build flags for sm_90a, disassembles it with line information (nvdisasm
--print-line-info) and splits each sra_chain2_kernel instantiation by its loop structure (backward branches): the tile loop
and, inside it, the `#pragma unroll 1` stage loops.  E1 (GEMM1 + Norm1) runs from the tile loop's head to the GEMM2 loop,
E2 (GEMM2 + GELU) is that loop, two trips per tile, E3 (GEMM3 + Norm2, y stores) runs to the GEMM4 loop or the end of the
tile loop, and E4 (GEMM4 + q|k|v stores, tail only) is the GEMM4 loop, three trips.  Static counts times the trip count
give the instructions one thread issues per 128-row tile, by opcode class.  Code laid out after the tile loop (mbarrier
wait retries, the early exit) is listed as out of line.

Every instruction of a stage counts once per trip, also the ones behind a uniform branch.  The normalisation of LayerNorm
and of folded BatchNorm layers are such branches: lines inside `if (affine) {...}` run only for BatchNorm layers and lines
inside `if (!affine) {...}` only for LayerNorm layers, so the tool keeps them apart and prints the stream of a LayerNorm
layer (the flagship's) and of a BatchNorm layer.  Masked stores and the elected thread's barrier and TMA work count in full.

    python tools/chain_sass_budget.py                 # the working tree
    python tools/chain_sass_budget.py --rev HEAD~1    # the sources of a git revision, side by side with the working tree
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sst_b200 import build as B  # noqa: E402

SRC = "sst_b200/csrc/sra_chain2.cu"
STAGES = ("prologue", "E1", "E2", "E3", "E4", "out of line")
TRIPS = {"prologue": 0, "E1": 1, "E2": 2, "E3": 1, "E4": 3, "out of line": 0}   # per tile; 0: not part of the tile stream
CLASSES = [
    ("HGMMA", ("HGMMA", "WARPGROUP")),
    ("MUFU", ("MUFU",)),
    ("FADD", ("FADD",)),
    ("FMUL", ("FMUL",)),
    ("FFMA", ("FFMA",)),
    ("fp other", ("FMNMX", "FSETP", "FSEL", "FCHK", "FRND", "FSWZADD")),
    ("convert", ("F2FP", "F2F", "F2I", "I2F", "I2FP", "F2IP")),
    ("shuffle", ("SHFL",)),
    ("global", ("LDG", "STG", "LD", "ST", "RED", "ATOM")),
    ("shared", ("LDS", "STS", "LDSM", "STSM", "ATOMS")),
    ("const", ("LDC", "ULDC")),
    ("sync/tma", ("BAR", "SYNCS", "UTMALDG", "UTMASTG", "UBLKCP", "UTMACMDFLUSH", "FENCE", "MEMBAR", "DEPBAR", "WARPSYNC", "ACQBULK",
                  "PREEXIT", "ELECT", "UTMAPF", "CCTL", "ERRBAR")),
    ("control", ("BRA", "BSSY", "BSYNC", "EXIT", "RET", "CALL", "YIELD", "BPT", "NANOSLEEP", "VOTE", "VOTEU", "PLOP3")),
]


def op_class(op):
    for name, ops in CLASSES:
        if op in ops:
            return name
    return "int/addr/other"


def norm_branches(src_lines):
    """{line: "bn_only" | "ln_only"} for the lines of the uniform `if (affine)` / `if (!affine)` normalisation branches"""
    branch = {}
    for i, l in enumerate(src_lines, 1):
        m = re.search(r"if \((!?)affine\) \{", l)
        if not m:
            continue
        depth, j = 0, i
        while True:
            depth += src_lines[j - 1].count("{") - src_lines[j - 1].count("}")
            if depth == 0:
                break
            j += 1
        for k in range(i, j + 1):
            branch[k] = "ln_only" if m.group(1) else "bn_only"
    return branch


def budget(src_root, work):
    path = os.path.join(src_root, SRC)
    cubin = os.path.join(work, "chain.cubin")
    flags = [f for f in B.FLAGS if f not in ("-Xcompiler", "-fPIC")]
    res = subprocess.run([B.NVCC] + flags + ["-I", os.path.join(src_root, "include"), "-Xptxas", "-v", "-cubin", path, "-o", cubin],
                         check=True, capture_output=True, text=True)
    regs = {}
    cur = None
    for l in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", l)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        if m and cur:
            regs.setdefault(cur, {})["spill"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", l)
        if m and cur:
            regs.setdefault(cur, {})["regs"] = int(m.group(1))
    nvdisasm = os.path.join(os.path.dirname(B.NVCC), "nvdisasm")
    sass = subprocess.run([nvdisasm, "--print-line-info", "-c", cubin], check=True, capture_output=True, text=True).stdout
    with open(path) as f:
        src_lines = f.read().splitlines()
    branch = norm_branches(src_lines)
    fns = {}
    fn, fline, ffile = None, 0, ""
    for l in sass.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", l)
        if m:
            fn = m.group(1) if "sra_chain2_kernel" in m.group(1) else None
            if fn:
                fns[fn] = ([], {})
            continue
        if fn is None:
            continue
        ins, labels = fns[fn]
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', l)
        if m:
            ffile, fline = m.group(1), int(m.group(2))
            continue
        m = re.match(r"(\.L_x_\d+):", l.strip())
        if m:
            labels[m.group(1)] = len(ins)
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)(.*)", l)
        if m:
            tag = branch.get(fline, "") if os.path.basename(ffile) == os.path.basename(SRC) else ""
            ins.append((m.group(1), m.group(2), tag))
    out = {}
    for fn, (ins, labels) in fns.items():
        # loops = backward branches; the tile loop is the largest, the stage loops (E2, and E4 with the tail) the large ones
        # inside it (the small ones are mbarrier wait loops)
        loops = []
        for i, (op, rest, _) in enumerate(ins):
            m = re.search(r"(\.L_x_\d+)", rest) if op == "BRA" else None
            if m and labels.get(m.group(1), len(ins)) <= i:
                loops.append((labels[m.group(1)], i))
        tile = max(loops, key=lambda ab: ab[1] - ab[0])
        inner = sorted(ab for ab in loops if ab != tile and tile[0] <= ab[0] and ab[1] <= tile[1] and ab[1] - ab[0] >= 200)
        assert len(inner) == (2 if "ILb1E" in fn else 1), f"unexpected loop structure in {fn}: {inner}"
        bounds = [("prologue", 0, tile[0]), ("E1", tile[0], inner[0][0]), ("E2", inner[0][0], inner[0][1] + 1)]
        if len(inner) == 2:
            bounds += [("E3", inner[0][1] + 1, inner[1][0]), ("E4", inner[1][0], inner[1][1] + 1)]
        else:
            bounds += [("E3", inner[0][1] + 1, tile[1] + 1)]
        bounds += [("out of line", tile[1] + 1, len(ins))]
        out[fn] = collections.defaultdict(collections.Counter)
        for stage, a, b in bounds:
            for op, _, tag in ins[a:b]:
                if op != "NOP":
                    out[fn][(stage, tag)][op_class(op)] += 1
    return out, regs


def per_tile(counts, layer):
    """{stage: Counter(class -> instructions per thread per tile)} of a LayerNorm ('ln') or BatchNorm ('bn') layer"""
    skip = "bn_only" if layer == "ln" else "ln_only"
    res = {}
    for s in STAGES:
        c = collections.Counter()
        for (st, tag), cc in counts.items():
            if st == s and tag != skip:
                for k, v in cc.items():
                    c[k] += v * max(TRIPS[s], 1)
        res[s] = c
    return res


def short(fn):
    return "sra_chain2_kernel<true>" if "ILb1E" in fn else "sra_chain2_kernel<false>"


def report(label, data):
    counts, regs = data
    print(f"== {label}")
    for fn in sorted(counts):
        r = regs.get(fn, {})
        print(f"  {short(fn)}: {r.get('regs', '?')} registers, {r.get('spill', '?')} spill bytes")
        for layer in ("ln", "bn"):
            pt = per_tile(counts[fn], layer)
            classes = [c for c, _ in CLASSES] + ["int/addr/other"]
            print(f"    {'LayerNorm' if layer == 'ln' else 'BatchNorm'} layer, instructions per thread per tile (prologue, out of line: static)")
            print("      " + f"{'stage':12s}" + "".join(f"{c[:8]:>9s}" for c in classes) + f"{'total':>9s}")
            tot = 0
            for s in STAGES:
                c = pt[s]
                n = sum(c.values())
                if TRIPS[s]:
                    tot += n
                print("      " + f"{s + (' x' + str(TRIPS[s]) if TRIPS[s] > 1 else ''):12s}" + "".join(f"{c[k]:9d}" for k in classes) + f"{n:9d}")
            print(f"      per-tile stream (E1-E4): {tot}")


def tile_total(data, fn_key, layer):
    counts, _ = data
    fn = next(f for f in counts if short(f) == fn_key)
    pt = per_tile(counts[fn], layer)
    return sum(sum(pt[s].values()) for s in STAGES if TRIPS[s]), {s: sum(pt[s].values()) for s in STAGES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rev", default=None, help="also count the sources of this git revision and compare")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as work:
        cur = budget(ROOT, work)
        report("working tree", cur)
        if a.rev:
            old_root = os.path.join(work, "rev")
            os.makedirs(old_root)
            tar = subprocess.run(["git", "-C", ROOT, "archive", a.rev, "sst_b200/csrc", "include"], check=True, capture_output=True).stdout
            subprocess.run(["tar", "-x", "-C", old_root], input=tar, check=True)
            old = budget(old_root, work)
            report(a.rev, old)
            print(f"== {a.rev} -> working tree, instructions per thread per tile")
            for k in ("sra_chain2_kernel<true>", "sra_chain2_kernel<false>"):
                for layer in ("ln", "bn"):
                    t0, s0 = tile_total(old, k, layer)
                    t1, s1 = tile_total(cur, k, layer)
                    per = "  ".join(f"{s} {s0[s]}->{s1[s]}" for s in STAGES if TRIPS[s])
                    print(f"  {k:26s} {layer.upper()}: {t0} -> {t1} ({100 * (t1 - t0) / t0:+.1f} %)   {per}")


if __name__ == "__main__":
    main()
