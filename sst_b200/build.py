"""Build libsstb200.so (sm_90a only) in-tree with nvcc.  `python -m sst_b200.build [-f]`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsstb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-warn-spills"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    d = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    d.append(os.path.join(HERE, "..", "include", "sstb200.h"))
    return d


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(p) > t for p in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in sources():
        o = os.path.join(HERE, "build", os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if not force and os.path.exists(o) and os.path.getmtime(o) > max(os.path.getmtime(p) for p in _deps() if not p.endswith(".cu") or p == s):
            continue
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if out.strip():
            print(out)
        if p.returncode != 0:
            failed = True
            print(f"nvcc failed on {s}", file=sys.stderr)
    if failed:
        raise RuntimeError("libsstb200 build failed")
    subprocess.check_call([NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT] + objs + ["-lcudart"])
    return OUT


if __name__ == "__main__":
    build(force="-f" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
