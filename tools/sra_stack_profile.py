"""Per-kernel time of the bf16 SRA encoder stack (the 12-layer `sstb200_sra_stack_forward` call that bench.py's roofline times).

Builds the bench's engine (flagship SST-6 config, one 150k-point synthetic sweep, bf16), runs one frame through it, then calls the
stack exactly as bench.py's roofline section does: `--calls` times, each after a 512 MB L2 flush, recorded with torch.profiler
(CUDA activities) in a run of its own.  Writes per-kernel launch counts, total and median microseconds, the exclusive time (the
part of each launch after its predecessor ended; launches overlap under programmatic dependent launch), each kernel's share of
the stack's span, and the card's name and power limit (read in the same run) to OUT/sra_stack_profile.json.

    python tools/sra_stack_profile.py [--out DIR] [--calls 20] [--warmup 3] [--points 150000]
"""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return name, q or "unknown"


def short_name(n):
    # "void (anonymous namespace)::sra_chain2_kernel<true>(...)" -> "sra_chain2_kernel<true>"
    n = n.replace("(anonymous namespace)::", "").split("(")[0]
    return re.sub(r"^void ", "", n).strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="sra_stack_profile_out")
    ap.add_argument("--calls", type=int, default=20, help="profiled stack calls, each after an L2 flush")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=int, default=150000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sra_stack_profile.py needs a CUDA device")
    from sst_b200 import _lib as L, build, flagship as fl
    from sst_b200.engine import SSTEngine
    build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = fl.sst_cfg()
    vfe, il, bb = fl.build_sst(cfg)
    eng = SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe.to(dev), il, bb.to(dev), max_points=a.points, batch_size=1, precision="bf16", device=dev)
    eng.load_frames_device(fl.synth_frame(1000, a.points).to(dev), torch.tensor([0, a.points], dtype=torch.int32, device=dev))
    _, _, num = eng.run()
    torch.cuda.synchronize()
    voxels = int(num.item())
    nl = len(eng._layers)
    lib = L.lib()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    st = eng.stream

    def stack_call(c):
        L.check(c, lib.sstb200_sra_stack_forward(c, eng._layer_array, nl, C.byref(eng._plan_structs[0]), C.byref(eng._plan_structs[1]),
                                                 eng.vf.data_ptr(), eng.x[0].data_ptr(), eng.x[1].data_ptr(), eng.cap,
                                                 eng.num.data_ptr(), 1))

    with torch.cuda.stream(st):
        c = L.ctx(dev)
        for _ in range(a.warmup):
            flush.zero_()
            stack_call(c)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(st):
            for _ in range(a.calls):
                flush.zero_()
                stack_call(c)
        torch.cuda.synchronize()

    # Every kernel of the stack is launched with programmatic dependent launch: it may start while its predecessor still runs
    # and then wait in griddepcontrol.wait, so launches overlap and their durations add up to more than the stack's time.
    # "exclusive" is the part of a launch after its predecessor ended (end - max(start, previous end)); the exclusive times of
    # one call add up to its span.
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    per, prev_end = {}, None
    for e in evs:
        t0, t1 = e.time_range.start, e.time_range.end
        if "at::native" in e.name or "Memset" in e.name or "Memcpy" in e.name:
            prev_end = None   # the L2 flush (torch fill kernel) between calls, not part of the stack
            continue
        excl = t1 - (t0 if prev_end is None else max(t0, prev_end))
        prev_end = t1 if prev_end is None else max(prev_end, t1)
        d = per.setdefault(e.name, ([], []))
        d[0].append(t1 - t0)
        d[1].append(excl)
    kernels = {}
    for name, (ts, ex) in per.items():
        kernels[short_name(name)] = {"count": len(ts), "count_per_call": len(ts) / a.calls, "total_us": sum(ts),
                                     "median_us": statistics.median(ts), "exclusive_total_us": sum(ex),
                                     "exclusive_median_us": statistics.median(ex), "full_name": name}
    stack_us = sum(k["exclusive_total_us"] for k in kernels.values())
    for k in kernels.values():
        k["share_of_stack"] = k["exclusive_total_us"] / stack_us if stack_us else None
    name, power = card()
    res = {"gpu": name, "power_limit_and_max_sm_clock": power, "points": a.points, "voxels": voxels, "layers": nl, "calls": a.calls,
           "stack_span_us_per_call": stack_us / a.calls,
           "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["exclusive_total_us"]))}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "sra_stack_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{name}, power limit / max SM clock {power}: {voxels} voxels, {nl} layers, stack span {stack_us / a.calls:.1f} us per call")
    for n, k in res["kernels"].items():
        print(f"  {n:40s} x{k['count_per_call']:5.1f}/call  median {k['median_us']:8.2f} us  exclusive median {k['exclusive_median_us']:8.2f} us"
              f"  exclusive total {k['exclusive_total_us'] / a.calls:8.1f} us/call  {100 * k['share_of_stack']:5.1f} % of the span")


if __name__ == "__main__":
    main()
