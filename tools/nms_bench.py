"""CUDA-event timing of rotated BEV NMS: this library (ops.box3d_multiclass_nms / ops.nms_gpu -> sstb200_nms_bev) against the reference's
own iou3d build (oracle/_ref/iou3d_ref*.so, driven by the reference's Python wrappers restated in oracle/iou3d_oracle.py), alternated in
one process, median of the rounds.  Every call includes its host round trip (both implementations return a host-sized result).
Prints the card name and power limit read in the same run; writes OUT/nms_bench.json.  `python tools/nms_bench.py [--rounds R]`
Workloads: (1) FSD-shaped box3d_multiclass_nms, 3 classes x 2 samples (one call per sample) at 2k and 20k boxes per sample;
(2) CenterHead-shaped nms_gpu, 10k boxes, pre_maxsize 4096, post_max_size 500; (3) one nms_gpu over 20k boxes."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

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


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nms_bench needs a CUDA device")
    from oracle import build_ref, iou3d_oracle as IO
    from sst_b200 import ops
    R = build_ref.load_module("iou3d_ref")
    if R is None:
        raise SystemExit("oracle/_ref/iou3d_ref*.so not built (python -m oracle.build_ref_iou3d)")

    def ref_nms(boxes, scores, thresh, pre_maxsize=None, post_max_size=None, rotated=True):
        order = scores.sort(0, descending=True)[1]
        if pre_maxsize is not None:
            order = order[:pre_maxsize]
        b = boxes[order].contiguous()
        keep = torch.zeros(b.size(0), dtype=torch.long)
        num = (R.nms_gpu if rotated else R.nms_normal_gpu)(b, keep, float(thresh), b.device.index)
        keep = order[keep[:num].cuda(b.device)].contiguous()
        return keep[:post_max_size] if post_max_size is not None else keep

    cfg = types.SimpleNamespace(use_rotate_nms=True, nms_thr=[0.25, 0.1, 0.1])
    work = {}
    for n in (2000, 20000):
        samples = []
        for s in range(2):
            bfn = IO.synth_boxes(60 + s + n, n, objects=max(1, n // 20)).cuda()
            scores = torch.rand(n, 4, generator=torch.Generator().manual_seed(70 + s + n)).cuda()
            samples.append((torch.rand(n, 7, device="cuda"), bfn, scores))
        work[f"fsd_multiclass_3cls_2samples_{n}"] = (
            lambda smp=samples: [ops.box3d_multiclass_nms(b, f, sc, 0.1, 500, cfg) for b, f, sc in smp],
            lambda smp=samples: [IO.box3d_multiclass_nms(b, f, sc, 0.1, 500, cfg, nms_gpu=ref_nms) for b, f, sc in smp])
    b10, s10 = IO.synth_boxes(80, 10000, objects=500).cuda(), torch.rand(10000, device="cuda")
    work["centerhead_nms_gpu_10k_pre4096_post500"] = (lambda: ops.nms_gpu(b10, s10, 0.2, 4096, 500),
                                                      lambda: ref_nms(b10, s10, 0.2, 4096, 500))
    b20, s20 = IO.synth_boxes(81, 20000, objects=1000).cuda(), torch.rand(20000, device="cuda")
    work["nms_gpu_20k"] = (lambda: ops.nms_gpu(b20, s20, 0.25), lambda: ref_nms(b20, s20, 0.25))
    rows = {k: {"sstb200": [], "reference": []} for k in work}
    same = {}
    for _ in range(a.rounds):
        for k, (ours, ref) in work.items():
            t0, o = timed(ours, a.iters)
            t1, r = timed(ref, a.iters)
            rows[k]["sstb200"].append(t0)
            rows[k]["reference"].append(t1)
            flat = lambda x: torch.cat([t.flatten().float() for t in (x if isinstance(x, list) else [x]) for t in (t if isinstance(t, tuple) else (t,))])
            same[k] = bool(torch.equal(flat(o), flat(r)))
    name, power = card()
    res = {"gpu": name, "power_limit_and_max_sm_clock": power, "rounds": a.rounds, "iters_per_round": a.iters, "same_result": same,
           "ms_per_call": {k: {impl: statistics.median(v) for impl, v in d.items()} for k, d in rows.items()}, "rounds_ms": rows}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "nms_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{name}, power limit / max SM clock {power}; median of {a.rounds} alternating rounds x {a.iters} calls")
    for k, d in res["ms_per_call"].items():
        print(f"  {k}: sstb200 {d['sstb200']:.3f} ms, reference {d['reference']:.3f} ms, x{d['reference'] / d['sstb200']:.1f}, "
              f"same result: {same[k]}")


if __name__ == "__main__":
    main()
