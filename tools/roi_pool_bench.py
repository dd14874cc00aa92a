"""CUDA-event timing of FSD's RoI point pooling (ops.dynamic_point_pool -> sstb200_dynamic_point_pool) at the FSD second-stage shape
(100k points, 500 RoIs of car / pedestrian / cyclist size, extra_wlh 0.5, max_inbox_point 256), beside a dense torch formulation of the
same pooling on the same GPU tensors (every RoI against every point, fp32, then the first 256 hits per RoI).  Prints the card name and
power limit read in the same run; writes OUT/roi_pool_bench.json.  `python tools/roi_pool_bench.py [--points N] [--rois R] [--iters K]`"""
import argparse
import json
import math
import os
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


def dense_pool(rois, pts, extra, cap):
    """[R, N] box test in fp32 torch, first `cap` hits per RoI, the 13 features of the hits"""
    cx, cy, zb, w, l, h, rz = rois.unbind(1)
    ang = rz + math.pi / 2
    ca, sa = torch.cos(ang)[:, None], torch.sin(ang)[:, None]
    sx, sy = pts[None, :, 0] - cx[:, None], pts[None, :, 1] - cy[:, None]
    lx, ly = sx * ca - sy * sa, sx * sa + sy * ca
    cz = (zb + h / 2)[:, None]
    lz = pts[None, :, 2] - cz
    hl, hw, hh = ((l + extra[1]) / 2)[:, None], ((w + extra[0]) / 2)[:, None], ((h + extra[2]) / 2)[:, None]
    inside = (lz.abs() <= hh) & (lx.abs() < hl) & (ly.abs() < hw)
    keep = inside & (torch.cumsum(inside.int(), 1) <= cap)
    r, i = keep.nonzero(as_tuple=True)
    lxi, lyi, lzi = lx[r, i], ly[r, i], lz[r, i]
    half = torch.stack([l[r], w[r], h[r]], 1) / 2
    loc = torch.stack([lxi, lyi, lzi], 1)
    margin = ~((lzi.abs() <= half[:, 2]) & (lxi.abs() < half[:, 0]) & (lyi.abs() < half[:, 1]))
    return i, r, torch.cat([pts[i], loc, half + loc, half - loc, margin.float()[:, None]], 1)


def timed(fn, iters):
    for _ in range(3):
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
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--rois", type=int, default=500)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="roi_pool_bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("roi_pool_bench needs a CUDA device")
    from oracle import roi_pool_oracle as RO
    from sst_b200 import ops
    pts, rois, _, _ = RO.synth_roi_frame(11, n_pts=a.points, n_rois=a.rois)
    pts, rois = pts.cuda(), rois.cuda()
    extra, cap = [0.5, 0.5, 0.5], 256
    rows = []
    for _ in range(3):   # alternate the two forms
        t_op, got = timed(lambda: ops.dynamic_point_pool(rois, pts, extra, cap), a.iters)
        t_dense, dense = timed(lambda: dense_pool(rois, pts, extra, cap), max(a.iters // 5, 3))
        rows.append((t_op, t_dense))
    name, power = card()
    t_op = sorted(r[0] for r in rows)[1]
    t_dense = sorted(r[1] for r in rows)[1]
    res = {"gpu": name, "power_limit_and_max_sm_clock": power, "points": a.points, "rois": a.rois, "max_inbox_point": cap,
           "pairs_op": int(got[0].shape[0]), "pairs_dense": int(dense[0].shape[0]), "op_ms_median_of_3": t_op,
           "dense_torch_ms_median_of_3": t_dense, "rounds_ms": rows}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "roi_pool_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{name}, power limit / max SM clock {power}: {a.rois} RoIs x {a.points} points, {res['pairs_op']} pairs | "
          f"sstb200_dynamic_point_pool {t_op:.3f} ms per call (incl. the host round trip for the row count) | dense torch "
          f"{t_dense:.3f} ms ({res['pairs_dense']} pairs) | median of 3 alternating rounds")


if __name__ == "__main__":
    main()
