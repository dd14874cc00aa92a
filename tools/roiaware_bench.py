"""CUDA-event timing of mmdet3d/ops/roiaware_pool3d: this library (ops.points_in_boxes_gpu / _batch, ops.RoIAwarePool3dFunction) against
the reference's own roiaware_pool3d build (oracle/_ref/roiaware_pool3d_ext_ref*.so, driven as its Python wrappers drive it), alternated
in one process, median of the rounds.  Prints the card name and power limit read in the same run, the achieved write rate of
points_in_boxes_batch (B * M * T * 4 bytes) and the bytes each side saves for the backward; writes OUT/roiaware_bench.json.
`python tools/roiaware_bench.py [--rounds R]`
Workloads: points_in_boxes_gpu at 150k points x 200 and x 2000 boxes; points_in_boxes_batch at 20k x 64 and 150k x 200; PartA2-shaped
RoIAwarePool3d (2 samples x 16k points x 128 RoIs, out 14, m 128; C = 16 max and C = 4 avg), forward and forward + backward, one call
per sample on both sides."""
import argparse
import json
import os
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
        raise SystemExit("roiaware_bench needs a CUDA device")
    from oracle import build_ref, roi_pool_oracle as RO
    from sst_b200 import ops
    R = build_ref.load_module("roiaware_pool3d_ext_ref")
    if R is None:
        raise SystemExit("oracle/_ref/roiaware_pool3d_ext_ref*.so not built (python -m oracle.build_ref_roiaware)")

    def ref_pib(points, boxes, first):
        if first:
            out = points.new_zeros(points.shape[:2], dtype=torch.int).fill_(-1)
            R.points_in_boxes_gpu(boxes.contiguous(), points.contiguous(), out)
        else:
            out = points.new_zeros((*points.shape[:2], boxes.shape[1]), dtype=torch.int).fill_(0)
            R.points_in_boxes_batch(boxes.contiguous(), points.contiguous(), out)
        return out

    class RefPool(torch.autograd.Function):     # roiaware_pool3d.py:45-86 over the reference extension
        @staticmethod
        def forward(ctx, rois, pts, feats, out, m, mode):
            n, C = rois.shape[0], feats.shape[1]
            pooled = feats.new_zeros((n, out, out, out, C))
            argmax = feats.new_zeros((n, out, out, out, C), dtype=torch.int)
            pidx = feats.new_zeros((n, out, out, out, m), dtype=torch.int)
            R.forward(rois, pts, feats, argmax, pidx, pooled, mode)
            ctx.saved = (pidx, argmax, mode, pts.shape[0], C)
            return pooled

        @staticmethod
        def backward(ctx, g):
            pidx, argmax, mode, n, C = ctx.saved
            grad_in = g.new_zeros((n, C))
            R.backward(pidx, argmax, g.contiguous(), grad_in, mode)
            return None, None, grad_in, None, None, None

    saved = {}

    def saved_bytes(ctx_holder):
        return sum(t.numel() * t.element_size() for t in ctx_holder if torch.is_tensor(t))

    work, gbps = {}, {}
    pts, rois, _, _ = RO.synth_roi_frame(61, n_pts=150000, n_rois=2000, spread=40.0)
    P, B200, B2000 = pts[None].cuda(), rois[None, :200].cuda().contiguous(), rois[None].cuda()
    work["points_in_boxes_gpu_150k_x_200"] = (lambda: ops.points_in_boxes_gpu(P, B200), lambda: ref_pib(P, B200, True))
    work["points_in_boxes_gpu_150k_x_2000"] = (lambda: ops.points_in_boxes_gpu(P, B2000), lambda: ref_pib(P, B2000, True))
    P20, B64 = P[:, :20000].contiguous(), rois[None, :64].cuda().contiguous()
    work["points_in_boxes_batch_20k_x_64"] = (lambda: ops.points_in_boxes_batch(P20, B64), lambda: ref_pib(P20, B64, False))
    work["points_in_boxes_batch_150k_x_200"] = (lambda: ops.points_in_boxes_batch(P, B200), lambda: ref_pib(P, B200, False))
    gbps["points_in_boxes_batch_20k_x_64"] = 20000 * 64 * 4
    gbps["points_in_boxes_batch_150k_x_200"] = 150000 * 200 * 4
    samples = []
    for s in range(2):
        p, r, _, _ = RO.synth_roi_frame(70 + s, n_pts=16000, n_rois=128, spread=25.0)
        samples.append((p.cuda(), r.cuda()))
    for mode, C in ((0, 16), (1, 4)):
        feats = [torch.randn((16000, C), device="cuda") for _ in range(2)]
        name = f"roiaware_pool3d_parta2_{'max' if mode == 0 else 'avg'}_C{C}"

        def ours_fwd(mode=mode, feats=feats):
            return [ops.RoIAwarePool3dFunction.apply(r, p, f, 14, 128, mode) for (p, r), f in zip(samples, feats)]

        def ref_fwd(mode=mode, feats=feats):
            return [RefPool.apply(r, p, f, 14, 128, mode) for (p, r), f in zip(samples, feats)]

        def fwd_bwd(fn, feats=feats):
            fs = [f.clone().requires_grad_() for f in feats]
            outs = fn(feats=fs)
            torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
            return [f.grad for f in fs]

        work[name + "_forward"] = (ours_fwd, ref_fwd)
        work[name + "_forward_backward"] = (lambda f=ours_fwd: fwd_bwd(f), lambda f=ref_fwd: fwd_bwd(f))
        # bytes saved for the backward, per call over both samples
        s_ours = 0
        for (p, r), f in zip(samples, feats):
            _, st = ops.roiaware_pool3d_forward(r, p, f, 14, 128, mode)
            s_ours += saved_bytes(st)
        s_ref = 2 * 128 * 14 ** 3 * (128 + C) * 4
        saved[name] = {"sstb200": s_ours, "reference": s_ref}
    rows = {k: {"sstb200": [], "reference": []} for k in work}
    same = {}
    for _ in range(a.rounds):
        for k, (ours, ref) in work.items():
            t0, o = timed(ours, a.iters)
            t1, r = timed(ref, a.iters)
            rows[k]["sstb200"].append(t0)
            rows[k]["reference"].append(t1)
            flat = lambda x: torch.cat([t.flatten().float() for t in (x if isinstance(x, list) else [x])])
            fo, fr = flat(o), flat(r)
            same[k] = bool(torch.equal(fo, fr)) if "backward" not in k else bool(torch.allclose(fo, fr, rtol=1e-6, atol=1e-6))
    name, power = card()
    med = {k: {impl: statistics.median(v) for impl, v in d.items()} for k, d in rows.items()}
    res = {"gpu": name, "power_limit_and_max_sm_clock": power, "rounds": a.rounds, "iters_per_round": a.iters, "same_result": same,
           "ms_per_call": med, "rounds_ms": rows, "saved_bytes": saved,
           "write_GBps": {k: {impl: b / (med[k][impl] * 1e6) for impl in ("sstb200", "reference")} for k, b in gbps.items()}}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "roiaware_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{name}, power limit / max SM clock {power}; median of {a.rounds} alternating rounds x {a.iters} calls")
    for k, d in med.items():
        extra = ""
        if k in gbps:
            extra = f", write {res['write_GBps'][k]['sstb200']:.0f} GB/s vs {res['write_GBps'][k]['reference']:.0f} GB/s"
        print(f"  {k}: sstb200 {d['sstb200']:.3f} ms, reference {d['reference']:.3f} ms, x{d['reference'] / d['sstb200']:.1f}{extra}, "
              f"same result: {same[k]}")
    for k, d in saved.items():
        print(f"  {k}: bytes saved for backward (2 samples): sstb200 {d['sstb200']:,}, reference {d['reference']:,}")


if __name__ == "__main__":
    main()
