"""Deformable convolution on the CenterHead shape (1 x 64 x 468 x 468, 64 -> 64, 3x3, groups 4, N(0, 1.5^2)-pixel offsets):
ops.deform_conv2d forward, forward + backward and the backward alone, with achieved GB/s and FLOP/s from the counts below, the backward's
workspace bytes, and DCNSeparateHead forward + backward.  Comparator on the same GPU tensors: torchvision.ops.deform_conv2d when it imports,
else a dense torch formulation (grid_sample im2col + matmul); the tool prints which one ran and how far apart the results are.
CUDA events, median of 3 alternating rounds; the card name and power limit are read in the same run.  Writes OUT/dcn_bench.json.

    python tools/dcn_bench.py OUT
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, C, H, W, O, K, G = 1, 64, 468, 468, 64, 3, 4
REPS = 10


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # the numbers still stand beside the device name torch reports
        return [torch.cuda.get_device_name(0), f"unknown ({e})"]


def timed(fn):
    """median ms of REPS calls between CUDA events, after one warm-up call"""
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def dense_deform_conv2d(x, off, w, groups):
    """comparator without torchvision: bilinear im2col through grid_sample (zeros outside, align_corners=True = pixel-centre grid), then
    one matmul per group; stride 1, padding 1, dilation 1, one deformable group"""
    n, c, h, wd = x.shape
    k = w.shape[-1]
    ys, xs = torch.meshgrid(torch.arange(h, device=x.device), torch.arange(wd, device=x.device), indexing="ij")
    cols = []
    for t in range(k * k):
        i, j = divmod(t, k)
        ph = ys - 1 + i + off[:, 2 * t]
        pw = xs - 1 + j + off[:, 2 * t + 1]
        grid = torch.stack([pw / (wd - 1) * 2 - 1, ph / (h - 1) * 2 - 1], -1)
        cols.append(torch.nn.functional.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=True))
    col = torch.stack(cols, 2).view(n, groups, c // groups * k * k, h * wd)       # [n, G, Cg * K, HW] (c-major, tap-minor)
    wm = w.view(groups, -1, c // groups * k * k)
    return torch.einsum("gor,ngrp->ngop", wm, col).reshape(n, -1, h, wd)


def main(out_dir):
    assert torch.cuda.is_available(), "dcn_bench needs a GPU"
    from sst_b200 import ops
    from sst_b200.registry import MODELS
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(N, C, H, W, device=dev, generator=g)
    off = torch.randn(N, 2 * K * K, H, W, device=dev, generator=g) * 1.5
    w = torch.randn(O, C // G, K, K, device=dev, generator=g) / 12
    gy = torch.randn(N, O, H, W, device=dev, generator=g)
    geom = [N, C, H, W, O, K, K, 1, 1, 1, 1, 1, 1, G, 1]
    # counts: fp32 bytes the algorithm must move (inputs read once, outputs written once) and multiply-add FLOPs
    px = N * H * W
    fwd_bytes = 4 * (N * C * H * W + N * 2 * K * K * px + N * O * px + w.numel())
    bwd_bytes = 4 * (2 * N * C * H * W + 2 * N * 2 * K * K * px + N * O * px + 2 * w.numel())
    fwd_flop = 2 * px * O * (C // G) * K * K
    bwd_flop = 2 * fwd_flop                                                       # grad_col = W^T grad_y, grad_weight = grad_y S^T
    try:
        import torchvision
        comp_name = f"torchvision.ops.deform_conv2d ({torchvision.__version__})"
        comp = lambda a, o, ww: torchvision.ops.deform_conv2d(a, o, ww, None, 1, 1, 1)
    except Exception:
        comp_name = "dense torch formulation (grid_sample im2col + matmul)"
        comp = lambda a, o, ww: dense_deform_conv2d(a, o, ww, G)
    xr, orr, wr = (t.clone().requires_grad_(True) for t in (x, off, w))

    def ours_fb():
        xr.grad = orr.grad = wr.grad = None
        ops.deform_conv2d(xr, orr, wr, 1, 1, 1, G, 1).backward(gy)

    def comp_fb():
        xr.grad = orr.grad = wr.grad = None
        comp(xr, orr, wr).backward(gy)

    runs = {"fwd": [], "fwd_bwd": [], "bwd": [], "comp_fwd": [], "comp_fwd_bwd": []}
    for _ in range(3):
        runs["fwd"].append(timed(lambda: ops.deform_conv2d(x, off, w, 1, 1, 1, G, 1)))
        runs["comp_fwd"].append(timed(lambda: comp(x, off, w)))
        runs["fwd_bwd"].append(timed(ours_fb))
        runs["comp_fwd_bwd"].append(timed(comp_fb))
        runs["bwd"].append(timed(lambda: ops.deform_conv2d_backward(x, off, w, gy, geom)))
    med = {k: sorted(v)[1] for k, v in runs.items()}
    y = ops.deform_conv2d(x, off, w, 1, 1, 1, G, 1)
    yc = comp(x, off, w)
    ours_fb()
    ours_g = [t.grad.clone() for t in (xr, orr, wr)]
    comp_fb()
    comp_g = [t.grad.clone() for t in (xr, orr, wr)]
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    diffs = {"y": rel(y, yc), "grad_x": rel(ours_g[0], comp_g[0]), "grad_offset": rel(ours_g[1], comp_g[1]),
             "grad_weight": rel(ours_g[2], comp_g[2])}
    ws = ops.deform_conv2d_workspace_bytes(x, off, w, 1, 1, 1, G, 1)
    # DCNSeparateHead of configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py (one 3-class task), forward + backward, train mode
    heads = dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2), heatmap=(3, 2))
    head = MODELS.build(dict(type="DCNSeparateHead", init_bias=-2.19, final_kernel=3, in_channels=64, heads=heads, num_cls=3,
                             dcn_config=dict(type="DCN", in_channels=64, out_channels=64, kernel_size=3, padding=1, groups=4, bias=False),
                             norm_cfg=dict(type="naiveSyncBN2d", eps=1e-3, momentum=0.01))).to(dev).train()
    xh = x.clone().requires_grad_(True)

    def head_fb():
        head.zero_grad(set_to_none=True)
        sum(v.float().square().mean() for v in head(xh).values()).backward()

    head_ms = sorted(timed(head_fb) for _ in range(3))[1]
    name, power = card()
    res = {
        "card": name, "power_limit": power, "shape": [N, C, H, W, O, K, G], "comparator": comp_name,
        "fwd_ms": med["fwd"], "fwd_GBps": fwd_bytes / med["fwd"] / 1e6, "fwd_TFLOPs": fwd_flop / med["fwd"] / 1e9,
        "fwd_bwd_ms": med["fwd_bwd"], "bwd_ms": med["bwd"], "bwd_GBps": bwd_bytes / med["bwd"] / 1e6,
        "bwd_TFLOPs": bwd_flop / med["bwd"] / 1e9, "bwd_workspace_bytes": ws,
        "comparator_fwd_ms": med["comp_fwd"], "comparator_fwd_bwd_ms": med["comp_fwd_bwd"], "max_rel_diff_vs_comparator": diffs,
        "dcn_separate_head_fwd_bwd_ms": head_ms, "rounds_ms": runs,
        "counts": {"fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes, "fwd_flop": fwd_flop, "bwd_flop": bwd_flop},
    }
    print(json.dumps(res, indent=1))
    with open(os.path.join(out_dir, "dcn_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
