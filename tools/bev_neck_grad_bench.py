"""CUDA-event timing of the two training hand-offs: SSTv2.recover_bev (csrc/bev.cu) at config 2 (B=1, C=128, 468 x 468, ~30k voxels of a
synthetic sweep) and Voxel2PointScatterNeck (csrc/neck.cu) at the FSD shape (150k points, ~30k voxels, C = 64 + 3 and 128 + 3), each as
forward + backward through autograd and as the backward call alone, beside a torch autograd formulation of the same ops on the same GPU
tensors (the reference's per-sample zero canvas + index_put, and its gather / mask / concat).  Achieved GB/s of the backward calls are
computed from byte counts in this script.  Prints the card name and power limit read in the same run; writes OUT/bev_neck_grad_bench.json.
`python tools/bev_neck_grad_bench.py [--iters K] [--out DIR]`"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return name, q or "unknown"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def torch_recover_bev(voxel_feat, coors, batch_size, ny, nx):
    """sst_v2.py:161-196 restated: one zero canvas per sample, index_put of the transposed rows, stack."""
    out = []
    for b in range(batch_size):
        canvas = voxel_feat.new_zeros(voxel_feat.shape[1], nx * ny)
        m = coors[:, 0] == b
        idx = (coors[m, 2] * nx + coors[m, 3]).long()
        canvas[:, idx] = voxel_feat[m].t()
        out.append(canvas)
    return torch.stack(out, 0).view(batch_size, voxel_feat.shape[1], ny, nx)


def torch_neck(points, pts_coors, voxel_feats, inds, padding=-1):
    """voxel2point_neck.py:28-62 restated (with_xyz, no normalisation)."""
    pts_feats = voxel_feats[inds]
    mask = ~((pts_feats == padding).all(1))
    pts_feats, pts_coors, points = pts_feats[mask], pts_coors[mask], points[mask]
    vs = torch.tensor(VS, device=points.device).reshape(1, 3)
    mn = torch.tensor(RNG[:3], device=points.device).reshape(1, 3)
    center = (pts_coors[:, [3, 2, 1]].float() + 0.5) * vs + mn
    return torch.cat([pts_feats, points[:, :3] - center], 1), mask


def voxelize(pts):
    """(b=0, z, y, x) int64 voxel coordinates of every point on the config grid, by the library's own dynamic_voxelize."""
    from sst_b200 import ops
    c = torch.empty((pts.shape[0], 3), dtype=torch.int32, device=pts.device)
    ops.dynamic_voxelize(pts.contiguous(), c, list(VS), RNG)
    return torch.nn.functional.pad(c.long(), (1, 0), value=0)


def fwd_bwd(fn, x, grad):
    def run():
        x.grad = None
        out = fn(x)
        out.backward(grad)
    return run


def median_rounds(fns, iters):
    rounds = []
    for _ in range(3):  # alternate the forms
        rounds.append([timed(f, iters) for f in fns])
    return [sorted(r[i] for r in rounds)[1] for i in range(len(fns))], rounds


def bench_bev(iters, dev):
    from sst_b200 import _lib as L
    from sst_b200.flagship import synth_frame
    from sst_b200.sst_modules import SSTv2
    B, Cc, ny, nx = 1, 128, 468, 468
    coors = torch.unique(voxelize(synth_frame(139, 100000).to(dev)), dim=0)
    M = coors.shape[0]
    feat = torch.randn(M, Cc, device=dev)
    grad = torch.randn(B, Cc, ny, nx, device=dev)
    m = SSTv2(d_model=[Cc], nhead=[1], num_blocks=0, dim_feedforward=[Cc], output_shape=[ny, nx], num_attached_conv=0, to_bev=True)
    x = feat.clone().requires_grad_(True)
    gx = torch.empty(M, Cc, device=dev)
    c = L.ctx(dev)
    bwd = lambda: L.check(c, L.lib().sstb200_recover_bev_backward(c, grad.data_ptr(), coors.data_ptr(), M, Cc, B, ny, nx, gx.data_ptr()))
    (t_op, t_torch, t_bwd), rounds = median_rounds([fwd_bwd(lambda v: m.recover_bev(v, coors, B), x, grad),
                                                    fwd_bwd(lambda v: torch_recover_bev(v, coors, B, ny, nx), x, grad), bwd], iters)
    segments = int(torch.unique(coors[:, 0] * ny * ((nx + 127) // 128) + coors[:, 2] * ((nx + 127) // 128) + coors[:, 3] // 128).numel())
    written, read_bound = M * Cc * 4, B * Cc * ny * nx * 4
    read = segments * Cc * min(nx, 128) * 4
    return {"shape": f"B={B} C={Cc} {ny}x{nx}", "voxels": M, "occupied_128_cell_segments": segments,
            "op_fwd_bwd_ms": t_op, "torch_fwd_bwd_ms": t_torch, "op_backward_ms": t_bwd,
            "backward_bytes_written": written, "backward_bytes_read": read, "backward_bytes_read_bound": read_bound,
            "backward_GBps": (written + read) / t_bwd / 1e6, "rounds_ms": rounds}


def bench_neck(iters, dev, Cc):
    from sst_b200 import _lib as L
    from sst_b200.flagship import synth_frame
    from sst_b200.neck_modules import Voxel2PointScatterNeck
    N, M = 150000, 30000
    g = torch.Generator().manual_seed(Cc)
    pts = synth_frame(3, N, extra_dims=1)
    coors = voxelize(pts[:, :3].to(dev))
    vf = torch.randn(M, Cc, generator=g)
    vf[::7] = -1.0
    inds = torch.randint(0, M, (N,), generator=g).to(dev)
    pts, vf = pts.to(dev), vf.to(dev)
    neck = Voxel2PointScatterNeck(point_cloud_range=RNG, voxel_size=VS, with_xyz=True)
    x = vf.clone().requires_grad_(True)
    out, mask = neck(pts, coors, x, inds)
    K = out.shape[0]
    grad = torch.randn(K, Cc + 3, device=dev)
    gx = torch.empty(M, Cc, device=dev)
    mask_u8 = mask.contiguous()
    c = L.ctx(dev)
    bwd = lambda: L.check(c, L.lib().sstb200_voxel2point_backward(c, grad.data_ptr(), mask_u8.data_ptr(), inds.data_ptr(), N, K, M, Cc, 1,
                                                                   gx.data_ptr()))
    (t_op, t_torch, t_bwd), rounds = median_rounds([fwd_bwd(lambda v: neck(pts, coors, v, inds)[0], x, grad),
                                                    fwd_bwd(lambda v: torch_neck(pts, coors, v, inds)[0], x, grad), bwd], iters)
    read, written = K * (Cc + 3) * 4, M * Cc * 4
    return {"shape": f"N={N} M={M} C={Cc}+3", "kept_points": K, "op_fwd_bwd_ms": t_op, "torch_fwd_bwd_ms": t_torch,
            "op_backward_ms": t_bwd, "backward_bytes_read": read, "backward_bytes_written": written,
            "backward_GBps": (read + written) / t_bwd / 1e6, "rounds_ms": rounds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="bev_neck_grad_bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bev_neck_grad_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"recover_bev": bench_bev(a.iters, dev), "neck_c64": bench_neck(a.iters, dev, 64), "neck_c128": bench_neck(a.iters, dev, 128)}
    name, power = card()
    res = {"gpu": name, "power_limit_and_max_sm_clock": power, **res}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bev_neck_grad_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{name}, power limit / max SM clock {power} | median of 3 alternating rounds")
    for k in ("recover_bev", "neck_c64", "neck_c128"):
        r = res[k]
        print(f"{k} ({r['shape']}): fwd+bwd {r['op_fwd_bwd_ms']:.3f} ms vs torch autograd {r['torch_fwd_bwd_ms']:.3f} ms | backward call "
              f"{r['op_backward_ms']:.3f} ms = {r['backward_GBps']:.0f} GB/s")


if __name__ == "__main__":
    main()
