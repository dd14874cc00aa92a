"""BASELINE config 5 (front part): FSDv2 virtual-voxel front at nuScenes shape - 30k real points x batch 16 (+ 2k voted centres per
sample), 67-dim point features into DynamicScatterVFE [64,128], multiscale fusion with three coarse levels - through
sst_b200.fsdv2_modules.VirtualVoxelFront on one GPU: first everything `SingleStageFSDV2.extract_feat` does before and after its
`self.backbone(...)` call (identity mixer), then the whole extract_feat with the configs/fsdv2 VirtualVoxelMixer (sparse-conv U-Net,
SURVEY 8f next-1; spconv_modules.py) in both precisions.

    python tools/fsdv2_front_bench.py > fsdv2_config5.json"""
import json
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sst_b200.fsdv2_modules import VirtualVoxelFront  # noqa: E402
from sst_b200 import spconv_modules as SP  # noqa: E402

dev = torch.device("cuda:0")
B, P, V = 16, 30000, 2000
VS, RNG, TGT = (0.4, 0.4, 0.4), [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], [20, 270, 270]
norm = dict(type="naiveSyncBN1d", eps=1e-3, momentum=0.01)
m = VirtualVoxelFront(
    voxel_encoder=dict(type="DynamicScatterVFE", in_channels=67, feat_channels=[64, 128], with_cluster_center=True, with_voxel_center=True,
                       voxel_size=VS, point_cloud_range=RNG, norm_cfg=norm, unique_once=True, rel_dist_scaler=10.0),
    virtual_point_projector=dict(in_channels=75 + 64, hidden_dims=[64, 64], norm_cfg=norm, ori_in_channels=67 + 64, ori_hidden_dims=[64, 64]),
    multiscale_cfg=dict(multiscale_levels=[0, 1, 2], projector_hiddens=[[256, 128], [128, 128], [128, 128]], fusion_mode="avg",
                        target_sparse_shape=TGT, norm_cfg=norm),
    # configs/fsdv2/fsdv2_nusc_1x.py:142-154 (sparse_shape follows this bench's 0.4 m grid)
    backbone=dict(type="VirtualVoxelMixer", in_channels=128, sparse_shape=TGT, order=("conv", "norm", "act"), norm_cfg=norm, base_channels=64,
                  output_channels=128, encoder_channels=((64,), (64, 64), (64, 64)), encoder_paddings=((1,), (1, 1), (1, 1)),
                  decoder_channels=((64, 64, 64), (64, 64, 64), (64, 64, 64)), decoder_paddings=((1, 1), (1, 1), (1, 1)))).eval().to(dev)
g = torch.Generator().manual_seed(0)
lo, hi = torch.tensor(RNG[:3]), torch.tensor(RNG[3:])


def pts(n):
    r = torch.rand(n, 3, generator=g)
    r[:, :2] = 0.5 + (r[:, :2] - 0.5) * r[:, 2:3] ** 0.5   # denser towards the sensor
    return torch.cat([lo + (hi - lo) * (r * 0.98 + 0.01), torch.rand(n, 2, generator=g)], 1)


origin = dict(seg_points=pts(B * P), seg_feats=torch.randn(B * P, 131, generator=g), batch_idx=torch.arange(B).repeat_interleave(P))
sp = pts(B * V)
sampled = dict(seg_points=sp, center_preds=sp[:, :3] + torch.randn(B * V, 3, generator=g), seg_logits=torch.randn(B * V, 6, generator=g),
               seg_feats=torch.randn(B * V, 128, generator=g), batch_idx=torch.arange(B).repeat_interleave(V))
origin = {k: v.to(dev) for k, v in origin.items()}
sampled = {k: v.to(dev) for k, v in sampled.items()}
levels = []
for fin, shp, n in ((256, [20, 270, 270], 60000), (128, [10, 135, 135], 30000), (128, [5, 67, 67], 12000)):
    cells = torch.randperm(B * shp[0] * shp[1] * shp[2], generator=g)[:n]
    vol = shp[0] * shp[1] * shp[2]
    b, r = cells // vol, cells % vol
    idx = torch.stack([b, r // (shp[1] * shp[2]), (r // shp[2]) % shp[1], r % shp[2]], 1).int()
    levels.append(types.SimpleNamespace(features=torch.randn(n, fin, generator=g).to(dev), indices=idx.to(dev), spatial_shape=shp))
# (level 2's 67-cell axes do not divide 270: the reference asserts equal bev strides; use a level that does)
levels[2].spatial_shape = [5, 54, 54]
levels[2].indices = levels[2].indices % torch.tensor([B, 5, 54, 54], dtype=torch.int32, device=dev)


def step():
    with torch.no_grad():
        fr = m.front({k: v.clone() for k, v in sampled.items()}, origin, levels)
        return m.finish(fr, fr["voxel_feats"], fr["voxel_coors"]), fr


def full():
    with torch.no_grad():
        return m.extract_feat({k: v.clone() for k, v in sampled.items()}, origin, None, levels)


def timed(fn, reps=10):
    for _ in range(3):
        r = fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return r, ts


(out, fr), times = timed(step)
e2e = {}
for prec in ("fp32", "bf16", "fp32_tc"):
    SP.set_spconv_precision(m, prec)
    o, ts = timed(full)
    e2e[prec] = {"ms_median": ts[len(ts) // 2], "ms_min": ts[0], "frames_per_s": B / (ts[len(ts) // 2] * 1e-3),
                 "virtual_voxels": int(o["virtual_coors"].shape[0])}
print(json.dumps({"workload": "config 5 front: FSDv2 extract_feat without the sparse-conv mixer, 16 x (30k points + 2k votes), 0.4 m voxels, "
                              "67-dim VFE input, 3-level multiscale fusion", "ms_median": times[len(times) // 2], "ms_min": times[0],
                  "points": B * (P + V), "voxels": int(fr["voxel_coors"].shape[0]), "virtual_voxels": int(out["virtual_coors"].shape[0]),
                  "frames_per_s": B / (times[len(times) // 2] * 1e-3),
                  "with_mixer": dict(workload="config 5 end to end: extract_feat incl. VirtualVoxelMixer (configs/fsdv2 channels, 3 stages)", **e2e),
                  "note": "module API (stream launches, torch cat / projector MLPs through cuBLAS); not graph-captured"}))
