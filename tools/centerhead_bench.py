"""CenterHead's training path on the Waymo CenterHead geometry (1 task x 3 classes, 468 x 468, out_size_factor 1, max_objs 500), B = 2
and 4 samples of about 200 boxes each with a Waymo-like class mix (car 70 %, pedestrian 25 %, cyclist 5 %):
  native    CenterHead.get_targets alone, then get_targets + loss forward + backward (to the head outputs);
  baseline  the reference's per-box loop (centerpoint_head.py:421-552, with its host syncs and per-box numpy Gaussians) and its torch loss
            composition (clip_sigmoid, the elementwise Gaussian focal loss, permute + gather L1), restated here on the same GPU tensors.
Also the bytes each native loss pass moves (focal forward 8 B / element, backward 12 B / element) against the HBM bound of 3.35 TB/s
(H100 SXM data sheet).  CUDA events around each call (ended by a synchronise), median of 3 alternating rounds; the card name and power
limit are read in the same run.  Writes OUT/centerhead_bench.json.

    python tools/centerhead_bench.py [OUT]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
REPS = 5
CFG = dict(grid_size=[468, 468, 1], voxel_size=(0.32, 0.32, 6), out_size_factor=1, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
           min_radius=2, point_cloud_range=[-74.88, -74.88, -2, 74.88, 74.88, 4],
           code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0, 0.0])
HEAD = dict(in_channels=16, tasks=[dict(num_class=3, class_names=['car', 'pedestrian', 'cyclist'])],
            common_heads=dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)), share_conv_channel=16,
            separate_head=dict(type='SeparateHead', init_bias=-2.19, final_kernel=3),
            loss_cls=dict(type='GaussianFocalLoss', reduction='mean'), loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=2),
            train_cfg=CFG, norm_bbox=True)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:
        return [torch.cuda.get_device_name(0), f"unknown ({e})"]


def timed(fn):
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


def synth(B, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    boxes, labels = [], []
    for _ in range(B):
        n = 200
        lab = torch.multinomial(torch.tensor([0.70, 0.25, 0.05]), n, replacement=True, generator=g)
        size = torch.tensor([[2.0, 4.6, 1.7], [0.9, 0.9, 1.8], [0.8, 1.8, 1.7]])[lab] * (0.8 + 0.4 * torch.rand(n, 3, generator=g))
        xy = (torch.rand(n, 2, generator=g) * 2 - 1) * 74
        z = torch.rand(n, 1, generator=g) * 2 - 2
        yaw = (torch.rand(n, 1, generator=g) * 2 - 1) * np.pi
        boxes.append(torch.cat([xy, z, size, yaw], 1).float().to(dev))
        labels.append(lab.to(dev))
    return boxes, labels


# ---- baseline: the reference's loop and loss composition, restated ----
def _gaussian_2d(shape, sigma=1):
    m, n = [(ss - 1.) / 2. for ss in shape]
    y, x = np.ogrid[-m:m + 1, -n:n + 1]
    h = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    h[h < np.finfo(h.dtype).eps * h.max()] = 0
    return h


def _draw(heatmap, center, radius):
    diameter = 2 * radius + 1
    gaussian = _gaussian_2d((diameter, diameter), sigma=diameter / 6)
    x, y = int(center[0]), int(center[1])
    height, width = heatmap.shape[0:2]
    left, right = min(x, radius), min(width - x, radius + 1)
    top, bottom = min(y, radius), min(height - y, radius + 1)
    masked_heatmap = heatmap[y - top:y + bottom, x - left:x + right]
    masked_gaussian = torch.from_numpy(gaussian[radius - top:radius + bottom, radius - left:radius + right]).to(heatmap.device, torch.float32)
    if min(masked_gaussian.shape) > 0 and min(masked_heatmap.shape) > 0:
        torch.max(masked_heatmap, masked_gaussian, out=masked_heatmap)


def _radius(det_size, min_overlap):
    height, width = det_size
    b1 = height + width
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    r1 = (b1 + torch.sqrt(b1 ** 2 - 4 * c1)) / 2
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    r2 = (b2 + torch.sqrt(b2 ** 2 - 16 * c2)) / 2
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    r3 = (b3 + torch.sqrt(b3 ** 2 - 4 * (4 * min_overlap) * c3)) / 2
    return min(r1, r2, r3)


def baseline_targets_single(boxes, labels):
    dev = labels.device
    gb = torch.cat([boxes[:, :2], boxes[:, 2:3] + boxes[:, 5:6] * 0.5, boxes[:, 3:]], 1)
    vs, pc = torch.tensor(CFG['voxel_size']), torch.tensor(CFG['point_cloud_range'])
    W, H = 468, 468
    order = torch.cat([torch.where(labels == c)[0] for c in range(3)])
    tb, tc = gb[order], labels[order]
    heatmap = gb.new_zeros((3, H, W))
    anno_box = gb.new_zeros((500, 10))
    ind = labels.new_zeros((500,), dtype=torch.int64)
    mask = gb.new_zeros((500,), dtype=torch.uint8)
    for k in range(min(tb.shape[0], 500)):
        width, length = tb[k][3] / vs[0] / 1, tb[k][4] / vs[1] / 1
        if width > 0 and length > 0:
            radius = max(2, int(_radius((length, width), 0.1)))
            x, y, z = tb[k][0], tb[k][1], tb[k][2]
            center = torch.tensor([(x - pc[0]) / vs[0], (y - pc[1]) / vs[1]], dtype=torch.float32, device=dev)
            ci = center.to(torch.int32)
            if not (0 <= ci[0] < W and 0 <= ci[1] < H):
                continue
            _draw(heatmap[tc[k]], ci, radius)
            ind[k] = ci[1] * W + ci[0]
            mask[k] = 1
            rot = tb[k][6]
            anno_box[k] = torch.cat([center - torch.tensor([ci[0], ci[1]], device=dev), z.unsqueeze(0), tb[k][3:6].log(),
                                     torch.sin(rot).unsqueeze(0), torch.cos(rot).unsqueeze(0), rot.new_zeros(2)])
    return heatmap, anno_box, ind, mask


def baseline_targets(boxes, labels):
    out = [baseline_targets_single(b, l) for b, l in zip(boxes, labels)]
    return [torch.stack([o[i] for o in out]) for i in range(4)]


def baseline_loss(preds, hm, ab, ind, mask):
    p = torch.clamp(preds['heatmap'].sigmoid(), min=1e-4, max=1 - 1e-4)
    num_pos = hm.eq(1).float().sum().item()
    pos = -(p + 1e-12).log() * (1 - p).pow(2) * hm.eq(1)
    neg = -(1 - p + 1e-12).log() * p.pow(2) * (1 - hm).pow(4)
    loss_hm = (pos + neg).sum() / max(num_pos, 1)
    pred = torch.cat([preds[k] for k in ('reg', 'height', 'dim', 'rot', 'vel')], 1).permute(0, 2, 3, 1).contiguous()
    pred = pred.view(pred.size(0), -1, pred.size(3))
    pred = pred.gather(1, ind.unsqueeze(2).expand(ind.size(0), ind.size(1), 10))
    m = mask.unsqueeze(2).expand_as(ab).float() * (~torch.isnan(ab)).float()
    w = m * m.new_tensor(CFG['code_weights'])
    loss_bbox = 2 * ((pred - ab).abs() * w).sum() / (mask.float().sum() + 1e-4)
    return loss_hm + loss_bbox


def main(out_dir):
    assert torch.cuda.is_available(), "centerhead_bench needs a GPU"
    import sst_b200  # noqa: F401
    from sst_b200.centerhead_modules import CenterHead
    dev = torch.device("cuda:0")
    name, power = card()
    head = CenterHead(**HEAD)
    rows = []
    for B in (2, 4):
        boxes, labels = synth(B, dev, seed=B)
        g = torch.Generator(device=dev).manual_seed(1)
        shapes = dict(heatmap=3, reg=2, height=1, dim=3, rot=2, vel=2)
        preds = {k: (torch.randn(B, c, 468, 468, device=dev, generator=g) * (2 if k == 'heatmap' else 1)).requires_grad_(True)
                 for k, c in shapes.items()}

        def native_targets():
            head.get_targets(boxes, labels)

        def native_all():
            losses = head.loss(boxes, labels, [[preds]])
            sum(losses.values()).backward()

        def base_targets():
            baseline_targets(boxes, labels)

        def base_all():
            t = baseline_targets(boxes, labels)
            baseline_loss(preds, t[0], t[1], t[2], t[3]).backward()

        # the two sides compute the same targets (heatmaps within 1 ulp, ind / mask equal)
        nt, bt = head.get_targets(boxes, labels), baseline_targets(boxes, labels)
        same = torch.equal(nt[2][0], bt[2]) and torch.equal(nt[3][0], bt[3]) and \
            (nt[0][0].view(torch.int32) - bt[0].view(torch.int32)).abs().max().item() <= 1
        fns = dict(native_targets=native_targets, native_targets_loss_fwd_bwd=native_all, baseline_targets=base_targets,
                   baseline_targets_loss_fwd_bwd=base_all)
        rounds = {k: [] for k in fns}
        for _ in range(3):
            for k, f in fns.items():
                rounds[k].append(timed(f))
        med = {k: sorted(v)[1] for k, v in rounds.items()}
        n = B * 3 * 468 * 468
        from sst_b200 import ops
        x, t = preds['heatmap'].detach(), nt[0][0]
        fwd = timed(lambda: ops.gaussian_focal_loss(x, t))
        xg = x.clone().requires_grad_(True)
        bwd_only = timed(lambda: torch.autograd.grad(ops.gaussian_focal_loss(xg, t)[0], xg)) - fwd
        row = dict(B=B, boxes_per_sample=200, targets_agree=bool(same), median_ms=med,
                   speedup_targets=med['baseline_targets'] / med['native_targets'],
                   speedup_targets_loss=med['baseline_targets_loss_fwd_bwd'] / med['native_targets_loss_fwd_bwd'],
                   focal_forward_ms=fwd, focal_forward_bytes=8 * n, focal_forward_hbm_bound_ms=8 * n / HBM * 1e3,
                   focal_backward_ms=bwd_only, focal_backward_bytes=12 * n, focal_backward_hbm_bound_ms=12 * n / HBM * 1e3)
        rows.append(row)
        print(json.dumps(row))
    res = dict(card=name, power_limit=power, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power)))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "centerhead_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
