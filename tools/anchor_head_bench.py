"""Anchor3DHead's training path on the Waymo D5 geometry of the anchor-based SST configs (468 x 468 cells, 3 sizes x 2 rotations =
1,314,144 anchors per sample, 3 classes), B = 2 and 4 samples of about 200 GT boxes each with a Waymo-like class mix (car 70 %,
pedestrian 25 %, cyclist 5 %):
  native    ops.anchor3d_targets alone, then the targets + the focal, L1 and direction losses forward + backward (to the head outputs);
  baseline  the reference's composition restated here on the same GPU: per sample and size a dense [G, 438048] bbox_overlaps of the
            nearest BEV boxes, MaxIoUAssigner's Python low-quality loop over the GTs, PseudoSampler's nonzero, the encode; then
            loss_single's permuted copies, labels.max().item(), the nonzero gather of the positives and autograd.
Both are checked to give the same labels and losses first.  Peak device memory of each is reported (torch's allocator, reset per
call).  CUDA events around each call (ended by a synchronise), median of 3 alternating rounds; the card name and power limit are read
in the same run.  Writes OUT/anchor_head_bench.json.

    python tools/anchor_head_bench.py [OUT]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROUNDS = 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:
        return [torch.cuda.get_device_name(0), f"unknown ({e})"]


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), (torch.cuda.max_memory_allocated() - base) / 2**20, out


def synth(B, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    sizes = torch.tensor([[2.08, 4.73, 1.77], [0.84, 0.91, 1.74], [0.84, 1.81, 1.77]])    # car, pedestrian, cyclist
    boxes, labels = [], []
    for _ in range(B):
        n = 190 + int(torch.randint(0, 21, (1,), generator=g))
        kind = torch.multinomial(torch.tensor([0.70, 0.25, 0.05]), n, replacement=True, generator=g)
        lab = torch.tensor([0, 2, 1])[kind]                                              # config label order: car, cyclist, pedestrian
        ctr = (torch.rand((n, 2), generator=g) * 2 - 1) * 70
        dims = sizes[kind] * (0.85 + 0.3 * torch.rand((n, 3), generator=g))
        z = -0.05 + 0.2 * torch.randn((n, 1), generator=g)
        yaw = (torch.rand((n, 1), generator=g) * 2 - 1) * np.pi
        boxes.append(torch.cat([ctr, z, dims, yaw], 1).to(dev))
        labels.append(lab.to(dev))
    return boxes, labels


# ---- the reference's composition, restated on the GPU ----
def _limit_period(v, offset=0.5, period=np.pi):
    return v - torch.floor(v / period + offset) * period


def _nearest_bev(b):
    bev = b[:, [0, 1, 3, 4, 6]]
    cond = (torch.abs(_limit_period(bev[:, -1], 0.5, np.pi)) > np.pi / 4)[..., None]
    xywh = torch.where(cond, bev[:, [0, 1, 3, 2]], bev[:, :4])
    return torch.cat([xywh[:, :2] - xywh[:, 2:] / 2, xywh[:, :2] + xywh[:, 2:] / 2], -1)


def _overlaps(b1, b2):
    area1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    area2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt = torch.max(b1[:, None, :2], b2[None, :, :2])
    rb = torch.min(b1[:, None, 2:], b2[None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = torch.max(area1[:, None] + area2[None, :] - overlap, b1.new_tensor([1e-6]))
    return overlap / union


def _encode(a, g):
    xa, ya, za, wa, la, ha, ra = torch.split(a, 1, -1)
    xg, yg, zg, wg, lg, hg, rg = torch.split(g, 1, -1)
    za, zg = za + ha / 2, zg + hg / 2
    d = torch.sqrt(la**2 + wa**2)
    return torch.cat([(xg - xa) / d, (yg - ya) / d, (zg - za) / ha, torch.log(wg / wa), torch.log(lg / la), torch.log(hg / ha), rg - ra], -1)


def baseline_targets(anchors, boxes, labels, asg, C, dir_offset=0.7854):
    H, W, S, R, _ = anchors.shape
    outs = [[] for _ in range(6)]
    ntp = 0
    for gt, lab in zip(boxes, labels):
        per = [[] for _ in range(6)]
        npos = 0
        for s, (pos_thr, neg_thr, min_pos) in enumerate(asg):
            anc = anchors[:, :, s].reshape(-1, 7)
            n = anc.shape[0]
            ov = _overlaps(_nearest_bev(gt), _nearest_bev(anc))
            gi = ov.new_full((n,), -1, dtype=torch.long)
            mx, am = ov.max(0)
            gmx, gam = ov.max(1)
            gi[(mx >= 0) & (mx < neg_thr)] = 0
            p = mx >= pos_thr
            gi[p] = am[p] + 1
            for i in range(gt.shape[0]):
                if gmx[i] >= min_pos:
                    gi[ov[i, :] == gmx[i]] = i + 1
            pos, neg = torch.nonzero(gi > 0).squeeze(-1).unique(), torch.nonzero(gi == 0).squeeze(-1).unique()
            labels_t = torch.full((n,), C, dtype=torch.long, device=anc.device)
            lw, bt, bw = anc.new_zeros(n), torch.zeros_like(anc), torch.zeros_like(anc)
            dt, dw = torch.zeros(n, dtype=torch.long, device=anc.device), anc.new_zeros(n)
            if len(pos):
                t = _encode(anc[pos], gt[gi[pos] - 1])
                bt[pos], bw[pos] = t, 1.0
                rot = _limit_period(t[:, 6] + anc[pos, 6] - dir_offset, 0, 2 * np.pi)
                dt[pos], dw[pos] = torch.clamp(torch.floor(rot / np.pi).long(), 0, 1), 1.0
                labels_t[pos], lw[pos] = lab[gi[pos] - 1], 1.0
            lw[neg] = 1.0
            npos += len(pos)
            for k, v in enumerate((labels_t, lw, bt, bw, dt, dw)):
                per[k].append(v.reshape(H * W, 1, R, *v.shape[1:]))
        ntp += max(npos, 1)
        for k in range(6):
            outs[k].append(torch.cat(per[k], 1).reshape(H * W * S * R, *per[k][0].shape[3:]))
    return tuple(torch.stack(o) for o in outs) + (ntp,)


def baseline_losses(cls, reg, dr, t, C):
    labels, lw, bt, bw, dt, dw, ntp = t
    labels = labels.reshape(-1)
    x = cls.permute(0, 2, 3, 1).reshape(-1, C)
    assert labels.max().item() <= C
    tt = torch.nn.functional.one_hot(labels, C + 1)[:, :C].type_as(x)
    p = x.sigmoid()
    pt = (1 - p) * tt + p * (1 - tt)
    fw = (0.25 * tt + 0.75 * (1 - tt)) * pt.pow(2)
    lc = (torch.nn.functional.binary_cross_entropy_with_logits(x, tt, reduction='none') * fw * lw.reshape(-1, 1)).sum() / ntp
    pos = ((labels >= 0) & (labels < C)).nonzero(as_tuple=False).reshape(-1)
    pb = reg.permute(0, 2, 3, 1).reshape(-1, 7)[pos]
    tb = bt.reshape(-1, 7)[pos]
    wb = bw.reshape(-1, 7)[pos]
    pb = torch.cat([pb[:, :6], torch.sin(pb[:, 6:7]) * torch.cos(tb[:, 6:7])], 1)
    tb = torch.cat([tb[:, :6], torch.cos(reg.permute(0, 2, 3, 1).reshape(-1, 7)[pos][:, 6:7]) * torch.sin(tb[:, 6:7])], 1)
    lb = 0.5 * ((pb - tb).abs() * wb).sum() / ntp
    pd = dr.permute(0, 2, 3, 1).reshape(-1, 2)[pos]
    ld = 0.2 * (torch.nn.functional.cross_entropy(pd, dt.reshape(-1)[pos], reduction='none') * dw.reshape(-1)[pos]).sum() / ntp
    return lc, lb, ld


def main(out_dir):
    from sst_b200 import flagship as fl, ops
    from sst_b200.anchor3d_modules import AlignedAnchor3DRangeGenerator
    dev = torch.device("cuda:0")
    name, power = card()
    gen_cfg = dict(fl.ANCHOR_HEAD["anchor_generator"])
    gen_cfg.pop("type")
    gen = AlignedAnchor3DRangeGenerator(**gen_cfg)
    H = W = 468
    C, S, R = 3, 3, 2
    axes = gen.axes((H, W), dev)
    anchors = gen.grid_anchors([(H, W)], dev)[0][0]
    asg = [(a["pos_iou_thr"], a["neg_iou_thr"], a["min_pos_iou"]) for a in fl.ANCHOR_TRAIN_CFG["assigner"]]
    rec = {"card": name, "power_limit": power, "geometry": "Waymo D5: 468 x 468, 3 sizes x 2 rotations, 3 classes", "rounds": ROUNDS,
           "batches": []}
    for B in (2, 4):
        boxes, labels = synth(B, dev, seed=B)
        g = torch.Generator().manual_seed(B)
        preds = [torch.randn((B, S * R * k, H, W), generator=g).mul_(0.5).to(dev) for k in (C, 7, 2)]
        preds[0] -= 3.0

        def native_targets():
            return ops.anchor3d_targets(*axes, torch.cat(boxes), torch.cat(labels), [b.shape[0] for b in boxes], C, [a[0] for a in asg],
                                        [a[1] for a in asg], [a[2] for a in asg], True, False, 0.7854)

        def native_all():
            t = native_targets()
            ps = [p.clone().requires_grad_(True) for p in preds]
            lc = ops.anchor_focal_loss(ps[0], t[0], t[1], t[6], C, 1.0)
            lb, ld = ops.anchor_reg_dir_loss(ps[1], ps[2], t[0], t[2], t[3], t[4], t[5], t[6], C, [1.0] * 7, 0.5, 0.2)
            (lc + lb + ld).backward()
            return t, (lc, lb, ld)

        def base_targets():
            return baseline_targets(anchors, boxes, labels, asg, C)

        def base_all():
            t = base_targets()
            ps = [p.clone().requires_grad_(True) for p in preds]
            ls = baseline_losses(*ps, t, C)
            sum(ls).backward()
            return t, ls

        # same answer first
        (tn, ln), (tb, lb_) = native_all(), base_all()
        same_labels = bool(torch.equal(tn[0], tb[0])) and int(tn[6]) == tb[6]
        loss_rel = max(abs(a.item() - b.item()) / max(abs(b.item()), 1e-30) for a, b in zip(ln, lb_))
        times = {k: [] for k in ("native_targets", "native_all", "baseline_targets", "baseline_all")}
        mem = {}
        for _ in range(ROUNDS):
            for k, fn in (("native_targets", native_targets), ("baseline_targets", base_targets), ("native_all", native_all),
                          ("baseline_all", base_all)):
                ms, mb, _ = timed(fn)
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0.0), mb)
        med = {k: float(np.median(v)) for k, v in times.items()}
        row = {"B": B, "gts": [int(b.shape[0]) for b in boxes], "positives": int((tn[0] < C).sum()), "same_labels": same_labels,
               "loss_max_rel_diff": loss_rel, "median_ms": med, "peak_mib": mem,
               "speedup_targets": med["baseline_targets"] / med["native_targets"], "speedup_all": med["baseline_all"] / med["native_all"]}
        print(json.dumps(row))
        rec["batches"].append(row)
    print(f"card: {name}, power limit {power}")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "anchor_head_bench.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "bench_out"))
