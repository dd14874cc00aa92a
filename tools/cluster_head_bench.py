"""SparseClusterHeadV2's training step on the Waymo D1 shape of FSD's first stage: 3 single-class tasks (Car / Pedestrian / Cyclist,
focal gamma 2 alpha 0.25, L1 box losses), B = 2 and 4 samples of 2,000 clusters and about 200 GTs each.  2,000 clusters per sample is an
assumption, not a measured count of FSD's clusters.

Native: ops.cluster_head_targets + ops.cluster_head_loss forward + backward for every task (through SparseClusterHeadV2.loss), and
get_bboxes with the training `rpn` cfg (no NMS, score_thr 0.1, max_num 500).  Baseline: the reference's per-task, per-sample composition
restated here on the same GPU (modify_gt_for_single_task's class masks, split_by_batch with its `.item()` assert, the reference's own
points_in_boxes_gpu from oracle/_ref/roiaware_pool3d_ext_ref*.so, PseudoSampler's two nonzeros, the encode, combine_by_batch, mmdet's
py_sigmoid_focal_loss and L1Loss on the nonzero positives), and get_bboxes as one ops.box3d_multiclass_nms per (task, sample).  Both are
checked to give the same targets and losses first.  CUDA events around 20 back-to-back calls per round, median of 3 alternating rounds;
the GPU time of each call's kernels and copies alone (torch.profiler); peak extra device memory; card name and power limit read in the
same run.  Writes OUT/cluster_head_bench.json.

    python tools/cluster_head_bench.py [OUT]
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from voteseg_bench import card, device_ms, timed  # noqa: E402

ROUNDS = 3
CLUSTERS = 2000
GAMMA, ALPHA = 2.0, 0.25
W = (2.0, 0.5, 0.5, 0.2)


def baseline_loss(R, cls_ids, cls_logits, reg_preds, xyz, bidx, boxes, labels):
    """loss_single_task per single-class task (global class cls_ids[t]) over get_targets per sample (sparse_cluster_head{,_v2}.py),
    restated"""
    B = len(boxes)
    out = {}
    for t, cls_id in enumerate(cls_ids):
        assert bidx.max().item() + 1 <= B
        lab_full = torch.full((xyz.shape[0],), 1, dtype=torch.long, device=xyz.device)
        tg_full = xyz.new_zeros((xyz.shape[0], 8))
        for b in range(B):
            m = labels[b] == cls_id
            gb, gl = boxes[b][m], labels[b].new_ones(int(m.sum())) * 0
            sm = bidx == b
            p = xyz[sm]
            lab = gl.new_full((p.shape[0],), 1)
            tg = p.new_zeros((p.shape[0], 8))
            if gl.numel() and p.shape[0]:
                idx = p.new_zeros((1, p.shape[0]), dtype=torch.int).fill_(-1)
                R.points_in_boxes_gpu(gb[:, :7].unsqueeze(0).contiguous(), p.unsqueeze(0).contiguous(), idx)
                inbox = idx[0].long()
                gi = torch.where(inbox > -1, inbox + 1, torch.zeros_like(inbox))
                pos = torch.nonzero(gi > 0).squeeze(-1).unique()
                torch.nonzero(gi == 0).squeeze(-1).unique()
                g = gb[gi[pos] - 1]
                lab[pos] = gl[gi[pos] - 1]
                if len(pos) > 0:
                    tg[pos] = torch.cat([g[:, :3] - p[pos], (g[:, 3:6] + 1e-6).log(), g[:, 6:7].sin(), g[:, 6:7].cos()], 1)
            lab_full[sm] = lab
            tg_full[sm] = tg
        x = cls_logits[t]
        oh = F.one_hot(lab_full, 2)[:, :1].type_as(x)
        pr = x.sigmoid()
        pt = (1 - pr) * oh + pr * (1 - oh)
        fw = (ALPHA * oh + (1 - ALPHA) * (1 - oh)) * pt.pow(GAMMA)
        out[f"loss_cls.task{t}"] = W[0] * (F.binary_cross_entropy_with_logits(x, oh, reduction='none') * fw).sum() / float(xyz.shape[0])
        pos_inds = ((lab_full >= 0) & (lab_full < 1)).nonzero(as_tuple=False).reshape(-1)
        num_pos = len(pos_inds)
        pr_, pt_ = reg_preds[t][pos_inds], tg_full[pos_inds]
        for q, (k, a, b_) in enumerate((("loss_center", 0, 3), ("loss_size", 3, 6), ("loss_rot", 6, 8))):
            out[f"{k}.task{t}"] = W[q + 1] * (pr_[:, a:b_] - pt_[:, a:b_]).abs().sum() / float(num_pos) if num_pos else pr_.sum() * 0
    return out, lab_full, tg_full


def main(out_dir):
    from oracle import build_ref, cluster_head_oracle as CO
    from sst_b200 import ops
    from sst_b200.registry import MODELS
    R = build_ref.load_module("roiaware_pool3d_ext_ref")
    if R is None:
        raise SystemExit("oracle/_ref/roiaware_pool3d_ext_ref*.so not built (python -m oracle.build_ref_roiaware)")
    dev = torch.device("cuda:0")
    name, power = card()
    head = MODELS.build(dict(CO.FSD_D1_HEAD, in_channel=8, shared_mlp_dims=[8], train_cfg=CO.FSD_D1_TRAIN_CFG)).to(dev).train()
    rec = {"card": name, "power_limit": power, "shape": f"Waymo D1 head: 3 single-class tasks, {CLUSTERS} clusters and ~200 GTs per sample",
           "rounds": ROUNDS, "calls_per_round": 20, "batches": []}
    for B in (2, 4):
        g = torch.Generator().manual_seed(B)
        gts = [190 + int(torch.randint(0, 21, (1,), generator=g)) for _ in range(B)]
        xyz, inds, Bx, Lb = CO.synth_clusters(B, [CLUSTERS] * B, gts, CO.WAYMO_NAMES, spread=70.0, inside=0.5)
        xyz, inds, Bx, Lb = xyz.to(dev), inds.to(dev), [b.to(dev) for b in Bx], [lab.to(dev) for lab in Lb]
        M = xyz.shape[0]
        x = [(torch.randn((M, 1), generator=g) * 2 - 2).to(dev) for _ in range(3)]
        r = [torch.randn((M, 8), generator=g).to(dev) for _ in range(3)]
        metas = [dict()] * B

        def native_all():
            xg, rg = [a.clone().requires_grad_(True) for a in x], [a.clone().requires_grad_(True) for a in r]
            losses = head.loss(xg, rg, xyz, inds, Bx, Lb)
            sum(losses.values()).backward()
            return losses

        def base_all():
            xg, rg = [a.clone().requires_grad_(True) for a in x], [a.clone().requires_grad_(True) for a in r]
            losses, _, _ = baseline_loss(R, [0, 1, 2], xg, rg, xyz, inds[:, 1], Bx, Lb)
            sum(losses.values()).backward()
            return losses

        def native_boxes():
            return head.get_bboxes(x, r, xyz, inds, metas)

        cfg = CO.Cfg(CO.RPN_CFG)

        def base_boxes():
            out = []
            for b in range(B):
                sm = inds[:, 1] == b
                res = []
                for t in range(3):
                    s = torch.cat([x[t][sm].sigmoid(), x[t].new_zeros(int(sm.sum()), 1)], 1)
                    bb = CO.decode(r[t][sm], xyz[sm])
                    res.append(ops.box3d_multiclass_nms(bb, CO.xywhr2xyxyr(bb[:, [0, 1, 3, 4, 6]]), s, cfg.score_thr, cfg.max_num, cfg))
                out.append(res)
            return out

        # same targets and losses first
        lab, tg, npos = ops.cluster_head_targets(xyz, inds, Bx, Lb, CO.WAYMO_TASKS, CO.WAYMO_NAMES)
        same = True
        for t in range(3):
            _, bl, bt = baseline_loss(R, [t], [x[t]], [r[t]], xyz, inds[:, 1], Bx, Lb)
            same &= bool(torch.equal(bl, lab[t])) and (tg[t] - bt).abs().max().item() <= 1e-6
        ln, lb = native_all(), base_all()
        loss_rel = max(abs(ln[k].item() - lb[k].item()) / max(abs(lb[k].item()), 1e-30) for k in ln)
        nb, bb = native_boxes(), base_boxes()
        same_boxes = all(torch.equal(nb[b][0], torch.cat([res[0] for res in bb[b]])) for b in range(B))
        fns = (("native_loss", native_all), ("baseline_loss", base_all), ("native_get_bboxes", native_boxes),
               ("baseline_get_bboxes", base_boxes))
        times, mem = {k: [] for k, _ in fns}, {}
        for _ in range(ROUNDS):
            for k, fn in fns:
                ms, mb, _ = timed(fn)
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0.0), mb)
        med = {k: float(np.median(v)) for k, v in times.items()}
        row = {"B": B, "clusters": M, "gts": gts, "positives": [int(v) for v in npos.tolist()], "same_targets": same,
               "loss_max_rel_diff": loss_rel, "same_boxes": same_boxes, "median_ms": med, "peak_mib": mem,
               "device_ms": {k: device_ms(fn) for k, fn in fns}}
        print(json.dumps(row))
        rec["batches"].append(row)
    print(f"card: {name}, power limit {power}")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "cluster_head_bench.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "bench_out")
