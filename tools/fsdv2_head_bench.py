"""FSDV2Head's training step on the nuScenes shape of configs/fsdv2/fsdv2_nusc_1x.py: two 5-class tasks, code size 10 (focal gamma 2
alpha 0.25, L1 box and velocity losses), centroid assignment, B = 2 and 4 samples of 3,000 virtual voxels and about 40 GTs (9 columns,
with velocity) each.  3,000 virtual voxels per sample is an assumption, not a measured count of FSDv2's virtual voxels.

Native: ops.cluster_head_targets + ops.cluster_head_loss forward + backward for every task (through FSDV2Head.loss with aux_xyz), and
get_bboxes with the nuScenes test cfg (rotated NMS 0.25, score_thr 0.05, max_num 500, all_task_max_num 500).  Baseline: the reference's
per-task, per-sample composition restated here on the same GPU (modify_gt_for_single_task's class masks, split_by_batch with its
`.item()` assert, the reference's own points_in_boxes_gpu from oracle/_ref/roiaware_pool3d_ext_ref*.so on the centroids, PseudoSampler's
two nonzeros, the encode with velocity, combine_by_batch, mmdet's py_sigmoid_focal_loss, L1Loss on the nonzero positives and loss_vel's
mean), and get_bboxes as one ops.box3d_multiclass_nms per (task, sample), the tasks concatenated and cut by topk per sample.  Both are
checked to give the same targets, losses and boxes first.  CUDA events around 20 back-to-back calls per round, median of 3 alternating
rounds; the GPU time of each call's kernels and copies alone (torch.profiler); peak extra device memory; card name and power limit read
in the same run.  Writes OUT/fsdv2_head_bench.json.

    python tools/fsdv2_head_bench.py [OUT]
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
VOXELS = 3000
GAMMA, ALPHA = 2.0, 0.25
W = (4.0, 0.5, 0.5, 0.2, 0.2)


def baseline_loss(R, tasks, names, cls_logits, reg_preds, xyz, aux, bidx, boxes, labels):
    """loss_single_task per task over get_targets per sample (fsd_v2_head.py), restated"""
    B = len(boxes)
    out, labs, tgs = {}, [], []
    for t, task in enumerate(tasks):
        C = len(task)
        gbs, gls = [], []
        for b in range(B):                       # modify_gt_for_single_task
            sel, lab = [], []
            for i, n in enumerate(task):
                m = labels[b] == names.index(n)
                sel.append(boxes[b][m])
                lab.append(labels[b].new_ones(int(m.sum())) * i)
            gbs.append(torch.cat(sel)), gls.append(torch.cat(lab))
            assert gls[-1].max().item() < C if gls[-1].numel() else True
        assert bidx.max().item() + 1 <= B
        lab_full = torch.full((xyz.shape[0],), C, dtype=torch.long, device=xyz.device)
        tg_full = xyz.new_zeros((xyz.shape[0], 10))
        w_full = xyz.new_zeros((xyz.shape[0], 10))
        for b in range(B):
            gb, gl = gbs[b], gls[b]
            sm = bidx == b
            p, a = xyz[sm], aux[sm]
            lab = gl.new_full((p.shape[0],), C)
            tg = p.new_zeros((p.shape[0], 10))
            w = p.new_zeros((p.shape[0], 10))
            if gl.numel() and p.shape[0]:
                idx = p.new_zeros((1, p.shape[0]), dtype=torch.int).fill_(-1)
                R.points_in_boxes_gpu(gb[:, :7].unsqueeze(0).contiguous(), a.unsqueeze(0).contiguous(), idx)
                inbox = idx[0].long()
                gi = torch.where(inbox > -1, inbox + 1, torch.zeros_like(inbox))
                pos = torch.nonzero(gi > 0).squeeze(-1).unique()
                torch.nonzero(gi == 0).squeeze(-1).unique()
                g = gb[gi[pos] - 1]
                lab[pos] = gl[gi[pos] - 1]
                w[pos] = 1.0
                if len(pos) > 0:
                    tg[pos] = torch.cat([g[:, :3] - p[pos], (g[:, 3:6] + 1e-6).log(), g[:, 6:7].sin(), g[:, 6:7].cos(), g[:, 7:9]], 1)
            lab_full[sm] = lab
            tg_full[sm] = tg
            w_full[sm] = w
        x = cls_logits[t]
        oh = F.one_hot(lab_full, C + 1)[:, :C].type_as(x)
        pr = x.sigmoid()
        pt = (1 - pr) * oh + pr * (1 - oh)
        fw = (ALPHA * oh + (1 - ALPHA) * (1 - oh)) * pt.pow(GAMMA)
        out[f"loss_cls.task{t}"] = W[0] * (F.binary_cross_entropy_with_logits(x, oh, reduction='none') * fw).sum() / float(xyz.shape[0])
        pos_inds = ((lab_full >= 0) & (lab_full < C)).nonzero(as_tuple=False).reshape(-1)
        num_pos = len(pos_inds)
        pr_, pt_, pw_ = reg_preds[t][pos_inds], tg_full[pos_inds], w_full[pos_inds]
        for q, (k, a, b_) in enumerate((("loss_center", 0, 3), ("loss_size", 3, 6), ("loss_rot", 6, 8))):
            out[f"{k}.task{t}"] = W[q + 1] * (pr_[:, a:b_] - pt_[:, a:b_]).abs().sum() / float(num_pos) if num_pos else pr_.sum() * 0
        out[f"loss_vel.task{t}"] = W[4] * ((pr_[:, 8:] - pt_[:, 8:]).abs() * pw_[:, 8:]).mean() if num_pos else pr_.sum() * 0
        labs.append(lab_full), tgs.append(tg_full)
    return out, labs, tgs


def main(out_dir):
    from oracle import build_ref, cluster_head_oracle as CO, fsdv2_head_oracle as FO
    from sst_b200 import ops
    from sst_b200.registry import MODELS
    R = build_ref.load_module("roiaware_pool3d_ext_ref")
    if R is None:
        raise SystemExit("oracle/_ref/roiaware_pool3d_ext_ref*.so not built (python -m oracle.build_ref_roiaware)")
    dev = torch.device("cuda:0")
    name, power = card()
    tasks, names = FO.NUSC_TASKS, FO.NUSC_NAMES
    head = MODELS.build(dict(FO.NUSC_HEAD, in_channel=8, shared_mlp_dims=[8], train_cfg=FO.NUSC_TRAIN_CFG,
                             test_cfg=FO.NUSC_TEST_CFG)).to(dev).eval()
    cfg = CO.Cfg(FO.NUSC_TEST_CFG)
    rec = {"card": name, "power_limit": power,
           "shape": f"nuScenes head: two 5-class tasks, code size 10, {VOXELS} virtual voxels (assumed) and ~40 GTs per sample",
           "rounds": ROUNDS, "calls_per_round": 20, "batches": []}
    for B in (2, 4):
        g = torch.Generator().manual_seed(B)
        gts = [35 + int(torch.randint(0, 11, (1,), generator=g)) for _ in range(B)]
        xyz, aux, inds, Bx, Lb = FO.synth_clusters(B, [VOXELS] * B, gts, names, width=9, spread=50.0, inside=0.5)
        xyz, aux, inds, Bx, Lb = xyz.to(dev), aux.to(dev), inds.to(dev), [b.to(dev) for b in Bx], [lab.to(dev) for lab in Lb]
        M = xyz.shape[0]
        x = [(torch.randn((M, 5), generator=g) * 2 - 2).to(dev) for _ in range(2)]
        r = [torch.randn((M, 10), generator=g).to(dev) for _ in range(2)]
        metas = [dict()] * B

        def native_all():
            xg, rg = [a.clone().requires_grad_(True) for a in x], [a.clone().requires_grad_(True) for a in r]
            losses = head.loss(xg, rg, xyz, inds, Bx, Lb, aux_xyz=aux)
            sum(losses.values()).backward()
            return losses

        def base_all():
            xg, rg = [a.clone().requires_grad_(True) for a in x], [a.clone().requires_grad_(True) for a in r]
            losses, _, _ = baseline_loss(R, tasks, names, xg, rg, xyz, aux, inds[:, 1], Bx, Lb)
            sum(losses.values()).backward()
            return losses

        def native_boxes():
            return head.get_bboxes(x, r, xyz, inds, metas)

        def base_boxes():
            out = []
            for b in range(B):
                sm = inds[:, 1] == b
                bb, ss, ll = [], [], []
                for t in range(2):
                    s = torch.cat([x[t][sm].sigmoid(), x[t].new_zeros(int(sm.sum()), 1)], 1)
                    bx = FO.decode(r[t][sm], xyz[sm])
                    ob, os_, ol = ops.box3d_multiclass_nms(bx, CO.xywhr2xyxyr(bx[:, [0, 1, 3, 4, 6]]), s, cfg.score_thr, cfg.max_num, cfg)
                    glob = torch.zeros_like(ol) - 1
                    for i, n in enumerate(tasks[t]):
                        glob[ol == i] = names.index(n)
                    bb.append(ob), ss.append(os_), ll.append(glob)
                ob, os_, ol = torch.cat(bb), torch.cat(ss), torch.cat(ll)
                if len(os_) > cfg.all_task_max_num:
                    k = os_.topk(cfg.all_task_max_num)[1]
                    ob, os_, ol = ob[k], os_[k], ol[k]
                out.append((ob, os_, ol))
            return out

        # same targets, losses and boxes first
        lab, tg, npos = ops.cluster_head_targets(xyz, inds, Bx, Lb, tasks, names, assign_xyz=aux, code_size=10)
        _, bl, bt = baseline_loss(R, tasks, names, x, r, xyz, aux, inds[:, 1], Bx, Lb)
        same = all(bool(torch.equal(bl[t], lab[t])) and (tg[t][:, :10] - bt[t]).abs().max().item() <= 1e-6 for t in range(2))
        ln, lb = native_all(), base_all()
        loss_rel = max(abs(ln[k].item() - lb[k].item()) / max(abs(lb[k].item()), 1e-30) for k in ln)
        nb, bb = native_boxes(), base_boxes()
        same_boxes = all(torch.equal(nb[b][0], bb[b][0]) and torch.equal(nb[b][2], bb[b][2]) for b in range(B))
        fns = (("native_loss", native_all), ("baseline_loss", base_all), ("native_get_bboxes", native_boxes),
               ("baseline_get_bboxes", base_boxes))
        times, mem = {k: [] for k, _ in fns}, {}
        for _ in range(ROUNDS):
            for k, fn in fns:
                ms, mb, _ = timed(fn)
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0.0), mb)
        med = {k: float(np.median(v)) for k, v in times.items()}
        row = {"B": B, "voxels": M, "gts": gts, "positives": [int(v) for v in npos.tolist()], "same_targets": same,
               "loss_max_rel_diff": loss_rel, "same_boxes": same_boxes, "boxes": [int(o[1].shape[0]) for o in nb], "median_ms": med,
               "peak_mib": mem, "device_ms": {k: device_ms(fn) for k, fn in fns}}
        print(json.dumps(row))
        rec["batches"].append(row)
    print(f"card: {name}, power limit {power}")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "fsdv2_head_bench.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "bench_out")
