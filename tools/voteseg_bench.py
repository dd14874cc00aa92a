"""VoteSegHead's training path on the Waymo D1 shape of FSD's segmentor (3 classes, sigmoid focal loss gamma 3 alpha 0.8, vote L1 loss,
the recall logs of score_thresh (0.3, 0.25, 0.25)), B = 2 and 4 samples of 150k points and about 200 GT boxes each in a car / pedestrian /
cyclist mix (60 / 25 / 15 %):
  native    ops.voteseg_targets alone, then the targets + ops.voteseg_loss forward + backward (to the head outputs);
  baseline  the reference's composition restated on the same GPU: get_targets' per-sample loop (valid_gt_mask filter, the reference's own
            points_in_boxes_gpu from oracle/_ref/roiaware_pool3d_ext_ref*.so, the gathers and boolean masks), then `losses` with its
            .item() asserts, the boolean-mask vote gathers, mmdet's torch py_sigmoid_focal_loss (mmcv's kernel is not available) and the
            recall logs, then autograd.
Both are checked to give the same labels and losses first.  The native path is fast enough that a call's Python, ctypes and autograd
work outlasts its kernels, so device_ms also reports the GPU time of each call's kernels and copies alone (torch.profiler).  Peak extra device memory of each is reported (torch's allocator, reset per
round).  Each round times REPS back-to-back calls between two CUDA events (ended by a synchronise) and reports the time per call, so a
single sub-millisecond call's launch jitter does not decide the number; median of 3 alternating rounds.  The card name and power limit
are read in the same run.  Writes OUT/voteseg_bench.json.

    python tools/voteseg_bench.py [OUT]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROUNDS = 3
REPS = 20
C = 3
GAMMA, ALPHA = 3.0, 0.8
THRESH, NAMES = (0.3, 0.25, 0.25), ("Car", "Ped", "Cyc")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:
        return [torch.cuda.get_device_name(0), f"unknown ({e})"]


def timed(fn):
    """(ms per call over REPS calls, peak extra MiB, the last call's result)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(REPS):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / REPS, (torch.cuda.max_memory_allocated() - base) / 2**20, out


def device_ms(fn):
    """the GPU time per call of fn's kernels and copies alone (torch.profiler over REPS calls), without the host-side gaps between them"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            fn()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1e3 / REPS


def baseline_targets(R, points_list, boxes_list, labels_list):
    """get_targets (segmentation_head.py:212-283) with the reference's own points_in_boxes_gpu"""
    labs, vts, masks = [], [], []
    for points, bboxes, bbox_labels in zip(points_list, boxes_list, labels_list):
        points = points[:, :3]
        valid_gt_mask = bbox_labels >= 0
        bboxes, bbox_labels = bboxes[valid_gt_mask], bbox_labels[valid_gt_mask]
        if len(bbox_labels) == 0:
            labs.append(torch.ones(len(points), device=points.device, dtype=torch.long) * C)
            vts.append(torch.zeros_like(points))
            masks.append(torch.zeros(len(points), device=points.device, dtype=torch.bool))
            continue
        idx = points.new_zeros((1, points.shape[0]), dtype=torch.int).fill_(-1)
        R.points_in_boxes_gpu(bboxes[:, :7].unsqueeze(0).contiguous(), points.unsqueeze(0).contiguous(), idx)
        inbox = idx.squeeze(0).long()
        bg = inbox < 0
        lab = bbox_labels[inbox]
        lab[bg] = C
        gc = torch.cat([bboxes[:, :2], bboxes[:, 2:3] + bboxes[:, 5:6] * 0.5], 1)
        delta = gc[inbox] - points
        delta[bg] = 0
        labs.append(lab)
        vts.append(torch.sign(delta) * (delta.abs() ** 0.5))
        masks.append(~bg)
    return torch.cat(labs), torch.cat(vts), torch.cat(masks)


def baseline_losses(seg_logit, vote_preds, seg_label, vote_targets, vote_mask):
    """losses (segmentation_head.py:107-173) with mmdet's py_sigmoid_focal_loss and L1Loss"""
    num_classes = seg_logit.size(1)
    t = F.one_hot(seg_label, num_classes=num_classes + 1)[:, :num_classes].type_as(seg_logit)
    p = seg_logit.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    fw = (ALPHA * t + (1 - ALPHA) * (1 - t)) * pt.pow(GAMMA)
    loss = {"loss_sem_seg": (F.binary_cross_entropy_with_logits(seg_logit, t, reduction='none') * fw).mean()}
    vote_preds = vote_preds.reshape(-1, num_classes, 3)
    assert seg_label.max().item() == num_classes
    valid_vote_preds = vote_preds[vote_mask].reshape(-1, 3)
    num_valid = vote_mask.sum()
    valid_label = seg_label[vote_mask]
    if num_valid > 0:
        assert valid_label.max().item() < num_classes
        assert valid_label.min().item() >= 0
        indices = torch.arange(num_valid, device=valid_label.device) * num_classes + valid_label
        loss["loss_vote"] = (valid_vote_preds[indices, :] - vote_targets[vote_mask]).abs().mean()
    else:
        loss["loss_vote"] = vote_preds.sum() * 0
    scores = seg_logit.sigmoid()
    for i, thr in enumerate(THRESH):
        pred_true, real_true = scores[:, i] > thr, seg_label == i
        loss[f"recall_{NAMES[i]}"] = (pred_true & real_true).sum().float() / (real_true.sum().float() + 1e-5)
    return loss


def main(out_dir):
    from oracle import build_ref, voteseg_oracle as VO
    from sst_b200 import ops
    R = build_ref.load_module("roiaware_pool3d_ext_ref")
    if R is None:
        raise SystemExit("oracle/_ref/roiaware_pool3d_ext_ref*.so not built (python -m oracle.build_ref_roiaware)")
    dev = torch.device("cuda:0")
    name, power = card()
    cfg = ops.VoteSegLossConfig(C, True, gamma=GAMMA, alpha=ALPHA, score_thresh=THRESH, class_names=NAMES)
    rec = {"card": name, "power_limit": power, "shape": "Waymo D1: 3 classes, focal gamma 3 alpha 0.8, 150k points and ~200 GTs per sample",
           "rounds": ROUNDS, "calls_per_round": REPS, "batches": []}
    for B in (2, 4):
        g = torch.Generator().manual_seed(B)
        P, Bx, Lb = [], [], []
        for _ in range(B):
            n_gt = 190 + int(torch.randint(0, 21, (1,), generator=g))
            boxes, lab = VO.synth_boxes(g, n_gt, 3, spread=70.0, invalid=0.0)
            P.append(VO.points_around(g, boxes, 150000, spread=70.0, inside=0.3).to(dev))
            Bx.append(boxes.to(dev))
            Lb.append(lab.to(dev))
        N = sum(p.shape[0] for p in P)
        x = (torch.randn((N, C), generator=g) * 2 - 2).to(dev)
        v = torch.randn((N, 3 * C), generator=g).to(dev)

        def native_targets():
            return ops.voteseg_targets(P, None, Bx, Lb, C)

        def native_all():
            t = native_targets()
            xg, vg = x.clone().requires_grad_(True), v.clone().requires_grad_(True)
            seg, vote, met = ops.voteseg_loss(xg, vg, *t, cfg)
            (seg + vote).backward()
            return t, (seg, vote)

        def base_targets():
            return baseline_targets(R, P, Bx, Lb)

        def base_all():
            t = base_targets()
            xg, vg = x.clone().requires_grad_(True), v.clone().requires_grad_(True)
            loss = baseline_losses(xg, vg, *t)
            (loss["loss_sem_seg"] + loss["loss_vote"]).backward()
            return t, (loss["loss_sem_seg"], loss["loss_vote"])

        (tn, ln), (tb, lb) = native_all(), base_all()
        same = all(bool(torch.equal(a, b)) for a, b in zip(tn, tb))
        loss_rel = max(abs(a.item() - b.item()) / max(abs(b.item()), 1e-30) for a, b in zip(ln, lb))
        times = {k: [] for k in ("native_targets", "native_all", "baseline_targets", "baseline_all")}
        mem = {}
        for _ in range(ROUNDS):
            for k, fn in (("native_targets", native_targets), ("baseline_targets", base_targets), ("native_all", native_all),
                          ("baseline_all", base_all)):
                ms, mb, _ = timed(fn)
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0.0), mb)
        med = {k: float(np.median(v)) for k, v in times.items()}
        row = {"B": B, "points": N, "gts": [int(b.shape[0]) for b in Bx], "in_box": int(tn[2].sum()), "same_targets": same,
               "loss_max_rel_diff": loss_rel, "median_ms": med, "peak_mib": mem,
               "speedup_targets": med["baseline_targets"] / med["native_targets"], "speedup_all": med["baseline_all"] / med["native_all"],
               "device_ms": {"native_all": device_ms(native_all), "baseline_all": device_ms(base_all)}}
        print(json.dumps(row))
        rec["batches"].append(row)
    print(f"card: {name}, power limit {power}")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "voteseg_bench.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "bench_out"))
