"""TEST INFRASTRUCTURE - writes tests/golden/iou3d_bev.npz from the reference's OWN iou3d CUDA kernels (oracle/_ref/iou3d_ref*.so, built
by oracle/build_ref_iou3d.py), so that the CPU oracle (oracle/iou3d_oracle.py) is pinned to the reference where no GPU exists.  Needs a
CUDA device.  `python -m oracle.make_golden_iou3d [OUT_DIR]` (default tests/golden).

Contents: boxes_a [256, 5] / boxes_b [192, 5] (special cases, a dense cluster and spread boxes within +-75 m) with the reference's
overlap and IoU matrices; nms_boxes [3000, 5] + nms_scores (distinct) with no box pair whose fp64 IoU (rotated or axis-aligned) lies
within 1e-4 of a threshold, and the reference's nms_gpu / nms_normal_gpu keep lists at thresholds 0.01, 0.25 and 0.7."""
import os
import sys

import numpy as np
import torch

from oracle import build_ref, iou3d_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRESHOLDS = (0.01, 0.25, 0.7)


def ref_nms(R, boxes, scores, thresh, rotated):
    """iou3d_utils.py:31-56 / 106-124 over the reference extension"""
    order = scores.sort(0, descending=True)[1]
    b = boxes[order].contiguous()
    keep = torch.zeros(b.size(0), dtype=torch.long)
    num = (R.nms_gpu if rotated else R.nms_normal_gpu)(b, keep, float(thresh), b.device.index)
    return order[keep[:num].to(b.device)].contiguous()


def ref_matrix(R, fn, a, b):
    out = torch.zeros((a.shape[0], b.shape[0]), device=a.device)
    getattr(R, fn)(a.contiguous(), b.contiguous(), out)
    return out


def main(out_dir):
    R = build_ref.load_module("iou3d_ref")
    assert R is not None, "oracle/_ref/iou3d_ref*.so not built (python -m oracle.build_ref_iou3d)"
    dev = torch.device("cuda:0")
    sp = IO.special_boxes()
    dense = IO.synth_boxes(21, 300, objects=25)
    a = torch.cat([sp, dense[:150], IO.synth_boxes(22, 256 - sp.shape[0] - 150)])
    b = torch.cat([sp, dense[150:], IO.synth_boxes(23, 192 - sp.shape[0] - 150)])
    nb = IO.synth_boxes(24, 4000, objects=200)
    ok = np.intersect1d(IO.drop_near_threshold(nb, THRESHOLDS).numpy(), IO.drop_near_threshold(nb, THRESHOLDS, rotated=False).numpy())
    assert len(ok) >= 3000, len(ok)
    nb = nb[torch.from_numpy(ok[:3000])]
    ns = IO.distinct_scores(25, 3000)
    out = dict(boxes_a=a.numpy(), boxes_b=b.numpy(), nms_boxes=nb.numpy(), nms_scores=ns.numpy(),
               iou=ref_matrix(R, "boxes_iou_bev_gpu", a.to(dev), b.to(dev)).cpu().numpy(),
               overlap=ref_matrix(R, "boxes_overlap_bev_gpu", a.to(dev), b.to(dev)).cpu().numpy(),
               thresholds=np.array(THRESHOLDS, np.float64))
    for t in THRESHOLDS:
        out[f"keep_rot_{t}"] = ref_nms(R, nb.to(dev), ns.to(dev), t, True).cpu().numpy()
        out[f"keep_normal_{t}"] = ref_nms(R, nb.to(dev), ns.to(dev), t, False).cpu().numpy()
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "iou3d_bev.npz"), **out)
    print("wrote", os.path.join(out_dir, "iou3d_bev.npz"), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
