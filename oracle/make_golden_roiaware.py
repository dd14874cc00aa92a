"""TEST INFRASTRUCTURE - writes tests/golden/roiaware_pool3d.npz from the reference's OWN roiaware_pool3d CUDA kernels
(oracle/_ref/roiaware_pool3d_ext_ref*.so, built by oracle/build_ref_roiaware.py), so that the CPU oracle (oracle/roiaware_oracle.py) is
pinned to the reference where no GPU exists.  Needs a CUDA device.  `python -m oracle.make_golden_roiaware [OUT_DIR]` (default tests/golden).

Contents: the inputs of roiaware_oracle.golden_inputs() (overlapping RoIs, points on faces, a voxel with more than m - 1 points, out_size
(6, 4, 3), m = 8, features with ties, NaN and -inf); for mode 0 (max) and 1 (avg) the reference forward's pooled, argmax and
pts_idx_of_voxels and its backward's grad_in for a random grad_out; points_in_boxes_gpu / _batch on a 2-sample batch with padding boxes."""
import os
import sys

import numpy as np
import torch

from oracle import build_ref, roiaware_oracle as RA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ref_forward(R, rois, pts, feats, out_size, m, mode):
    """roiaware_pool3d.py:45-68 over the reference extension"""
    n = rois.shape[0]
    C = feats.shape[1]
    pooled = feats.new_zeros((n, *out_size, C))
    argmax = feats.new_zeros((n, *out_size, C), dtype=torch.int)
    pidx = feats.new_zeros((n, *out_size, m), dtype=torch.int)
    R.forward(rois.contiguous(), pts.contiguous(), feats.contiguous(), argmax, pidx, pooled, mode)
    return pooled, argmax, pidx


def ref_backward(R, pidx, argmax, grad_out, num_pts, mode):
    """roiaware_pool3d.py:70-86"""
    grad_in = grad_out.new_zeros((num_pts, grad_out.shape[-1]))
    R.backward(pidx, argmax, grad_out.contiguous(), grad_in, mode)
    return grad_in


def main(out_dir):
    R = build_ref.load_module("roiaware_pool3d_ext_ref")
    assert R is not None, "oracle/_ref/roiaware_pool3d_ext_ref*.so not built (python -m oracle.build_ref_roiaware)"
    dev = torch.device("cuda:0")
    x = RA.golden_inputs()
    out = {k: (v.numpy() if torch.is_tensor(v) else np.array(v)) for k, v in x.items()}
    rois, pts, feats, grad = (x[k].to(dev) for k in ("rois", "pts", "feats", "grad"))
    for mode in (0, 1):
        pooled, argmax, pidx = ref_forward(R, rois, pts, feats, x["out_size"], x["m"], mode)
        grad_in = ref_backward(R, pidx, argmax, grad, pts.shape[0], mode)
        out.update({f"pooled_{mode}": pooled.cpu().numpy(), f"argmax_{mode}": argmax.cpu().numpy(), f"pts_idx_{mode}": pidx.cpu().numpy(),
                    f"grad_in_{mode}": grad_in.cpu().numpy()})
    bp, bb = x["pib_pts"].to(dev), x["pib_boxes"].to(dev)
    first = torch.full(bp.shape[:2], -1, dtype=torch.int32, device=dev)
    R.points_in_boxes_gpu(bb, bp, first)
    every = torch.zeros((*bp.shape[:2], bb.shape[1]), dtype=torch.int32, device=dev)
    R.points_in_boxes_batch(bb, bp, every)
    out.update(pib_first=first.cpu().numpy(), pib_all=every.cpu().numpy())
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "roiaware_pool3d.npz"), **out)
    print("wrote", os.path.join(out_dir, "roiaware_pool3d.npz"), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
