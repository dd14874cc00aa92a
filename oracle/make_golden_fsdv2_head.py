"""TEST INFRASTRUCTURE - writes tests/golden/fsdv2_head_targets.npz from the reference's OWN FSDV2Head (modify_gt_for_single_task +
get_targets of fsd_v2_head.py, imported unmodified through oracle/fsdv2_head_ref.py) on the CPU, so that the GPU test of the native
targets is pinned to the reference itself where the reference tree is absent.  `python -m oracle.make_golden_fsdv2_head [OUT_DIR]`.

Contents, per case k: k/xyz [M, 3] (voxel centres), k/aux [M, 3] (centroids, the in-box test's points), k/inds [M, 3], k/boxes [G, W],
k/labels [G] global, k/box_sizes, and per task t the reference's k/labels_t{t} [M], k/targets_t{t} [M, 10] and k/weights_t{t} [M, 10].
nuScenes-shaped: two 5-class tasks, centroid assignment, 9-column GTs (velocity) and 10-column GTs (velocity and copy-paste flag),
boxes stacked across classes, yaws of +-pi."""
import os
import sys

import numpy as np
import torch

from oracle import cluster_head_oracle as CO
from oracle import fsdv2_head_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"nusc9": (9, [900, 700], [40, 30]), "nusc10": (10, [800, 0, 600], [35, 5, 30])}


def case(name):
    width, n, m = CASES[name]
    xyz, aux, inds, B, L = FO.synth_clusters(sum(map(ord, name)), n, m, FO.NUSC_NAMES, width=width)
    for b in B:
        if b.shape[0] > 1:
            CO.yaw_pi(b)
    return xyz, aux, inds, B, L


def compute():
    from oracle import fsdv2_head_ref as FR
    R = FR.load_fsdv2_head()
    out = {}
    head = FR.build_fsdv2_head(dict(FO.NUSC_HEAD, in_channel=8, shared_mlp_dims=[8]), FO.NUSC_TRAIN_CFG)
    for name in CASES:
        xyz, aux, inds, B, L = case(name)
        out[f"{name}/xyz"], out[f"{name}/aux"], out[f"{name}/inds"] = xyz.numpy(), aux.numpy(), inds.numpy()
        out[f"{name}/boxes"], out[f"{name}/labels"] = torch.cat(B).numpy(), torch.cat(L).numpy()
        out[f"{name}/box_sizes"] = np.array([b.shape[0] for b in B], np.int64)
        for t in range(len(FO.NUSC_TASKS)):
            gb, gl = head.modify_gt_for_single_task([R.Boxes(b) for b in B], L, t)
            lab, _, tg, w, _ = head.get_targets(len(FO.NUSC_TASKS[t]), xyz, inds[:, 1], gb, gl, aux_xyz=aux)
            out[f"{name}/labels_t{t}"], out[f"{name}/targets_t{t}"], out[f"{name}/weights_t{t}"] = lab.numpy(), tg.numpy(), w.numpy()
    return out


def main(out_dir):
    out = compute()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "fsdv2_head_targets.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
