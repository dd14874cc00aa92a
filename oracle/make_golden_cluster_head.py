"""TEST INFRASTRUCTURE - writes tests/golden/cluster_head_targets.npz from the reference's OWN SparseClusterHeadV2
(modify_gt_for_single_task + get_targets of sparse_cluster_head_v2.py, imported unmodified through oracle/cluster_head_ref.py) on the
CPU, so that the GPU test of the native targets is pinned to the reference itself where the reference tree is absent.
`python -m oracle.make_golden_cluster_head [OUT_DIR]`.

Contents, per case k: k/xyz [M, 3], k/inds [M, 3] (samples interleaved), k/boxes [G, 7], k/labels [G] global, k/box_sizes, and per task
t the reference's k/labels_t{t} [M] and k/targets_t{t} [M, 8].  Waymo's three single-class tasks and Argoverse 2's six multi-class groups,
with boxes stacked across classes, yaws of +-pi and a sample without clusters."""
import os
import sys

import numpy as np
import torch

from oracle import cluster_head_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"waymo": (CO.WAYMO_NAMES, CO.WAYMO_TASKS, [900, 0, 700], [40, 6, 30]),
         "argo": (CO.ARGO_NAMES, CO.ARGO_TASKS, [800, 600], [50, 35])}


def case(name):
    names, tasks, n, m = CASES[name]
    xyz, inds, B, L = CO.synth_clusters(sum(map(ord, name)), n, m, names)
    for b in range(len(B)):
        if B[b].shape[0] > 1:
            B[b][1::2] = B[b][0:-1:2]
            CO.yaw_pi(B[b])
    return names, tasks, xyz, inds, B, L


def compute():
    from oracle import cluster_head_ref as CR
    R = CR.load_cluster_head()
    out = {}
    for name in CASES:
        names, tasks, xyz, inds, B, L = case(name)
        head = CR.build_cluster_head(dict(CO.FSD_D1_HEAD, num_classes=len(names), class_names=names,
                                          tasks=[dict(class_names=t) for t in tasks], in_channel=8, shared_mlp_dims=[8]),
                                     CO.FSD_D1_TRAIN_CFG)
        out[f"{name}/xyz"], out[f"{name}/inds"] = xyz.numpy(), inds.numpy()
        out[f"{name}/boxes"], out[f"{name}/labels"] = torch.cat(B).numpy(), torch.cat(L).numpy()
        out[f"{name}/box_sizes"] = np.array([b.shape[0] for b in B], np.int64)
        for t in range(len(tasks)):
            gb, gl = head.modify_gt_for_single_task([R.Boxes(b) for b in B], L, t)
            lab, _, tg, _, _ = head.get_targets(len(tasks[t]), xyz, inds[:, 1], gb, gl)
            out[f"{name}/labels_t{t}"], out[f"{name}/targets_t{t}"] = lab.numpy(), tg.numpy()
    return out


def main(out_dir):
    out = compute()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "cluster_head_targets.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
