"""TEST INFRASTRUCTURE - writes tests/golden/voteseg_targets.npz from the reference's OWN VoteSegHead.get_targets
(segmentation_head.py:212-283, imported unmodified through oracle/voteseg_ref.py) on the CPU, so that the GPU test of the native targets
is pinned to the reference itself where the reference tree is absent.  `python -m oracle.make_golden_voteseg [OUT_DIR]`.

Contents, per case k of CASES: k/points [N, 5] (the samples concatenated), k/point_sizes, k/boxes [G, 7] bottom-centre, k/labels [G]
(-1 marks an invalid box), k/box_sizes, k/num_classes, and the reference's k/labels_t [N], k/vote_targets [N, 3], k/vote_mask [N].
The samples have overlapping boxes, invalid labels, yaws of +-pi, points on the faces and one ulp either side, a sample without GTs
and a sample without points."""
import os
import sys

import numpy as np
import torch

from oracle import voteseg_oracle as VO, voteseg_ref as VR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"waymo": (3, [2000, 800, 0, 1500], [60, 0, 8, 25]), "nusc": (10, [1500, 1000], [40, 30])}


def case(name):
    num_classes, n_points, n_boxes = CASES[name]
    P, B, L = VO.synth_batch(sum(map(ord, name)), n_points, n_boxes, num_classes)
    for b in range(len(P)):
        if n_points[b] and n_boxes[b]:
            P[b] = torch.cat([P[b], torch.nn.functional.pad(VO.face_points(B[b][:6]), (0, 2), value=0.5)])
    return num_classes, P, B, L


def main(out_dir):
    R = VR.load_voteseg_head()
    out = {}
    for name in CASES:
        num_classes, P, B, L = case(name)
        head = VR.build_voteseg_head(dict(in_channel=8, num_classes=num_classes, loss_decode=dict(type="CrossEntropyLoss"),
                                          loss_vote=dict(type="L1Loss")))
        t = head.get_targets(P, [R.Boxes(b) for b in B], L)
        out[f"{name}/points"] = torch.cat(P).numpy()
        out[f"{name}/point_sizes"] = np.array([p.shape[0] for p in P], np.int64)
        out[f"{name}/boxes"] = torch.cat(B).numpy()
        out[f"{name}/labels"] = torch.cat(L).numpy()
        out[f"{name}/box_sizes"] = np.array([b.shape[0] for b in B], np.int64)
        out[f"{name}/num_classes"] = np.array(num_classes, np.int64)
        for k, key in enumerate(("labels_t", "vote_targets", "vote_mask")):
            out[f"{name}/{key}"] = t[k].numpy()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "voteseg_targets.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
