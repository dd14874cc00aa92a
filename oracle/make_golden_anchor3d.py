"""TEST INFRASTRUCTURE - writes tests/golden/anchor3d_targets.npz from the reference's OWN anchor_target_3d (train_mixins.py, with
anchor3d_head.py and the reference's anchor generator, box coder and IoU calculator, imported unmodified through
oracle/anchor3d_ref.py) on the CPU, so that the GPU test of the native targets is pinned to the reference itself where the reference
tree is absent.  `python -m oracle.make_golden_anchor3d [OUT_DIR]`.

Contents, per case k of CASES (a 60 x 44 map, 3 sizes x 2 rotations, two samples, the second without GTs): k/boxes (bottom-centre,
both samples concatenated), k/labels, k/sizes, and the reference's k/labels_t, k/label_weights, k/bbox_targets, k/bbox_weights,
k/dir_targets, k/dir_weights [2, A(, 7)] and k/num_total_pos."""
import os
import sys

import numpy as np
import torch

from oracle import anchor3d_oracle as AO, anchor3d_ref as AR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"default": {}, "per_class": dict(assign_per_class=True), "argmax_only": dict(gt_max_assign_all=False)}
SIZES = [60, 0]


def main(out_dir):
    R = AR.load_anchor_head()
    out = {}
    for name, kw in CASES.items():
        geom = AO.geometry(**kw)
        head = AR.build_anchor_head(geom)
        boxes, labels = AO.synth_batch(7, geom, SIZES)
        anchors = head.get_anchors([(geom["H"], geom["W"])], [{}] * len(SIZES), device="cpu")
        t = head.anchor_target_3d(anchors, [R.Boxes(b) for b in boxes], [{}] * len(SIZES), gt_labels_list=labels,
                                  num_classes=geom["head"]["num_classes"], label_channels=1, sampling=False)
        out[f"{name}/boxes"] = torch.cat(boxes).numpy()
        out[f"{name}/labels"] = torch.cat(labels).numpy()
        out[f"{name}/sizes"] = np.array(SIZES, np.int64)
        for k, key in enumerate(("labels_t", "label_weights", "bbox_targets", "bbox_weights", "dir_targets", "dir_weights")):
            out[f"{name}/{key}"] = t[k][0].numpy()
        out[f"{name}/num_total_pos"] = np.array(t[6], np.int64)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "anchor3d_targets.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
