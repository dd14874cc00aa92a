"""TEST INFRASTRUCTURE - writes tests/golden/centerpoint_targets.npz from the reference's OWN CenterHead.get_targets
(centerpoint_head.py, imported unmodified through oracle/centerpoint_ref.py) on the CPU, so that the GPU test of the native targets is
pinned to the reference itself where the reference tree is absent.  `python -m oracle.make_golden_centerpoint [OUT_DIR]`.

Contents, per geometry g of oracle/centerpoint_oracle.GEOMETRIES ('waymo', 'nusc'): g/boxes (raw LiDAR boxes, bottom-centre z, all samples
concatenated), g/labels, g/sizes (boxes per sample, edge cases included; an empty sample and one above max_objs), and per task t: g/t/anno_box, g/t/ind,
g/t/mask, and the heatmap as its non-zero support g/t/hm_index (flat int64) and g/t/hm_value."""
import os
import sys

import numpy as np

from oracle import centerpoint_oracle as CO, centerpoint_ref as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = {"waymo": [30, 0, 520], "nusc": [25, 40]}


def main(out_dir):
    R = CR.load_center_head()
    out = {}
    for geom, sizes in SIZES.items():
        boxes, labels = CO.synth_batch(2024, geom, sizes)
        head = CR.build_center_head(CO.head_cfg(geom))
        hm, ab, ind, mask = head.get_targets([R.Boxes(b) for b in boxes], labels)
        import torch
        out[f"{geom}/boxes"] = torch.cat(boxes).numpy()
        out[f"{geom}/labels"] = torch.cat(labels).numpy()
        out[f"{geom}/sizes"] = np.array([b.shape[0] for b in boxes], np.int64)
        for t in range(len(hm)):
            flat = hm[t].reshape(-1)
            nz = torch.nonzero(flat)[:, 0]
            out[f"{geom}/{t}/hm_index"] = nz.numpy()
            out[f"{geom}/{t}/hm_value"] = flat[nz].numpy()
            out[f"{geom}/{t}/anno_box"] = ab[t].numpy()
            out[f"{geom}/{t}/ind"] = ind[t].numpy()
            out[f"{geom}/{t}/mask"] = mask[t].numpy()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "centerpoint_targets.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
