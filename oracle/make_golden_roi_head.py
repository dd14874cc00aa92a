"""Writes tests/golden/roi_head_targets.npz: the reference's own FSD second-stage assignment, sampling and targets (through
oracle/roi_head_ref.py, fp32) for a seeded two-sample batch.  Also the shared settings of the second-stage tests.

    python -m oracle.make_golden_roi_head
"""
import os

import numpy as np
import torch

from oracle import roi_head_oracle as RO

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "roi_head_targets.npz")
ASSIGNERS = [(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)]
POS_THR, NEG_THR = (0.8, 0.65, 0.65), (0.2, 0.15, 0.15)
THRESHOLDS = [0.45, 0.35, 0.55, 0.1, 0.8, 0.65, 0.2, 0.15]
CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']


def train_cfg(per_class=True, num=256):
    a = [dict(type='MaxIoUAssigner', iou_calculator=dict(type='BboxOverlaps3D', coordinate='lidar'), pos_iou_thr=p, neg_iou_thr=n,
              min_pos_iou=m, ignore_iof_thr=-1) for p, n, m in ASSIGNERS]
    return dict(assigner=a if per_class else a[0],
                sampler=dict(type='IoUNegPiecewiseSampler', num=num, pos_fraction=0.55, neg_piece_fractions=[0.8, 0.2],
                             neg_iou_piece_thrs=[0.55, 0.1], neg_pos_ub=-1, add_gt_as_proposals=False, return_iou=True),
                cls_pos_thr=POS_THR, cls_neg_thr=NEG_THR, sync_reg_avg_factor=True, sync_cls_avg_factor=True, corner_loss_only_car=True,
                class_names=CLASS_NAMES)


def small_head():
    """a 2-block FullySparseBboxHead with the FSD loss settings"""
    return dict(type='FullySparseBboxHead', num_classes=3, num_blocks=2, in_channels=[3 + 8 + 13, 3 + 32 + 13],
                feat_channels=[[32, 32], [32, 32]], rel_mlp_hidden_dims=[[16, 32]] * 2, rel_mlp_in_channels=[13] * 2, reg_mlp=[32],
                cls_mlp=[32], mode='max', xyz_normalizer=[20, 20, 4], act='gelu', geo_input=True, with_corner_loss=True,
                corner_loss_weight=1.0, norm_cfg=dict(type='LN', eps=1e-3), unique_once=True,
                loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=2.0),
                loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='mean', loss_weight=1.0), cls_dropout=0.1,
                reg_dropout=0.1)


def batch(specs, seed=0, gt_width=7, per_class=True):
    """(props, plabels, gt, gt labels) per sample for specs (n_props, n_gt), re-drawn until no IoU the assigner sees lies within 1e-4
    of a threshold"""
    out = []
    for b, (n, g) in enumerate(specs):
        s = seed * 100 + b
        while True:
            p, l, gt, gl = RO.synth_sample(s, n, g, gt_width=gt_width)
            if not RO.near_threshold(p, l, gt, gl, THRESHOLDS, per_class=per_class):
                break
            s += 1000
        out.append((p, l, gt, gl))
    return out


def golden_inputs(seed=7):
    data = batch([(400, 120), (300, 90)], seed=seed)
    keys = [torch.rand(len(p), generator=torch.Generator().manual_seed(seed + b)) for b, (p, _, _, _) in enumerate(data)]
    return data, keys


def reference_sampling(N, cfg, inp, dtype=torch.float32):
    data, keys = inp
    props = [(N.Boxes(p.to(dtype)), torch.rand(len(p)), l) for p, l, _, _ in data]
    return N.assign_and_sample(cfg, props, [N.Boxes(g.to(dtype)) for _, _, g, _ in data], [l for _, _, _, l in data],
                               [k.to(dtype) for k in keys])


def reference_targets(N, cfg, inp):
    """inputs and the reference's fp32 sampling and targets as numpy arrays"""
    data, keys = inp
    head = N.build_head(small_head(), cfg)
    res = reference_sampling(N, cfg, inp)
    label, bbox_targets, bidx, pos_gt, pos_lab, reg_mask, _, _ = head.get_targets(res, cfg)
    out = {}
    for b, ((p, l, g, gl), k) in enumerate(zip(data, keys)):
        out[f"props{b}"], out[f"plabels{b}"], out[f"gt{b}"], out[f"gt_labels{b}"], out[f"keys{b}"] = \
            p.numpy(), l.numpy(), g.numpy(), gl.numpy(), k.numpy()
        r = res[b]
        out[f"inds{b}"] = torch.cat([r.pos_inds, r.neg_inds]).numpy()
        out[f"num_pos{b}"] = np.array(len(r.pos_inds))
        out[f"iou{b}"] = r.iou.float().numpy()
        out[f"gt_rows{b}"] = r.pos_assigned_gt_inds.numpy()
    out["soft_labels"] = label.float().numpy()
    out["bbox_targets"] = bbox_targets.float().numpy()
    out["reg_mask"] = reg_mask.numpy()
    out["pos_gt_labels"] = pos_lab.numpy()
    return out



def main():
    from oracle import roi_head_ref as RR
    N = RR.load_roi_head()
    out = reference_targets(N, RR.Cfg(train_cfg()), golden_inputs())
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
