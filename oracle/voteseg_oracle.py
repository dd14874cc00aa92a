"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of VoteSegHead's training path (mmdet3d/models/decode_heads/segmentation_head.py): get_targets (lines 212-283) with
the reference's fp32 expressions, the two losses of `losses` (lines 107-142) in whatever dtype the predictions have (float64 for the
gradient checks, through autograd), and the training-log metrics (lines 146-171).  Pinned to the reference's own head by
tests/test_oracle_voteseg_vs_reference.py; also the synthetic frames the GPU tests and the benchmark use."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import roiaware_oracle as RA

# Waymo D1 (configs/fsd/fsd_waymoD1_1x.py): car / pedestrian / cyclist sizes (w, l, h) and bottom z
WAYMO_SIZES = ((2.1, 4.7, 1.7), (0.9, 0.9, 1.75), (0.85, 1.8, 1.6))
WAYMO_CFG = dict(use_sigmoid=True, gamma=3.0, alpha=0.8, score_thresh=(0.3, 0.25, 0.25), class_names=("Car", "Ped", "Cyc"))


def gravity_center(boxes):
    return torch.cat([boxes[:, :2], boxes[:, 2:3] + boxes[:, 5:6] * 0.5], 1)


def ieee_sqrt(x):
    """the correctly rounded fp32 square root, as torch's `** 0.5` gives it on the GPU where the reference runs get_targets.  torch's CPU
    kernel (a vectorised approximation) can be one ulp off it, so the reference run on the CPU is compared within one ulp."""
    return torch.from_numpy(np.sqrt(x.numpy()))


def targets(points_list, boxes_list, labels_list, bg_label):
    """(labels int64 [N], vote_targets f32 [N, 3], vote_mask bool [N]) of get_targets: the lowest-index valid box holding a point
    (points_in_boxes_gpu's first hit among the boxes with label >= 0), sign(d) sqrt(|d|) of gravity_center - point in fp32 with a correctly
    rounded square root"""
    labs, vts, masks = [], [], []
    for pts, boxes, lab in zip(points_list, boxes_list, labels_list):
        p = pts[:, :3].float()
        valid = lab >= 0
        b, bl = boxes[valid][:, :7].float(), lab[valid].long()
        n = p.shape[0]
        if bl.numel() == 0 or n == 0:
            labs.append(torch.full((n,), bg_label, dtype=torch.long))
            vts.append(torch.zeros((n, 3)))
            masks.append(torch.zeros((n,), dtype=torch.bool))
            continue
        inbox = RA.points_in_boxes_gpu(p[None], b[None])[0].long()
        hit = inbox >= 0
        k = inbox.clamp(min=0)
        delta = gravity_center(b)[k] - p
        delta[~hit] = 0
        labs.append(torch.where(hit, bl[k], torch.full_like(k, bg_label)))
        vts.append(torch.sign(delta) * ieee_sqrt(delta.abs()))
        masks.append(hit)
    return torch.cat(labs), torch.cat(vts), torch.cat(masks)


def losses(seg_logits, vote_preds, labels, vote_targets, vote_mask, use_sigmoid, gamma=2.0, alpha=0.25, class_weight=None,
           logit_scale=1.0, loss_weight=1.0, loss_weight_vote=1.0, **_):
    """(loss_sem_seg, loss_vote) in the predictions' dtype: sigmoid focal mean over N C elements or softmax cross-entropy w[y] / N, and
    the L1 of the valid points' own-class vote channels over 3 n_valid (vote_preds.sum() * 0 with no valid point)"""
    x = seg_logits * logit_scale
    N, C = x.shape
    if use_sigmoid:
        t = F.one_hot(labels, C + 1)[:, :C].to(x.dtype)
        p = x.sigmoid()
        loss = alpha * t * (1 - p).pow(gamma) * F.softplus(-x) + (1 - alpha) * (1 - t) * p.pow(gamma) * F.softplus(x)
        seg = loss_weight * loss.sum() / (N * C)
    else:
        w = x.new_ones(C) if class_weight is None else x.new_tensor(class_weight)
        nll = torch.logsumexp(x, 1) - x.gather(1, labels[:, None])[:, 0]
        seg = loss_weight * (w[labels] * nll).sum() / N
    m = vote_mask.bool()
    nv = int(m.sum())
    if nv == 0:
        return seg, vote_preds.sum() * 0
    v = vote_preds.reshape(N, C, 3)[m]
    v = v[torch.arange(nv), labels[m]]
    vote = loss_weight_vote * (v - vote_targets[m].to(v.dtype)).abs().sum() / (3 * nv)
    return seg, vote


def scores(seg_logits, use_sigmoid, logit_scale=1.0, class_names=None, group_names=None, **_):
    """[N, G] float64 scores the training log thresholds: sigmoid per class, or the group sums of the softmax (background excluded)"""
    x = seg_logits.double() * logit_scale
    if use_sigmoid:
        return x.sigmoid()
    p = x.softmax(1)[:, :-1]
    return torch.stack([p[:, [list(class_names).index(n) for n in g]].sum(1) for g in group_names], 1)


def metrics(seg_logits, labels, use_sigmoid, score_thresh, class_names, group_names=None, logit_scale=1.0, **_):
    """the training-log dict of lines 146-171: recall_<name> = tp / (real + 1e-5) in fp32, and num_fg [1] for softmax heads"""
    s = scores(seg_logits, use_sigmoid, logit_scale, class_names, group_names)
    out = {}
    if use_sigmoid:
        for i, thr in enumerate(score_thresh):
            pred, real = s[:, i] > thr, labels == i
            out[f"recall_{class_names[i]}"] = (pred & real).sum().float() / (real.sum().float() + 1e-5)
        return out
    num_fg = torch.zeros(1)
    for gi, g in enumerate(group_names):
        pred = s[:, gi] > score_thresh[gi]
        num_fg += pred.sum().float()
        for n in g:
            real = labels == list(class_names).index(n)
            out[f"recall_{n}"] = (pred & real).sum().float() / (real.sum().float() + 1e-5)
    out["num_fg"] = num_fg
    return out


# ---- the loss settings of the tests: C = 3 (Waymo), 1, 10 + 1 (nuScenes) and 26 + 1 (Argoverse 2) ----
ARGO_NAMES = tuple(f"c{i}" for i in range(26))
LOSS_MODES = {
    "waymo_focal": dict(num_classes=3, loss_decode=dict(type="FocalLoss", use_sigmoid=True, gamma=3.0, alpha=0.8, loss_weight=1.0),
                        train_cfg=dict(score_thresh=(0.3, 0.25, 0.25), class_names=("Car", "Ped", "Cyc"))),
    "focal_one_class": dict(num_classes=1, loss_decode=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
                            logit_scale=0.5, train_cfg=dict(score_thresh=(0.4,), class_names=("Car",))),
    "nusc_ce": dict(num_classes=10, loss_decode=dict(type="CrossEntropyLoss", use_sigmoid=False, class_weight=[1.0] * 10 + [0.1],
                                                     loss_weight=3.0), logit_scale=2.0,
                    train_cfg=dict(score_thresh=(0.25, 0.25, 0.25, 0.25), class_names=tuple(f"n{i}" for i in range(10)),
                                   group_names=[["n0", "n1"], ["n2", "n3", "n4"], ["n5", "n6", "n7"], ["n8", "n9"]])),
    "argo_ce": dict(num_classes=26, loss_decode=dict(type="CrossEntropyLoss", use_sigmoid=False,
                                                     class_weight=[float(1 + i % 3) for i in range(26)] + [0.1], loss_weight=3.0),
                    train_cfg=dict(score_thresh=(0.1, 0.05, 0.08, 0.04), class_names=ARGO_NAMES,
                                   group_names=[list(ARGO_NAMES[:7]), list(ARGO_NAMES[7:13]), list(ARGO_NAMES[13:20]),
                                                list(ARGO_NAMES[20:])])),
}


def head_cfg(mode):
    m = LOSS_MODES[mode]
    return dict(type="VoteSegHead", in_channel=16, hidden_dims=[32], num_classes=m["num_classes"], dropout_ratio=0.0,
                loss_decode=m["loss_decode"], loss_vote=dict(type="L1Loss", loss_weight=1.5), logit_scale=m.get("logit_scale", 1))


def loss_kwargs(mode):
    """the oracle's / ops.VoteSegLossConfig's keywords for a mode"""
    m = LOSS_MODES[mode]
    d = m["loss_decode"]
    sig = d["type"] == "FocalLoss"
    return dict(use_sigmoid=sig, gamma=d.get("gamma", 2.0), alpha=d.get("alpha", 0.25), class_weight=d.get("class_weight"),
                logit_scale=m.get("logit_scale", 1.0), loss_weight=d.get("loss_weight", 1.0), loss_weight_vote=1.5,
                **m["train_cfg"])


# ---- synthetic data ----
def _ulp(x, k):
    v = np.float32(x)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return float(v)


def synth_boxes(g, n, num_classes=3, spread=40.0, invalid=0.1, sizes=WAYMO_SIZES):
    """[n, 7] bottom-centre boxes in a car / pedestrian / cyclist mix (60 / 25 / 15 %), some overlapping (every fifth box is moved onto
    its predecessor), yaws over [-pi, pi] with +-pi exactly among them, and about `invalid` of the labels set to -1"""
    if n == 0:
        return torch.zeros((0, 7)), torch.zeros((0,), dtype=torch.long)
    probs = torch.tensor([0.6, 0.25, 0.15])[:min(num_classes, 3)]
    kind = torch.multinomial(probs / probs.sum(), n, replacement=True, generator=g)
    wlh = torch.tensor(sizes)[kind] * (0.8 + 0.4 * torch.rand((n, 3), generator=g))
    ctr = (torch.rand((n, 2), generator=g) * 2 - 1) * spread
    z = -1.0 + 0.3 * torch.randn((n, 1), generator=g)
    yaw = (torch.rand((n, 1), generator=g) * 2 - 1) * math.pi
    boxes = torch.cat([ctr, z, wlh, yaw], 1).float()
    boxes[4::5, :2] = boxes[3:-1:5, :2][:boxes[4::5].shape[0]] + 0.4          # overlapping pairs
    boxes[::7, 6] = torch.tensor([math.pi, -math.pi], dtype=torch.float32).repeat(n)[:boxes[::7].shape[0]]
    lab = torch.randint(0, num_classes, (n,), generator=g) if num_classes > 3 else kind.clone()
    lab[torch.rand(n, generator=g) < invalid] = -1
    return boxes, lab.long()


def points_around(g, boxes, n, spread=40.0, cols=5, inside=0.5):
    """[n, cols] fp32 points: `inside` of them drawn in the boxes' local frames (slightly beyond the faces too), the rest uniform"""
    k = int(n * inside) if boxes.shape[0] else 0
    pts = torch.empty((n, cols))
    pts[:, :2] = (torch.rand((n, 2), generator=g) * 2 - 1) * spread
    pts[:, 2] = -2 + 4 * torch.rand(n, generator=g)
    if k:
        b = boxes[torch.randint(0, boxes.shape[0], (k,), generator=g)]
        loc = (torch.rand((k, 3), generator=g) - 0.5) * 1.1 * b[:, [4, 3, 5]]
        c, s = torch.cos(b[:, 6]), torch.sin(b[:, 6])
        pts[:k, 0] = b[:, 0] + loc[:, 0] * c - loc[:, 1] * s
        pts[:k, 1] = b[:, 1] + loc[:, 0] * s + loc[:, 1] * c
        pts[:k, 2] = b[:, 2] + b[:, 5] * 0.5 + loc[:, 2]
    if cols > 3:
        pts[:, 3:] = torch.rand((n, cols - 3), generator=g)
    return pts.float()


def face_points(boxes):
    """points on the faces of each box along its local x / y / z axes, and one fp32 ulp either side of them"""
    out = []
    for b in boxes:
        x, y, zb, w, l, h, yaw = (float(v) for v in b)
        c, s = math.cos(yaw + math.pi / 2), math.sin(yaw + math.pi / 2)
        cz = zb + h / 2
        for lx, ly, z in ((l / 2, 0.0, cz), (-l / 2, 0.0, cz), (0.0, w / 2, cz), (0.0, -w / 2, cz), (0.0, 0.0, zb), (0.0, 0.0, zb + h)):
            # local (lx, ly) -> world with the in-box test's rotation by yaw + pi / 2 inverted
            px, py = x + lx * c + ly * s, y - lx * s + ly * c
            for k in (-1, 0, 1):
                out.append([_ulp(px, k), py, z])
                out.append([px, _ulp(py, k), z])
                out.append([px, py, _ulp(z, k)])
    return torch.tensor(out, dtype=torch.float32).reshape(-1, 3)


def synth_batch(seed, n_points, n_boxes, num_classes=3, spread=40.0, cols=5, invalid=0.1):
    """lists over samples of points [n_b, cols], boxes [g_b, 7] and labels [g_b]; n_points / n_boxes: one entry per sample"""
    g = torch.Generator().manual_seed(seed)
    P, Bx, Lb = [], [], []
    for n, m in zip(n_points, n_boxes):
        boxes, lab = synth_boxes(g, m, num_classes, spread, invalid)
        P.append(points_around(g, boxes, n, spread, cols))
        Bx.append(boxes)
        Lb.append(lab)
    return P, Bx, Lb


def synth_preds(seed, n, num_logits, scale=3.0):
    """seg_logits [n, C] and vote_preds [n, 3 C] fp32"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, num_logits), generator=g) * scale, torch.randn((n, 3 * num_logits), generator=g)


def clear_of_thresholds(seg_logits, cfg, margin=1e-5, seed=0, tries=50):
    """seg_logits with every row whose score lies within `margin` of its threshold redrawn, so that fp32 scores on the GPU and the
    float64 scores here make the same comparison"""
    if cfg.get("score_thresh") is None:
        return seg_logits
    g = torch.Generator().manual_seed(seed)
    x = seg_logits.clone()
    thr = torch.tensor(cfg["score_thresh"], dtype=torch.float64)
    for _ in range(tries):
        bad = ((scores(x, **cfg) - thr).abs() < margin).any(1)
        if not bad.any():
            return x
        x[bad] = torch.randn((int(bad.sum()), x.shape[1]), generator=g) * 3
    raise AssertionError("could not draw logits clear of the thresholds")


# the `segmentor` dict of configs/fsd/fsd_waymoD1_1x.py (pinned to the config by tests/test_oracle_voteseg_vs_reference.py), for the GPU
# training test where the reference tree is absent
FSD_D1_SEGMENTOR = dict(
    type='VoteSegmentor',
    voxel_layer=dict(voxel_size=(0.25, 0.25, 0.2), max_num_points=-1, point_cloud_range=[-80, -80, -2, 80, 80, 4], max_voxels=(-1, -1)),
    voxel_encoder=dict(type='DynamicScatterVFE', in_channels=5, feat_channels=[64, 64], voxel_size=(0.25, 0.25, 0.2),
                       with_cluster_center=True, with_voxel_center=True, point_cloud_range=[-80, -80, -2, 80, 80, 4],
                       norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01), unique_once=True),
    middle_encoder=dict(type='PseudoMiddleEncoderForSpconvFSD'),
    backbone=dict(type='SimpleSparseUNet', in_channels=64, sparse_shape=[32, 640, 640], order=('conv', 'norm', 'act'),
                  norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01), base_channels=64, output_channels=128,
                  encoder_channels=((64, ), (64, 64, 64), (64, 64, 64), (128, 128, 128), (256, 256, 256)),
                  encoder_paddings=((1, ), (1, 1, 1), (1, 1, 1), ((0, 1, 1), 1, 1), (1, 1, 1)),
                  decoder_channels=((256, 256, 128), (128, 128, 64), (64, 64, 64), (64, 64, 64), (64, 64, 64)),
                  decoder_paddings=((1, 1), (1, 0), (1, 0), (0, 0), (0, 1))),
    decode_neck=dict(type='Voxel2PointScatterNeck', voxel_size=(0.25, 0.25, 0.2), point_cloud_range=[-80, -80, -2, 80, 80, 4]),
    segmentation_head=dict(type='VoteSegHead', in_channel=67, hidden_dims=[128, 128], num_classes=3, dropout_ratio=0.0,
                           conv_cfg=dict(type='Conv1d'), norm_cfg=dict(type='naiveSyncBN1d'), act_cfg=dict(type='ReLU'),
                           loss_decode=dict(type='FocalLoss', use_sigmoid=True, gamma=3.0, alpha=0.8, loss_weight=1.0),
                           loss_vote=dict(type='L1Loss', loss_weight=1.0)),
    train_cfg=dict(point_loss=True, score_thresh=(0.3, 0.25, 0.25), class_names=('Car', 'Ped', 'Cyc'), centroid_offset=False),
)


def waymo_sweeps(seed, batch, n_points, n_boxes, spread=60.0):
    """Waymo-shaped training sweeps inside the D1 range: [n, 5] points (x, y, z, intensity, elongation) with half of them on ~n_boxes
    car / pedestrian / cyclist boxes, and the boxes / labels per sample (no invalid labels)"""
    P, B, L = synth_batch(seed, [n_points] * batch, [n_boxes] * batch, 3, spread=spread, invalid=0.0)
    for p in P:
        p[:, 2].clamp_(-1.9, 3.9)
    return P, B, L
