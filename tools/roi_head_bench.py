"""FSD's second-stage training path on the GPU: assign + sample + targets + losses, forward and backward, native (GroupCorrectionHead /
FullySparseBboxHead of sst_b200) against a torch composition that follows the reference's per-sample, per-class loop
(fsd_roi_head.py:213-296, MaxIoUAssigner, IoUNegPiecewiseSampler, fsd_bbox_head.py get_targets / loss with the corner loss) over ops.boxes_overlap_bev for
the BEV term; and simple_test end to end.  Shape: FSD Waymo D1, B = 2 and 4, 500 proposals (the rpn max_num; real counts are not
measured) and about 200 GTs per sample, 150k points per sample.  Medians of alternating rounds: per-call time (CUDA events around
REPS calls), the GPU time of each call's kernels and copies alone (torch.profiler), peak extra device memory; card name and power
limit read in the same run.  Writes OUT/roi_head_bench.json.

    python tools/roi_head_bench.py [OUT]
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import voteseg_bench as VB  # noqa: E402

ROUNDS = 3
VB.REPS = 10
PROPS, GTS, POINTS = 500, 200, 150_000
ASSIGNERS = [(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)]
POS_THR, NEG_THR = (0.8, 0.65, 0.65), (0.2, 0.15, 0.15)
FSD_D1_BBOX_HEAD = dict(  # configs/fsd/fsd_waymoD1_1x.py roi_head.bbox_head
    type='FullySparseBboxHead', num_classes=3, num_blocks=6, in_channels=[213, 146, 146, 146, 146, 146], feat_channels=[[128, 128]] * 6,
    rel_mlp_hidden_dims=[[16, 32]] * 6, rel_mlp_in_channels=[13] * 6, reg_mlp=[512, 512], cls_mlp=[512, 512], mode='max',
    xyz_normalizer=[20, 20, 4], act='gelu', geo_input=True, with_corner_loss=True, corner_loss_weight=1.0,
    bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'), norm_cfg=dict(type='LN', eps=1e-3), unique_once=True,
    loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=2.0),
    loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='mean', loss_weight=1.0), cls_dropout=0.1, reg_dropout=0.1)


def iou3d_torch(ops, gt, p):
    from sst_b200.anchor3d_modules import xywhr2xyxyr
    bev = lambda b: xywhr2xyxyr(b[:, [0, 1, 3, 4, 6]])  # noqa: E731
    ov = ops.boxes_overlap_bev(bev(gt), bev(p))
    h = (torch.min((gt[:, 2] + gt[:, 5])[:, None], (p[:, 2] + p[:, 5])[None]) - torch.max(gt[:, 2][:, None], p[:, 2][None])).clamp(min=0)
    o3 = ov * h
    v = lambda b: b[:, 3] * b[:, 4] * b[:, 5]  # noqa: E731
    return o3 / (v(gt)[:, None] + v(p)[None] - o3).clamp(min=1e-8)


def choose(gallery, k, keys):
    return gallery[torch.argsort(keys[gallery], stable=True)[:k]]


def baseline(ops, props_l, plab_l, keys_l, gt_l, gl_l, cls, pred, num=256):
    """the reference's loops, restated on torch: returns the summed loss (backward-able)"""
    rows = []
    for props, plab, keys, gt, gl in zip(props_l, plab_l, keys_l, gt_l, gl_l):
        N = len(props)
        gi = gl.new_zeros(N)
        mo = props.new_zeros(N)
        lab = gl.new_full((N,), -1)
        for i, (pt, nt, mp) in enumerate(ASSIGNERS):
            gm, pm = gl == i, plab == i
            ov = iou3d_torch(ops, gt[gm], props[pm])
            G, n = ov.shape
            a = ov.new_full((n,), -1, dtype=torch.long)
            if G == 0 or n == 0:
                if G == 0:
                    a[:] = 0
                m_i = ov.new_zeros(n)
            else:
                m_i, arg = ov.max(0)
                gmax = ov.max(1)[0]
                a[(m_i >= 0) & (m_i < nt)] = 0
                a[m_i >= pt] = arg[m_i >= pt] + 1
                for g in range(G):
                    if gmax[g] >= mp:
                        a[ov[g] == gmax[g]] = g + 1
            pad = torch.cat([gl.new_tensor([-1, 0]), torch.nonzero(gm).view(-1) + 1])
            gi[pm] = pad[a + 1]
            mo[pm] = m_i
            lab[pm] = torch.where(a > 0, i, -1)
        pos = torch.nonzero(gi > 0).view(-1)
        if len(pos) > int(num * 0.55):
            pos = choose(pos, int(num * 0.55), keys)
        pos = pos.unique()
        nexp = num - len(pos)
        neg = torch.nonzero(gi == 0).view(-1)
        if len(neg) > nexp:
            choice, extend, m = neg.new_zeros([0]), 0, mo[neg]
            for q, (lo, hi) in enumerate(((0.1, 0.55), (0.0, 0.1))):
                want = int(nexp * 0.8) + extend if q == 0 else nexp - len(choice)
                piece = neg[(m >= lo) & (m < hi)]
                if len(piece) < want:
                    choice, extend = torch.cat([choice, piece]), extend + want - len(piece)
                else:
                    choice, extend = torch.cat([choice, choose(piece, want, keys)]), 0
            neg = choice
        neg = neg.unique()
        rows.append((props[torch.cat([pos, neg])], mo[torch.cat([pos, neg])], gt[gi[pos] - 1], lab[pos], len(pos)))
    labels, tg, pg, pl, rm, rois = [], [], [], [], [], []
    for r, iou, g, l, npos in rows:
        soft = torch.zeros_like(iou)
        for i in range(3):
            m = torch.zeros_like(iou, dtype=torch.bool)
            m[:npos] = l == i
            v = iou[m]
            s = (v > POS_THR[i]).float()
            mid = ~(v > POS_THR[i]) & ~(v < NEG_THR[i])
            s[mid] = (v[mid] - NEG_THR[i]) / (POS_THR[i] - NEG_THR[i])
            soft[m] = s
        p = r[:npos]
        ry = p[:, 6] % (2 * np.pi)
        ct = g.clone()
        d = g[:, :3] - p[:, :3]
        a = -(ry + np.pi / 2)
        ct[:, 0], ct[:, 1] = d[:, 0] * a.cos() + d[:, 1] * a.sin(), -d[:, 0] * a.sin() + d[:, 1] * a.cos()
        yl = (g[:, 6] - ry) % (2 * np.pi)
        opp = (yl > np.pi / 2) & (yl < np.pi * 1.5)
        yl[opp] = (yl[opp] + np.pi) % (2 * np.pi)
        yl[yl > np.pi] -= 2 * np.pi
        diag = (p[:, 4] ** 2 + p[:, 3] ** 2).sqrt()
        tg.append(torch.stack([ct[:, 0] / diag, ct[:, 1] / diag, (d[:, 2] + g[:, 5] / 2 - p[:, 5] / 2) / p[:, 5], (g[:, 3] / p[:, 3]).log(),
                               (g[:, 4] / p[:, 4]).log(), (g[:, 5] / p[:, 5]).log(), yl.clamp(-np.pi / 2, np.pi / 2)], 1))
        labels.append(soft), pg.append(g), pl.append(l), rois.append(r)
        m = torch.zeros(len(r), dtype=torch.long, device=r.device)
        m[:npos] = 1
        rm.append(m)
    labels, rm, rois = torch.cat(labels), torch.cat(rm), torch.cat(rois)
    x = cls[:len(labels)].view(-1)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(x, labels, reduction='sum') / len(labels)
    pos = rm > 0
    npos = int(pos.sum().item())
    pp = pred[:len(labels)][pos]
    loss = loss + 2.0 * (pp - torch.cat(tg)).abs().sum() / max(npos, 1)
    # get_corner_loss_lidar on the Car positives: decode against the RoI, corners, nearer of GT / flipped GT, Huber
    car = torch.cat(pl) == 0
    pb, rb, g = pp[car], rois[pos][car], torch.cat(pg)[car]
    if len(g):
        diag = (rb[:, 4] ** 2 + rb[:, 3] ** 2).sqrt()
        h = pb[:, 5].exp() * rb[:, 5]
        loc = torch.stack([pb[:, 0] * diag, pb[:, 1] * diag, pb[:, 2] * rb[:, 5] + rb[:, 5] / 2 - h / 2], 1)
        a = rb[:, 6] + np.pi / 2
        xyz = torch.stack([loc[:, 0] * a.cos() + loc[:, 1] * a.sin(), -loc[:, 0] * a.sin() + loc[:, 1] * a.cos(), loc[:, 2]], 1) + rb[:, :3]
        box = torch.cat([xyz, (pb[:, 3].exp() * rb[:, 3])[:, None], (pb[:, 4].exp() * rb[:, 4])[:, None], h[:, None],
                         (pb[:, 6] + rb[:, 6])[:, None]], 1)
        gf = g.clone()
        gf[:, 6] += np.pi
        d = torch.min(torch.norm(corners(box) - corners(g), dim=2), torch.norm(corners(box) - corners(gf), dim=2))
        q = d.clamp(max=1.0)
        loss = loss + (0.5 * q ** 2 + (d - q)).mean()
    return loss


def corners(b):
    """LiDARInstance3DBoxes.corners"""
    u = b.new_tensor([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]]) - b.new_tensor([0.5, 0.5, 0])
    c = b[:, None, 3:6] * u[None]
    s, co = b[:, 6:7].sin(), b[:, 6:7].cos()
    return torch.stack([c[..., 0] * co + c[..., 1] * s, -c[..., 0] * s + c[..., 1] * co, c[..., 2]], -1) + b[:, None, :3]


def main(out_dir):
    from oracle import roi_head_oracle as RO
    from sst_b200 import ops
    from sst_b200.roi_head_modules import FullySparseBboxHead
    from sst_b200.roi_head_modules import GroupCorrectionHead
    dev = torch.device("cuda:0")
    name, power = VB.card()
    rec = {"card": name, "power_limit": power, "shape": f"FSD Waymo D1: {PROPS} proposals (rpn max_num) and ~{GTS} GTs per sample, "
           f"{POINTS} points per sample", "reps": VB.REPS, "rounds": ROUNDS, "results": {}}
    for B in (2, 4):
        data = [RO.synth_sample(1000 + b, PROPS, GTS, spread=60.0) for b in range(B)]
        props_l = [d[0].to(dev) for d in data]
        plab_l = [d[1].to(dev) for d in data]
        gt_l = [d[2].to(dev) for d in data]
        gl_l = [d[3].to(dev) for d in data]
        props, plab, gt, gl = torch.cat(props_l), torch.cat(plab_l), torch.cat(gt_l), torch.cat(gl_l)
        keys = torch.rand(len(props), device=dev)
        keys_l = list(keys.split([PROPS] * B))
        cfg = ops.RoiSampleConfig([a[0] for a in ASSIGNERS], [a[1] for a in ASSIGNERS], [a[2] for a in ASSIGNERS], True, 256, 0.55,
                                  [0.8, 0.2], [0.55, 0.1])
        head = FullySparseBboxHead(num_classes=3, num_blocks=1,
                                   in_channels=[16], feat_channels=[[8]], rel_mlp_hidden_dims=[[8]], rel_mlp_in_channels=[13],
                                   reg_mlp=None, cls_mlp=None, with_corner_loss=True, norm_cfg=dict(type='LN', eps=1e-3),
                                   loss_bbox=dict(type='L1Loss', loss_weight=2.0),
                                   loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='mean'))
        head.train_cfg = dict(cls_pos_thr=POS_THR, cls_neg_thr=NEG_THR, class_names=['Car', 'Pedestrian', 'Cyclist'])
        cls = torch.randn(B * 256, 1, device=dev, requires_grad=True)
        pred = (0.1 * torch.randn(B * 256, 7, device=dev)).requires_grad_()

        def native():
            inds, iou, gt_rows, lab, num_pos, num_rows = ops.roi_assign_sample(props, plab, [PROPS] * B, keys, gt, gl, [GTS] * B, cfg)
            from sst_b200.roi_head_modules import RoiSampling
            bidx = torch.cat([torch.full((n,), b, device=dev) for b, n in enumerate(num_rows)])
            s = RoiSampling(bidx, props[inds], iou, gt_rows, lab, gt, num_pos, num_rows)
            t = head.get_targets(s, head.train_cfg)
            R = len(inds)
            rois = torch.cat([bidx[:, None].float(), s.bboxes], 1)
            ne = torch.ones(R, dtype=torch.bool, device=dev)
            l = head.loss(cls[:R], pred[:R], ne, rois, *t)
            (l['loss_rcnn_cls'] + l['loss_rcnn_bbox'] + l['loss_rcnn_corner']).backward()

        def torch_ref():
            baseline(ops, props_l, plab_l, keys_l, gt_l, gl_l, cls, pred).backward()

        res = {"native": [], "torch": []}
        for fn in (native, torch_ref):
            fn()
        for _ in range(ROUNDS):
            for k, fn in (("native", native), ("torch", torch_ref)):
                ms, mib, _ = VB.timed(fn)
                res[k].append((ms, VB.device_ms(fn), mib))
        out = {}
        for k, v in res.items():
            a = np.array(v)
            out[k] = {"ms_per_call": float(np.median(a[:, 0])), "gpu_ms_per_call": float(np.median(a[:, 1])),
                      "peak_extra_mib": float(np.median(a[:, 2]))}
        out["speedup"] = out["torch"]["ms_per_call"] / out["native"]["ms_per_call"]
        rec["results"][f"train_B{B}"] = out
        print(f"B={B}: native {out['native']}, torch {out['torch']}, speedup {out['speedup']:.1f}x")
    # simple_test end to end: FSD Waymo D1 head (6 SIR blocks), one sample
    head = GroupCorrectionHead(num_classes=3, roi_extractor=dict(type='DynamicPointROIExtractor', extra_wlh=[0.5, 0.5, 0.5],
                                                                 max_inbox_point=256, debug=False),
                               bbox_head=FSD_D1_BBOX_HEAD).to(dev).eval()
    head.test_cfg = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=0.25, score_thr=0.1, min_bbox_size=0, max_num=500)
    head.bbox_head.test_cfg = head.test_cfg
    props, plab, gt, gl = RO.synth_sample(7, PROPS, GTS, spread=60.0)
    g = torch.Generator().manual_seed(0)
    k = torch.randint(0, GTS, (POINTS,), generator=g)
    xyz = (gt[k, :3] + torch.randn(POINTS, 3, generator=g) * torch.tensor([1.5, 1.5, 0.5])).to(dev)
    xyz = torch.cat([xyz, torch.rand(POINTS, 2, device=dev)], 1)   # x, y, z, intensity, elongation: 5 + 195 + 13 = 213 inputs
    feats = torch.randn(POINTS, 195, device=dev)
    bidx = torch.zeros(POINTS, dtype=torch.long, device=dev)
    pr = [(props.to(dev), torch.rand(PROPS, device=dev), plab.to(dev))]

    def st():
        with torch.no_grad():
            head.simple_test(xyz, feats, bidx, [{}], [(a.clone(), b.clone(), c.clone()) for a, b, c in pr], None, None)

    st()
    v = []
    for _ in range(ROUNDS):
        ms, mib, _ = VB.timed(st)
        v.append((ms, VB.device_ms(st), mib))
    a = np.array(v)
    rec["results"]["simple_test_B1"] = {"ms_per_call": float(np.median(a[:, 0])), "gpu_ms_per_call": float(np.median(a[:, 1])),
                                        "peak_extra_mib": float(np.median(a[:, 2]))}
    print("simple_test:", rec["results"]["simple_test_B1"])
    print(f"card: {name}, power limit {power}")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "roi_head_bench.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "bench_out")
