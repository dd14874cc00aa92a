"""GPU: FSD's second stage (sst_b200/roi_head_modules.py, csrc/roi_head.cu) against the float64 restatement oracle/roi_head_oracle.py:
assignment and sampling (indices exact on box sets with no IoU near a threshold, IoU within 1e-5), targets, the three losses and their
gradients, determinism and host syncs, simple_test and one training step of GroupCorrectionHead."""
import math

import pytest
import torch

import numpy as np

from oracle import make_golden_roi_head as MG
from oracle import roi_head_oracle as RO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ASSIGNERS, POS_THR, NEG_THR, CLASS_NAMES = MG.ASSIGNERS, MG.POS_THR, MG.NEG_THR, MG.CLASS_NAMES


def _ops():
    from sst_b200 import ops
    return ops


def _cfg(num=256, pos_fraction=0.55, per_class=True):
    a = ASSIGNERS if per_class else ASSIGNERS[:1]
    return _ops().RoiSampleConfig([x[0] for x in a], [x[1] for x in a], [x[2] for x in a], per_class, num, pos_fraction, [0.8, 0.2],
                                  [0.55, 0.1])


def _batch(specs, seed=0, gt_width=7, per_class=True):
    """specs: (n_props, n_gt) per sample, no IoU the assigner sees within 1e-4 of a threshold"""
    return MG.batch(specs, seed, gt_width=gt_width, per_class=per_class)


def _native(batch, cfg, keys):
    ops = _ops()
    props = torch.cat([p for p, _, _, _ in batch]).to(DEV)
    plab = torch.cat([l for _, l, _, _ in batch]).to(DEV)
    gt = torch.cat([g for _, _, g, _ in batch]).to(DEV)
    gl = torch.cat([l for _, _, _, l in batch]).to(DEV)
    return ops.roi_assign_sample(props, plab, [len(p) for p, _, _, _ in batch], keys.to(DEV), gt, gl, [len(g) for _, _, g, _ in batch],
                                 cfg)


def _oracle(batch, keys, num=256, pos_fraction=0.55, per_class=True):
    rows, at, gat = [], 0, 0
    for props, plab, gt, gl in batch:
        k = keys[at:at + len(props)]
        inds, iou, grows, lab, npos = RO.assign_and_sample(props, plab, k, gt, gl, ASSIGNERS if per_class else ASSIGNERS[:1], per_class,
                                                           num, pos_fraction, [0.8, 0.2], [0.55, 0.1])
        rows.append((inds + at, iou, torch.where(grows >= 0, grows + gat, grows), lab, npos))
        at += len(props)
        gat += len(gt)
    return rows


@pytest.mark.parametrize("specs,num,gt_width,per_class", [
    ([(500, 200), (500, 180)], 256, 7, True),         # more proposals than num
    ([(120, 40), (60, 30)], 256, 7, True),            # fewer
    ([(300, 60), (1, 0), (200, 50)], 128, 7, True),   # a sample of one proposal without GTs
    ([(400, 100)], 128, 9, True),
    ([(400, 100), (300, 80)], 128, 10, False),        # one assigner over every GT
])
def test_assign_sample_matches_oracle(specs, num, gt_width, per_class):
    batch = _batch(specs, seed=len(specs) + num, gt_width=gt_width, per_class=per_class)
    P = sum(len(b[0]) for b in batch)
    keys = torch.rand(P, generator=torch.Generator().manual_seed(5))
    cfg = _cfg(num, per_class=per_class)
    inds, iou, gt_rows, lab, num_pos, num_rows = _native(batch, cfg, keys)
    ref = _oracle(batch, keys, num, per_class=per_class)
    assert num_pos == [r[4] for r in ref]
    assert num_rows == [len(r[0]) for r in ref]
    assert torch.equal(inds.cpu(), torch.cat([r[0] for r in ref]))
    assert torch.equal(gt_rows.cpu(), torch.cat([r[2] for r in ref]))
    assert torch.equal(lab.cpu(), torch.cat([r[3] for r in ref]))
    assert (iou.cpu().double() - torch.cat([r[1] for r in ref])).abs().max().item() < 1e-5


def test_class_without_gt_and_low_quality_match():
    # class 2 has no GT: its proposals are negatives with IoU 0.  Proposal 1 overlaps GT 0 most (0.77) but is GT 1's best proposal
    # (0.64 >= min_pos_iou): match_low_quality gives it to GT 1.
    gt = torch.tensor([[0, 0, 0, 2, 4.5, 1.6, 0], [0, 1.6, 0, 2, 4.5, 1.6, 0]], dtype=torch.float32)
    gl = torch.tensor([0, 0])
    props = torch.tensor([[0, 0.05, 0, 2, 4.5, 1.6, 0], [0, 0.6, 0, 2, 4.5, 1.6, 0], [12.5, 1.0, 0, 2, 4.5, 1.6, 0],
                          [0, 0, 0, 2, 4.5, 1.6, 0], [30, 30, 0, 2, 2, 2, 0]], dtype=torch.float32)
    plab = torch.tensor([0, 0, 0, 2, 2])
    batch = [(props, plab, gt, gl)]
    keys = torch.rand(5, generator=torch.Generator().manual_seed(1))
    inds, iou, gt_rows, lab, num_pos, _ = _native(batch, _cfg(), keys)
    ref = _oracle(batch, keys)[0]
    assert torch.equal(inds.cpu(), ref[0]) and torch.equal(gt_rows.cpu(), ref[2]) and torch.equal(lab.cpu(), ref[3])
    ov = RO.iou3d(gt, props)
    assert ov[0, 1] > ov[1, 1] > 0.45
    assert gt_rows.cpu()[inds.cpu() == 1].tolist() == [1]     # the low-quality match
    assert iou.cpu()[inds.cpu() >= 3].abs().max() == 0        # class 2: IoU 0


def test_targets_match_oracle():
    ops = _ops()
    batch = _batch([(500, 150), (400, 120)], seed=11, gt_width=9)
    P = sum(len(b[0]) for b in batch)
    keys = torch.rand(P, generator=torch.Generator().manual_seed(2))
    inds, iou, gt_rows, lab, num_pos, num_rows = _native(batch, _cfg(), keys)
    props = torch.cat([b[0] for b in batch]).to(DEV)
    gt = torch.cat([b[2] for b in batch]).to(DEV)
    soft, reg_mask, bt, pg = ops.roi_head_targets(props[inds], iou, gt_rows, lab, gt, POS_THR, NEG_THR)
    pos = gt_rows >= 0
    assert torch.equal(reg_mask.cpu(), pos.long().cpu())
    assert torch.equal(pg[pos].cpu(), gt[gt_rows[pos], :7].cpu())
    assert (bt[~pos] == 0).all() and (pg[~pos] == 0).all()
    # oracle per sample: positives are the first num_pos rows of each sample
    at = 0
    for b, (npos, n) in enumerate(zip(num_pos, num_rows)):
        rs = slice(at, at + n)
        s_ref, bt_ref = RO.targets(props[inds[rs]].cpu(), iou[rs].cpu().double(), gt[gt_rows[rs][:npos]].cpu(), lab[rs][:npos].cpu(),
                                   POS_THR, NEG_THR)
        assert (soft[rs].cpu().double() - s_ref).abs().max().item() < 1e-6
        err = (bt[rs][:npos].cpu().double() - bt_ref).abs()
        assert (err <= 2e-6 * (1 + bt_ref.abs())).all(), err.max()
        at += n


def _loss_inputs(seed, R=300, npos=80, empty=0.2, car_frac=0.5):
    g = torch.Generator().manual_seed(seed)
    rois = torch.zeros((R, 7))
    rois[:, :2] = torch.randn(R, 2, generator=g) * 20
    rois[:, 2] = torch.randn(R, generator=g) * 0.3
    rois[:, 3:6] = torch.tensor([2.0, 4.5, 1.6]) * (1 + 0.2 * torch.rand(R, 3, generator=g))
    rois[:, 6] = (torch.rand(R, generator=g) * 2 - 1) * math.pi
    gt = rois.clone()
    gt[:, :3] += torch.randn(R, 3, generator=g) * 0.3
    gt[:, 3:6] *= 1 + 0.1 * torch.randn(R, 3, generator=g)
    gt[:, 6] += 0.3 * torch.randn(R, generator=g) + (torch.rand(R, generator=g) < 0.2).float() * math.pi
    lab = torch.where(torch.rand(R, generator=g) < car_frac, 0, torch.randint(1, 3, (R,), generator=g))
    gt_rows = torch.where(torch.arange(R) < npos, torch.arange(R), torch.full((R,), -1))
    lab = torch.where(gt_rows >= 0, lab, torch.full_like(lab, -1))
    iou = torch.rand(R, generator=g)
    nonempty = torch.rand(R, generator=g) >= empty
    cls = torch.randn(R, 1, generator=g) * 2
    pred = torch.randn(R, 7, generator=g) * 0.3
    return rois, gt, gt_rows, lab, iou, nonempty, cls, pred


@pytest.mark.parametrize("case", ["normal", "smoothl1_codeweights", "no_pos", "pos_on_empty", "no_car", "all_empty", "all_car"])
def test_losses_and_grads_match_float64(case):
    ops = _ops()
    npos = {"no_pos": 0}.get(case, 80)
    empty = {"all_empty": 1.0, "pos_on_empty": 0.5}.get(case, 0.2)
    car = {"no_car": 0.0, "all_car": 1.0}.get(case, 0.5)
    rois, gt, gt_rows, lab, iou, nonempty, cls, pred = _loss_inputs(7, npos=npos, empty=empty, car_frac=car)
    if case == "pos_on_empty":
        nonempty[:npos:2] = False
    smooth = case == "smoothl1_codeweights"
    cw = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.5] if smooth else None
    soft, reg_mask, bt, pg = ops.roi_head_targets(rois.to(DEV), iou.to(DEV), gt_rows.to(DEV), lab.to(DEV), gt.to(DEV), POS_THR, NEG_THR)
    x, p = cls.to(DEV).requires_grad_(), pred.to(DEV).requires_grad_()
    ne = nonempty.to(DEV)
    npos_dev = ((reg_mask > 0) & ne).sum().float().reshape(1)
    cfg = ops.RoiLossConfig(1.0, 2.0, smooth, 1.0 / 9.0, True, 0, 1.0, cw)
    R = x.shape[0]
    losses = ops.roi_head_loss(x, p, ne, soft, reg_mask, bt, pg, lab.to(DEV), rois.to(DEV), torch.full((1,), float(R), device=DEV),
                               npos_dev, cfg)
    gw = torch.tensor([1.0, 0.7, 1.3], device=DEV)
    (losses * gw).sum().backward()
    xd, pd = cls.double().requires_grad_(), pred.double().requires_grad_()
    ref = RO.losses(xd, pd, nonempty, soft.cpu(), reg_mask.cpu(), bt.cpu(), pg.cpu(), lab, rois,
                    dict(w_cls=1.0, w_bbox=2.0, smooth_l1=smooth, beta=1.0 / 9.0, code_weights=cw, with_corner=True, corner_class=0,
                         w_corner=1.0))
    rv = torch.stack([ref['loss_rcnn_cls'], ref['loss_rcnn_bbox'], ref['loss_rcnn_corner']])
    (rv * gw.cpu().double()).sum().backward()
    assert torch.allclose(losses.detach().cpu().double(), rv.detach(), rtol=1e-5, atol=1e-7), (losses, rv)
    if case in ("no_pos", "all_empty"):
        assert losses[1].item() == 0 and losses[2].item() == 0 and (p.grad == 0).all()
    if case == "no_car":
        assert losses[2].item() == 0
    assert torch.allclose(x.grad.cpu().double(), xd.grad, rtol=1e-4, atol=1e-7)
    assert torch.allclose(p.grad.cpu().double(), pd.grad, rtol=1e-4, atol=1e-6), (p.grad.cpu().double() - pd.grad).abs().max()


def test_losses_bit_identical_and_no_sync():
    ops = _ops()
    rois, gt, gt_rows, lab, iou, nonempty, cls, pred = _loss_inputs(3, R=2000, npos=700)
    soft, reg_mask, bt, pg = ops.roi_head_targets(rois.to(DEV), iou.to(DEV), gt_rows.to(DEV), lab.to(DEV), gt.to(DEV), POS_THR, NEG_THR)
    cfg = ops.RoiLossConfig(1.0, 2.0, False, 1.0, True, 0, 1.0)
    lab_d, rois_d = lab.to(DEV), rois.to(DEV)
    outs = []
    for _ in range(2):
        x, p = cls.to(DEV).requires_grad_(), pred.to(DEV).requires_grad_()
        ne = nonempty.to(DEV)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            npos_dev = ((reg_mask > 0) & ne).sum().float().reshape(1)
            losses = ops.roi_head_loss(x, p, ne, soft, reg_mask, bt, pg, lab_d, rois_d,
                                       torch.full((1,), 2000.0, device=DEV), npos_dev, cfg)
            losses.sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        outs.append((losses.detach().clone(), x.grad.clone(), p.grad.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_assign_sample_one_sync_and_deterministic():
    batch = _batch([(500, 200), (500, 180)], seed=3)
    keys = torch.rand(1000, generator=torch.Generator().manual_seed(4))
    a = _native(batch, _cfg(), keys)
    b = _native(batch, _cfg(), keys)
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)
    props = torch.cat([p for p, _, _, _ in batch]).to(DEV)
    plab = torch.cat([l for _, l, _, _ in batch]).to(DEV)
    gt = torch.cat([g for _, _, g, _ in batch]).to(DEV)
    gl = torch.cat([l for _, _, _, l in batch]).to(DEV)
    k = keys.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    import warnings
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        _ops().roi_assign_sample(props, plab, [500, 500], k, gt, gl, [200, 180], _cfg())
    torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]


def _head(train=True):
    from sst_b200.roi_head_modules import GroupCorrectionHead
    test_cfg = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=0.25, score_thr=0.1, min_bbox_size=0, max_num=500)
    head = GroupCorrectionHead(num_classes=3, roi_extractor=dict(type='DynamicPointROIExtractor', extra_wlh=[0.5, 0.5, 0.5],
                                                                 max_inbox_point=256, debug=False),
                               bbox_head=MG.small_head(), train_cfg=MG.train_cfg(num=128) if train else None, test_cfg=test_cfg)
    return head.to(DEV)


def _points(batch, per_box=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    xyz, bidx = [], []
    for b, (_, _, gt, _) in enumerate(batch):
        c = gt[:, :3].repeat_interleave(per_box, 0) + torch.randn(len(gt) * per_box, 3, generator=g) * torch.tensor([0.8, 0.8, 0.4])
        c[:, 2] += 0.8
        xyz.append(c)
        bidx.append(torch.full((len(c),), b))
    return torch.cat(xyz).to(DEV), torch.cat(bidx).to(DEV)


def test_training_step():
    """one forward_train-equivalent step + backward + AdamW: the sampling and the loss dict against the oracle, finite gradients"""
    torch.manual_seed(0)
    head = _head().train()
    batch = _batch([(200, 30), (150, 25)], seed=21)
    xyz, bidx = _points(batch)
    feats = torch.randn(len(xyz), 8, device=DEV)
    proposals = [(p.to(DEV), torch.rand(len(p), device=DEV), l.to(DEV)) for p, l, _, _ in batch]
    gts, gls = [b[2].to(DEV) for b in batch], [b[3].to(DEV) for b in batch]
    s = head._assign_and_sample(proposals, gts, gls, generator=torch.Generator(device=DEV).manual_seed(9))
    keys = torch.rand(350, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV).cpu()
    ref = _oracle(batch, keys, num=128)
    assert torch.equal(s.gt_rows.cpu(), torch.cat([r[2] for r in ref]))
    assert s.num_pos == [r[4] for r in ref]
    res = head._bbox_forward_train(xyz, feats, bidx, s)
    losses = res['loss_bbox']
    assert set(losses) == {'loss_rcnn_cls', 'loss_rcnn_bbox', 'loss_rcnn_corner', 'num_pos_rois', 'num_neg_rois'}
    soft, reg_mask, bt, pg = _ops().roi_head_targets(s.bboxes, s.iou, s.gt_rows, s.gt_labels, s.gt_bboxes, POS_THR, NEG_THR)
    ne = res['valid_roi_mask']
    o = RO.losses(res['cls_score'].detach().cpu().double(), res['bbox_pred'].detach().cpu().double(), ne.cpu(), soft.cpu(),
                  reg_mask.cpu(), bt.cpu(), pg.cpu(), s.gt_labels.cpu(), s.bboxes.cpu(),
                  dict(w_cls=1.0, w_bbox=2.0, smooth_l1=False, beta=1.0, code_weights=None, with_corner=True, corner_class=0, w_corner=1.0))
    for k in ('loss_rcnn_cls', 'loss_rcnn_bbox', 'loss_rcnn_corner'):
        assert abs(losses[k].item() - o[k].item()) <= 1e-5 * (1 + abs(o[k].item())), k
    npos = int(((reg_mask > 0) & ne).sum())
    assert losses['num_pos_rois'].item() == npos and losses['num_neg_rois'].item() == len(ne) - npos
    total = losses['loss_rcnn_cls'] + losses['loss_rcnn_bbox'] + losses['loss_rcnn_corner']
    assert torch.isfinite(total) and npos > 0
    opt = torch.optim.AdamW(head.parameters(), lr=1e-3)
    opt.zero_grad()
    total.backward()
    for n, p in head.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    opt.step()


def test_fake_box_for_a_sample_without_proposals():
    """GroupCorrectionHead._assign_and_sample puts the reference's fake box [0, 0, 5, 1, 1, 1, 0] (label 0) in an empty sample"""
    head = _head()
    batch = _batch([(150, 30), (0, 10), (100, 20)], seed=5)
    proposals = [(p.to(DEV), torch.rand(len(p), device=DEV), l.to(DEV)) for p, l, _, _ in batch]
    s = head._assign_and_sample(proposals, [b[2].to(DEV) for b in batch], [b[3].to(DEV) for b in batch],
                                generator=torch.Generator(device=DEV).manual_seed(3))
    keys = torch.rand(251, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV).cpu()
    fake = (torch.tensor([[0, 0, 5, 1, 1, 1, 0]], dtype=torch.float32), torch.tensor([0]), batch[1][2], batch[1][3])
    ref = _oracle([batch[0], fake, batch[2]], keys, num=128)
    assert s.num_rows[1] == 1 and torch.equal(s.bboxes[s.num_rows[0]].cpu(), fake[0][0])
    assert torch.equal(s.gt_rows.cpu(), torch.cat([r[2] for r in ref]))
    assert torch.equal(s.gt_labels.cpu(), torch.cat([r[3] for r in ref]))


def test_golden_targets():
    """tests/golden/roi_head_targets.npz (the reference's own fp32 sampling and targets): sampled rows equal; given the reference's
    IoUs, soft labels bit-equal and box targets within the reference's fp32 rounding"""
    ops = _ops()
    z = np.load(MG.GOLDEN)
    batch = [(torch.from_numpy(z[f"props{b}"]), torch.from_numpy(z[f"plabels{b}"]), torch.from_numpy(z[f"gt{b}"]),
              torch.from_numpy(z[f"gt_labels{b}"])) for b in range(2)]
    keys = torch.cat([torch.from_numpy(z[f"keys{b}"]) for b in range(2)])
    inds, iou, gt_rows, lab, num_pos, num_rows = _native(batch, _cfg(), keys)
    off = [0, len(batch[0][0])]
    goff = [0, len(batch[0][2])]
    assert num_pos == [int(z[f"num_pos{b}"]) for b in range(2)]
    assert torch.equal(inds.cpu(), torch.cat([torch.from_numpy(z[f"inds{b}"]) + off[b] for b in range(2)]))
    ref_iou = torch.cat([torch.from_numpy(z[f"iou{b}"]) for b in range(2)])
    assert (iou.cpu() - ref_iou).abs().max().item() < 1e-5
    pos = gt_rows >= 0
    assert torch.equal(gt_rows[pos].cpu(), torch.cat([torch.from_numpy(z[f"gt_rows{b}"]) + goff[b] for b in range(2)]))
    props = torch.cat([b[0] for b in batch]).to(DEV)
    gt = torch.cat([b[2] for b in batch]).to(DEV)
    soft, reg_mask, bt, pg = ops.roi_head_targets(props[inds], ref_iou.to(DEV), gt_rows, lab, gt, POS_THR, NEG_THR)
    assert torch.equal(soft.cpu(), torch.from_numpy(z["soft_labels"]))
    assert torch.equal(reg_mask.cpu(), torch.from_numpy(z["reg_mask"]))
    assert torch.equal(lab[pos].cpu(), torch.from_numpy(z["pos_gt_labels"]))
    ref_bt = torch.from_numpy(z["bbox_targets"]).double()
    assert ((bt[pos].cpu().double() - ref_bt).abs() <= 2e-6 * (1 + ref_bt.abs())).all()


@pytest.mark.parametrize("rcnn_score_nms", [False, True])
def test_simple_test_matches_oracle(rcnn_score_nms):
    torch.manual_seed(1)
    head = _head(train=False).eval()
    head.test_cfg['rcnn_score_nms'] = rcnn_score_nms
    batch = _batch([(300, 40)], seed=31)
    xyz, bidx = _points(batch)
    feats = torch.randn(len(xyz), 8, device=DEV)
    props, plab = batch[0][0].to(DEV), batch[0][1].to(DEV)
    probs = torch.rand(len(props), device=DEV)
    with torch.no_grad():
        rois = torch.cat([props.new_zeros((len(props), 1)), props], 1)
        res = head._bbox_forward(xyz, feats, bidx, rois)
        out = head.simple_test(xyz, feats, bidx, [{}], [(props, probs.clone(), plab)], None, None)[0]
    boxes, scores, labels = RO.get_bboxes(rois.cpu(), res['cls_score'].cpu(), res['bbox_pred'].cpu(), res['valid_roi_mask'].cpu(),
                                          plab.cpu(), probs.cpu(), 3, 0.1, 0.25, rcnn_score_nms)
    assert out['labels_3d'].device.type == 'cpu' and torch.equal(out['labels_3d'], labels)
    assert torch.allclose(out['boxes_3d'].cpu().double(), boxes, atol=1e-4)
    assert torch.allclose(out['scores_3d'].cpu().double(), scores, atol=1e-6)
    # no proposals: the fake RoI
    with torch.no_grad():
        out = head.simple_test(xyz, feats, bidx, [{}], [(props[:0], probs[:0], plab[:0])], None, None)[0]
    assert out['boxes_3d'].shape[1] == 7
