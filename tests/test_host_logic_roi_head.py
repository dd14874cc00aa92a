"""CPU: GroupCorrectionHead / FullySparseBboxHead refuse the settings no FSD config uses (ValueError), and build the reference's
state-dict keys for the FSD Waymo D1 head."""
import pytest

ASSIGNER = dict(type='MaxIoUAssigner', iou_calculator=dict(type='BboxOverlaps3D', coordinate='lidar'), pos_iou_thr=0.45,
                neg_iou_thr=0.45, min_pos_iou=0.45, ignore_iof_thr=-1)
SAMPLER = dict(type='IoUNegPiecewiseSampler', num=256, pos_fraction=0.55, neg_piece_fractions=[0.8, 0.2], neg_iou_piece_thrs=[0.55, 0.1],
               neg_pos_ub=-1, add_gt_as_proposals=False, return_iou=True)
BBOX_HEAD = dict(type='FullySparseBboxHead', num_classes=3, num_blocks=6, in_channels=[213, 146, 146, 146, 146, 146],
                 feat_channels=[[128, 128]] * 6, rel_mlp_hidden_dims=[[16, 32]] * 6, rel_mlp_in_channels=[13] * 6, reg_mlp=[512, 512],
                 cls_mlp=[512, 512], mode='max', xyz_normalizer=[20, 20, 4], act='gelu', geo_input=True, with_corner_loss=True,
                 corner_loss_weight=1.0, bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'), norm_cfg=dict(type='LN', eps=1e-3),
                 unique_once=True, loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=2.0),
                 loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='mean', loss_weight=1.0), cls_dropout=0.1,
                 reg_dropout=0.1)


def _build(bbox_head=None, assigner=None, sampler=None, extra=None):
    from sst_b200.roi_head_modules import GroupCorrectionHead
    train_cfg = dict(assigner=[dict(ASSIGNER, **(assigner or {}))] * 3, sampler=dict(SAMPLER, **(sampler or {})),
                     cls_pos_thr=(0.8, 0.65, 0.65), cls_neg_thr=(0.2, 0.15, 0.15), class_names=['Car', 'Pedestrian', 'Cyclist'],
                     **(extra or {}))
    return GroupCorrectionHead(num_classes=3, roi_extractor=dict(type='DynamicPointROIExtractor', extra_wlh=[0.5, 0.5, 0.5],
                                                                 max_inbox_point=256, debug=False),
                               bbox_head=dict(BBOX_HEAD, **(bbox_head or {})), train_cfg=train_cfg, test_cfg=None)


def test_fsd_head_builds_with_reference_keys():
    sd = _build().state_dict()
    assert 'bbox_head.block_list.5.vfe_layers.1.linear.weight' in sd
    assert 'bbox_head.conv_cls.2.weight' in sd and sd['bbox_head.conv_cls.2.weight'].shape == (1, 512)
    assert sd['bbox_head.conv_reg.2.weight'].shape == (7, 512)
    assert sd['bbox_head.conv_cls.0.0.weight'].shape == (512, 6 * 256)


@pytest.mark.parametrize("kw", [
    dict(sampler=dict(add_gt_as_proposals=True)),
    dict(sampler=dict(neg_pos_ub=3)),
    dict(sampler=dict(type='RandomSampler')),
    dict(sampler=dict(neg_piece_fractions=[0.8, 0.5, 0.1], neg_iou_piece_thrs=[0.55, 0.3, 0.1])),
    dict(sampler=dict(neg_iou_piece_thrs=[0.1, 0.55])),
    dict(assigner=dict(gt_max_assign_all=False)),
    dict(assigner=dict(match_low_quality=False)),
    dict(assigner=dict(ignore_iof_thr=0.5)),
    dict(bbox_head=dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True))),
    dict(bbox_head=dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False))),
    dict(bbox_head=dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='none'))),
    dict(bbox_head=dict(loss_bbox=dict(type='IoULoss'))),
    dict(extra=dict(class_wise_cls_weights=[1, 2, 2])),
])
def test_refusals(kw):
    with pytest.raises(ValueError):
        _build(**kw)


def _rows(n_neg, num, fractions, thrs, seed, npos=0):
    """the oracle sampler's row count for one sample: npos positives and n_neg negatives with IoUs drawn over [0, 0.6)"""
    import torch
    from oracle import roi_head_oracle as RO
    g = torch.Generator().manual_seed(seed)
    gi = torch.cat([torch.ones(npos, dtype=torch.int64), torch.zeros(n_neg, dtype=torch.int64)])
    mo = torch.cat([torch.full((npos,), 0.9, dtype=torch.float64), torch.rand(n_neg, generator=g, dtype=torch.float64) * 0.6])
    # quantised IoUs leave some pieces empty, so the carry-over runs
    mo = torch.where(torch.rand(len(mo), generator=g) < 0.5, (mo * 4).floor() / 4, mo)
    p, n = RO.sample(gi, mo, torch.rand(len(gi), generator=g), num, 0.5, fractions, thrs)
    return len(p) + len(n)


def test_oracle_sampler_never_exceeds_num_with_three_pieces():
    """with 1 to 3 pieces, fractions >= 0 and a non-last sum <= 1, the reference's carry-over keeps every sample within num rows (the
    bound the native sampler's output layout relies on)"""
    import random
    rng = random.Random(0)
    for t in range(300):
        k = rng.choice([1, 2, 3])
        head = [rng.random() for _ in range(k - 1)]
        if sum(head) > 1:
            head = [h / sum(head) for h in head]
        fr = head + [rng.random()]
        thrs = sorted((rng.random() * 0.6 for _ in range(k)), reverse=True)
        num = rng.choice([1, 7, 64, 100, 256])
        rows = _rows(rng.choice([0, 5, 150, 600]), num, fr, thrs, t, npos=rng.choice([0, 3, 40]))
        assert rows <= num, (fr, thrs, num, rows)


def test_oracle_sampler_exceeds_num_with_four_pieces():
    """the example the refusal guards against: pieces 0 and 1 empty, the carry-over doubles and piece 2 is asked for 120 of 100 rows"""
    import torch
    from oracle import roi_head_oracle as RO
    N = 200
    p, n = RO.sample(torch.zeros(N, dtype=torch.int64), torch.full((N,), 0.25, dtype=torch.float64), torch.rand(N), 100, 0.55,
                     [0.3, 0.3, 0.3, 0.1], [0.55, 0.45, 0.3, 0.1])
    assert len(p) + len(n) == 120


@pytest.mark.parametrize("fr,th", [
    ([0.3, 0.3, 0.3, 0.1], [0.55, 0.45, 0.3, 0.1]),     # four pieces
    ([0.5, -0.1, 0.6], [0.55, 0.3, 0.1]),               # a negative fraction
    ([0.7, 0.4, 0.1], [0.55, 0.3, 0.1]),                # non-last fractions summing past 1
])
def test_refuses_piece_settings_that_could_overflow(fr, th):
    with pytest.raises(ValueError):
        _build(sampler=dict(neg_piece_fractions=fr, neg_iou_piece_thrs=th))


@pytest.mark.parametrize("fr,th", [([1.0], [0.55]), ([0.8, 0.2], [0.55, 0.1]), ([0.5, 0.5, 0.2], [0.55, 0.3, 0.1])])
def test_accepts_one_to_three_pieces(fr, th):
    assert _build(sampler=dict(neg_piece_fractions=fr, neg_iou_piece_thrs=th)).sample_cfg.struct.num_pieces == len(fr)
