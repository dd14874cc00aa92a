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
