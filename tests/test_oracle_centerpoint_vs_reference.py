"""CPU: the CenterHead oracle (oracle/centerpoint_oracle.py) against the reference's own CenterHead (centerpoint_head.py, imported unmodified
through oracle/centerpoint_ref.py): targets bit-identical on the edge-case batches of both geometries, losses within 1e-12 relative in
float64, decode equal on distinct scores; sst_b200's CenterHead has the reference's state-dict layout and builds from both CenterHead
configs' bbox_head dicts."""
import copy

import pytest
import torch

from oracle import centerpoint_oracle as CO
from oracle import centerpoint_ref as CR

GEOMS = ("waymo", "nusc")
BATCHES = ([80, 0, 30], [700, 45], [200])


def _ref():
    if not CR.available():
        pytest.skip("reference tree not present")
    return CR.load_center_head()


@pytest.mark.parametrize("sizes", BATCHES, ids=lambda s: "-".join(map(str, s)))
@pytest.mark.parametrize("geom", GEOMS)
def test_oracle_targets_bit_identical_to_reference(geom, sizes):
    R = _ref()
    G = CO.GEOMETRIES[geom]
    boxes, labels = CO.synth_batch(11 + BATCHES.index(sizes), geom, sizes)
    ref = CR.build_center_head(CO.head_cfg(geom)).get_targets([R.Boxes(b) for b in boxes], labels)
    got = CO.targets([CO.gravity(b) for b in boxes], labels, G['tasks'], G['train_cfg'])
    for i, name in enumerate(("heatmap", "anno_box", "ind", "mask")):
        for t, (a, b) in enumerate(zip(ref[i], got[i])):
            assert a.dtype == b.dtype and a.shape == b.shape, (name, t)
            assert torch.equal(a, b), f"{name} of task {t} differs in {int((a != b).sum())} elements"


# non-square maps, and an out_size_factor of 2 with 9-dim boxes and two tasks: the shapes tests/test_gpu_centerpoint_edges.py builds on
NONSQUARE = {"200x136": dict(width=200, height=136),
             "osf2_256x176": dict(width=256, height=176, out_size_factor=2, voxel_size=(0.2, 0.2), tasks=(1, 2), box_dim=9)}


@pytest.mark.parametrize("name", list(NONSQUARE))
def test_oracle_targets_bit_identical_to_reference_nonsquare(name):
    R = _ref()
    G = CO.geometry(**NONSQUARE[name])
    W, H = CO.feature_map_size(G['train_cfg'])
    assert W != H
    boxes, labels = CO.synth_batch(17, G, [400, 0, 50])
    ref = CR.build_center_head(CO.head_cfg(G)).get_targets([R.Boxes(b) for b in boxes], labels)
    got = CO.targets([CO.gravity(b) for b in boxes], labels, G['tasks'], G['train_cfg'])
    for i, name in enumerate(("heatmap", "anno_box", "ind", "mask")):
        for t, (a, b) in enumerate(zip(ref[i], got[i])):
            assert a.dtype == b.dtype and a.shape == b.shape, (name, t)
            assert torch.equal(a, b), f"{name} of task {t} differs in {int((a != b).sum())} elements"
    assert ref[0][0].shape[-2:] == (H, W)


def test_edge_cases_are_exercised():
    """the synthetic batches hold what the targets' semantics hinge on"""
    G = CO.GEOMETRIES["waymo"]
    cfg = G['train_cfg']
    boxes, labels = CO.synth_batch(11, "waymo", [80])
    gb = CO.gravity(boxes[0])
    vs = torch.tensor(cfg['voxel_size'])
    cx = (gb[:, 0] - torch.tensor(cfg['point_cloud_range'])[0]) / vs[0]
    assert ((cx > -1) & (cx < 0)).any() and (cx < -1).any() and (cx >= 468).any()
    assert (gb[:, 3] <= 0).any() and (gb[:, 4] <= 0).any()
    assert (labels[0] >= 3).any()
    r = CO.gaussian_radius(gb[:, 4] / vs[1], gb[:, 3] / vs[0], 0.1)
    assert (r > 468).any()
    frac = (r - r.round()).abs()
    assert ((frac > 0) & (frac <= r.abs() * 2.4e-7)).sum() >= 2, "no radius within an ulp of an integer"
    _, _, ind, mask = CO.targets([gb], labels, G['tasks'], cfg)
    cells = ind[0][mask[0].bool()]
    assert cells.numel() > torch.unique(cells).numel(), "no shared centre cell"
    assert (mask[0].bool() & (ind[0] == 0)).any() or (cells % 468 == 0).any()


@pytest.mark.parametrize("geom", GEOMS)
def test_oracle_losses_match_reference(geom):
    R = _ref()
    G = CO.GEOMETRIES[geom]
    boxes, labels = CO.synth_batch(5, geom, [60, 25])
    head = CR.build_center_head(CO.head_cfg(geom)).double()
    preds = CO.synth_preds(5, geom, 2)
    ref_preds = [[{k: v.double() for k, v in pd[0].items()}] for pd in preds]
    ref = head.loss([R.Boxes(b) for b in boxes], labels, ref_preds)
    hm, ab, ind, mask = CO.targets([CO.gravity(b) for b in boxes], labels, G['tasks'], G['train_cfg'])
    for t, pd in enumerate(preds):
        p = {k: v.double() for k, v in pd[0].items()}
        lh, _ = CO.focal_loss(p['heatmap'], hm[t])     # the fp32 target, as the reference's loss() receives it
        lb = CO.l1_loss(p, ab[t], ind[t], mask[t], G['train_cfg']['code_weights'], G['loss_bbox_weight'])
        for name, got in ((f"task{t}.loss_heatmap", lh), (f"task{t}.loss_bbox", lb)):
            r = ref[name]
            assert abs(got.item() - r.item()) <= 1e-12 * abs(r.item()), name


@pytest.mark.parametrize("geom", GEOMS)
def test_oracle_decode_matches_reference(geom):
    R = _ref()
    G = CO.GEOMETRIES[geom]
    head = CR.build_center_head(CO.head_cfg(geom))
    g = torch.Generator().manual_seed(9)
    preds = CO.synth_preds(9, geom, 2, scale=0.3)
    for pd in preds:        # distinct scores; small boxes
        p = pd[0]
        p['heatmap'] = (torch.randperm(p['heatmap'].numel(), generator=g).float() / p['heatmap'].numel() * 8 - 6).view(p['heatmap'].shape)
        p['dim'] = p['dim'] * 0.2 - 1.5
    metas = [dict(box_type_3d=R.Boxes) for _ in range(2)]
    ref = head.get_bboxes(copy.deepcopy(preds), metas)
    got = CO.get_bboxes(preds, G['tasks'], G['bbox_coder'], G['test_cfg'])
    for (rb, rs, rl), (gb, gs, gl) in zip(ref, got):
        assert torch.equal(rb.tensor, gb) and torch.equal(rs, gs) and torch.equal(rl, gl)
        assert gb.shape[0] > 0


def test_state_dict_layout_matches_reference():
    _ref()
    import sst_b200  # noqa: F401
    from sst_b200.registry import MODELS
    for geom in GEOMS:
        for dcn in (False, True):
            cfg = CO.head_cfg(geom, in_channels=32, share_conv_channel=16, dcn=dcn)
            ref = CR.build_center_head(copy.deepcopy(cfg))
            ours = MODELS.build(copy.deepcopy(cfg))
            a = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
            b = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
            assert list(a) == list(b) and a == b
            assert any(k.startswith("shared_conv.conv.") for k in b) and any(k.startswith("shared_conv.bn.") for k in b)


# configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py:84-140 (sst_waymoD1_2x_3class_centerhead.py inherits it unchanged)
WAYMO_BBOX_HEAD = dict(
    type='CenterHead', _delete_=True, in_channels=128, tasks=[dict(num_class=3, class_names=['car', 'pedestrian', 'cyclist'])],
    common_heads=dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)), share_conv_channel=64,
    bbox_coder=dict(type='CenterPointBBoxCoder', post_center_range=[-74.88, -74.88, -10.0, 74.88, 74.88, 10.0], max_num=4096,
                    score_threshold=0.1, out_size_factor=1, voxel_size=(0.32, 0.32), pc_range=[-74.88, -74.88], code_size=9),
    separate_head=dict(type='DCNSeparateHead', init_bias=-2.19, final_kernel=3,
                       dcn_config=dict(type='DCN', in_channels=64, out_channels=64, kernel_size=3, padding=1, groups=4, bias=False),
                       norm_cfg=dict(type='naiveSyncBN2d', eps=1e-3, momentum=0.01)),
    norm_cfg=dict(type='naiveSyncBN2d', eps=1e-3, momentum=0.01), loss_cls=dict(type='GaussianFocalLoss', reduction='mean'),
    loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=2), norm_bbox=True)


def _config_bbox_head(name):
    """the bbox_head dict of a CenterHead config, with the model's train_cfg / test_cfg as the detector passes them"""
    import os
    from oracle.ref_shim import REF_ROOT
    path = os.path.join(REF_ROOT, "configs/sst_refactor", name)
    if not os.path.exists(path):
        return dict(WAYMO_BBOX_HEAD, train_cfg=CO.WAYMO['train_cfg'], test_cfg=CO.WAYMO['test_cfg'])
    while True:
        g = {}
        exec(compile(open(path).read(), path, "exec"), g)
        if "model" in g:
            m = g["model"]
            return dict(m["bbox_head"], train_cfg=m["train_cfg"], test_cfg=m["test_cfg"])
        path = os.path.join(os.path.dirname(path), g["_base_"][0] if isinstance(g["_base_"], list) else g["_base_"])


@pytest.mark.parametrize("config", ["sst_waymoD5_1x_3class_centerhead.py", "sst_waymoD1_2x_3class_centerhead.py"])
def test_center_head_builds_from_configs(config):
    import sst_b200  # noqa: F401
    from sst_b200.registry import MODELS
    cfg = _config_bbox_head(config)
    cfg.pop("_delete_", None)
    head = MODELS.build(cfg)
    assert type(head).__name__ == "CenterHead" and len(head.task_heads) == 1
    assert type(head.task_heads[0]).__name__ == "DCNSeparateHead"
    assert head.loss_bbox_weight == 2.0 and head.train_cfg['max_objs'] == 500
    with pytest.raises(ValueError):
        MODELS.build(dict(cfg, loss_bbox=dict(type='L1Loss', reduction='none', loss_weight=0.25)))
    with pytest.raises(ValueError):
        MODELS.build(dict(cfg, loss_cls=dict(type='FocalLoss', reduction='mean')))
