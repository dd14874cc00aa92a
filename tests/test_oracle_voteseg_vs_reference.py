"""CPU: oracle/voteseg_oracle.py against the reference's own VoteSegHead (segmentation_head.py and decode_head.py, imported unmodified
through oracle/voteseg_ref.py): targets identical to get_targets, float64 losses and gradients within 1e-12 relative of `losses`, the
training-log metrics identical; the golden file equal to the reference; and sst_b200's VoteSegHead with the reference's state-dict keys
and shapes for every configs/fsd* and configs/fsdv2* file."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_voteseg as MG
from oracle import voteseg_oracle as VO
from oracle import voteseg_ref as VR

pytestmark = pytest.mark.skipif(not VR.available(), reason="reference tree not present")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES, head_cfg, loss_kwargs = VO.LOSS_MODES, VO.head_cfg, VO.loss_kwargs


def frame(mode, seed, n_points=(1500, 0, 900), n_boxes=(30, 4, 0)):
    """points / boxes / labels of a batch and the reference's targets, and logits / vote predictions clear of the log thresholds"""
    R = VR.load_voteseg_head()
    m = MODES[mode]
    P, B, L = VO.synth_batch(seed, list(n_points), list(n_boxes), m["num_classes"])
    head = VR.build_voteseg_head(head_cfg(mode), m["train_cfg"])
    t = head.get_targets(P, [R.Boxes(b) for b in B], L)
    C = head.num_classes
    x, v = VO.synth_preds(seed, t[0].shape[0], C, scale=4.0)
    x = VO.clear_of_thresholds(x, loss_kwargs(mode), seed=seed)
    return head, (P, B, L), t, x, v


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_targets_identical_to_reference(seed):
    R = VR.load_voteseg_head()
    for num_classes in (1, 3, 10):
        P, B, L = VO.synth_batch(seed * 10 + num_classes, [1200, 0, 700, 300], [25, 6, 0, 9], num_classes)
        P[3] = torch.cat([P[3], torch.nn.functional.pad(VO.face_points(B[3]), (0, 2))])
        B[0][3] = B[0][2]                       # an invalid-label copy of a valid box, lower index
        L[0][2], L[0][3] = -1, min(1, num_classes - 1)
        head = VR.build_voteseg_head(dict(in_channel=8, num_classes=num_classes, loss_decode=dict(type="CrossEntropyLoss"),
                                          loss_vote=dict(type="L1Loss")))
        ref = head.get_targets(P, [R.Boxes(b) for b in B], L)
        got = VO.targets(P, B, L, num_classes)
        _same_targets(ref, got)
        assert ref[2].any() and not ref[2].all()


def _same_targets(ref, got):
    """labels and mask identical; vote targets identical up to the square root, which the reference run on the CPU takes from torch's
    vectorised kernel (within one ulp of the correctly rounded root the GPU gives, and the oracle restates)"""
    for a, b in zip(ref, got):
        assert a.dtype == b.dtype and a.shape == b.shape
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[2], got[2])
    assert (ref[1].view(torch.int32).long() - got[1].view(torch.int32).long()).abs().max().item() <= 1
    assert torch.equal(torch.sign(ref[1]), torch.sign(got[1]))


def test_golden_file_is_the_reference():
    g = np.load(os.path.join(ROOT, "tests", "golden", "voteseg_targets.npz"))
    R = VR.load_voteseg_head()
    for name in MG.CASES:
        num_classes, P, B, L = MG.case(name)
        head = VR.build_voteseg_head(dict(in_channel=8, num_classes=num_classes, loss_decode=dict(type="CrossEntropyLoss"),
                                          loss_vote=dict(type="L1Loss")))
        ref = head.get_targets(P, [R.Boxes(b) for b in B], L)
        assert np.array_equal(g[f"{name}/points"], torch.cat(P).numpy())
        for k, key in enumerate(("labels_t", "vote_targets", "vote_mask")):
            assert np.array_equal(g[f"{name}/{key}"], ref[k].numpy()), (name, key)


@pytest.mark.parametrize("mode", list(MODES))
def test_oracle_losses_and_gradients_match_reference(mode):
    head, _, t, x, v = frame(mode, sum(map(ord, mode)))
    x64, v64 = x.double().requires_grad_(True), v.double().requires_grad_(True)
    ref = head.losses(x64, v64, *t)
    (ref["loss_sem_seg"] + 0.7 * ref["loss_vote"]).backward()
    xo, vo = x.double().requires_grad_(True), v.double().requires_grad_(True)
    seg, vote = VO.losses(xo, vo, *t, **loss_kwargs(mode))
    (seg + 0.7 * vote).backward()
    for a, b in ((seg, ref["loss_sem_seg"]), (vote, ref["loss_vote"])):
        assert abs(a.item() - b.item()) <= 1e-12 * abs(b.item())
    for a, b in ((xo.grad, x64.grad), (vo.grad, v64.grad)):
        assert (a - b).abs().max().item() <= 1e-12 * b.abs().max().item()


@pytest.mark.parametrize("mode", list(MODES))
def test_oracle_metrics_identical_to_reference(mode):
    head, _, t, x, v = frame(mode, 7 + sum(map(ord, mode)))
    ref = head.losses(x, v, *t)
    got = VO.metrics(x, t[0], **loss_kwargs(mode))
    keys = [k for k in ref if k.startswith("recall_") or k == "num_fg"]
    assert keys == list(got)
    for k in keys:
        assert torch.equal(ref[k].float(), got[k].float()), k


def test_oracle_no_valid_point_matches_reference():
    head, _, t, x, v = frame("waymo_focal", 3)
    labels = torch.full_like(t[0], 3)
    mask = torch.zeros_like(t[2])
    for bad in (None, float("nan"), float("inf")):
        vv = v.double().clone()
        if bad is not None:
            vv[5, 4] = bad
        vv.requires_grad_(True)
        ref = head.losses(x.double(), vv, labels, t[1], mask)["loss_vote"]
        got = VO.losses(x.double(), vv, labels, t[1], mask, **loss_kwargs("waymo_focal"))[1]
        assert (ref.isnan().item() and got.isnan().item()) or ref.item() == got.item() == 0.0


def _find_heads(d, out):
    if isinstance(d, dict):
        if d.get("type") == "VoteSegHead":
            out.append(d)
        for v in d.values():
            _find_heads(v, out)
    elif isinstance(d, (list, tuple)):
        for v in d:
            _find_heads(v, out)
    return out


def test_state_dict_keys_and_shapes_match_reference_for_every_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    from sst_b200.registry import MODELS
    seen = 0
    paths = sorted(glob.glob(os.path.join(REF_ROOT, "configs", "fsd", "*.py")) + glob.glob(os.path.join(REF_ROOT, "configs", "fsdv2", "*.py")))
    assert len(paths) == 11
    for path in paths:
        m = Config.fromfile(path)["model"]
        heads = _find_heads(m, [])
        assert heads, path
        for cfg in heads:
            ref = VR.build_voteseg_head(cfg)
            mine = MODELS.build(cfg)
            assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, path
            mine.load_state_dict(ref.state_dict())
            _same_forward(ref, mine, cfg)
            seen += 1
    assert seen >= 11


def _same_forward(ref, mine, cfg):
    """the reference head and this one, same weights, give the same logits and vote predictions in train and eval mode"""
    feats = torch.randn((300, cfg["in_channel"]), generator=torch.Generator().manual_seed(cfg["in_channel"]))
    for train in (True, False):
        ref.train(train), mine.train(train)
        with torch.no_grad():
            for a, b in zip(ref.forward(feats), mine.forward(feats)):
                assert a.shape == b.shape and torch.allclose(a, b, rtol=1e-6, atol=1e-6)


def test_training_segmentor_dict_is_the_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    cfg = Config.fromfile(os.path.join(REF_ROOT, "configs", "fsd", "fsd_waymoD1_1x.py"))
    assert _plain(cfg["segmentor"]) == _plain(VO.FSD_D1_SEGMENTOR)


def _plain(d):
    if isinstance(d, dict):
        return {k: _plain(v) for k, v in d.items()}
    if isinstance(d, (list, tuple)):
        return [_plain(v) for v in d]
    return d


def test_refused_settings_raise():
    from sst_b200.voteseg_modules import VoteSegHead
    base = head_cfg("waymo_focal")
    base.pop("type")
    bad = [dict(loss_aux=dict(type="LovaszLoss")), dict(loss_decode=dict(type="FocalLoss", use_sigmoid=True, gamma=0.5)),
           dict(loss_decode=dict(type="FocalLoss", use_sigmoid=False)), dict(loss_decode=dict(type="LovaszLoss")),
           dict(loss_decode=dict(type="FocalLoss", gamma=2.0, alpha=0.25)),   # use_sigmoid missing: the head would read it as False
           dict(loss_decode=dict(type="CrossEntropyLoss", use_sigmoid=True)), dict(loss_vote=dict(type="SmoothL1Loss"))]
    for kw in bad:
        with pytest.raises(ValueError):
            VoteSegHead(**dict(base, **kw))
    head = VoteSegHead(**base)
    for cfg in (dict(centroid_offset=True), dict(extra_width=0.1)):
        with pytest.raises(ValueError):
            head.train_cfg = cfg
    head.train_cfg = dict(centroid_offset=False, score_thresh=(0.3, 0.25, 0.25), class_names=("Car", "Ped", "Cyc"))
