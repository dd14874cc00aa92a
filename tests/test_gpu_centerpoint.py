"""GPU: CenterHead's native training path (ops.centerpoint_targets, ops.gaussian_focal_loss, ops.centerpoint_l1_loss, CenterHead.loss
and get_bboxes) against the CPU oracle (oracle/centerpoint_oracle.py), on the Waymo CenterHead geometry (1 task x 3 classes, 468^2,
out_size_factor 1, 7-dim boxes) and the reference unit test's (6 tasks, 10 classes, 512^2, out_size_factor 4, 9-dim boxes), each with the
oracle's edge cases, plus the reference's own targets in tests/golden/centerpoint_targets.npz."""
import os

import numpy as np
import pytest
import torch

from oracle import centerpoint_oracle as CO
from oracle import iou3d_oracle as IO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
GEOMS = ("waymo", "nusc")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "centerpoint_targets.npz")
BATCHES = {"edges": [80, 0, 30], "over_max_objs": [700, 45], "single": [200]}


def _native_targets(geom, boxes, labels):
    from sst_b200 import ops
    G = CO.GEOMETRIES[geom]
    cfg = G['train_cfg']
    return ops.centerpoint_targets(torch.cat([CO.gravity(b) for b in boxes]).to(dev), torch.cat(labels).to(dev),
                                   [b.shape[0] for b in boxes], G['tasks'], cfg['point_cloud_range'][:2], cfg['voxel_size'][:2],
                                   cfg['out_size_factor'], CO.feature_map_size(cfg), cfg['gaussian_overlap'], cfg['min_radius'],
                                   cfg['max_objs'] * cfg['dense_reg'])


def _check_targets(name, got, ref):
    hm, ab, ind, mask = (list(x) for x in got)
    rhm, rab, rind, rmask = ref
    for t in range(len(rhm)):
        assert torch.equal(ind[t].cpu(), rind[t]), f"{name} task {t}: ind differs"
        assert torch.equal(mask[t].cpu(), rmask[t]), f"{name} task {t}: mask differs"
        g, r = hm[t].cpu(), rhm[t]
        assert torch.equal(g != 0, r != 0), f"{name} task {t}: heatmap support differs"
        assert torch.equal(g == 1, r == 1), f"{name} task {t}: heatmap centres differ"
        ulp = (g.view(torch.int32).long() - r.view(torch.int32).long()).abs()
        print(f"{name} task {t}: {int((ulp > 0).sum())} of {int((r != 0).sum())} heatmap values differ (by 1 ulp)")
        assert int(ulp.max()) <= 1, f"{name} task {t}: heatmap off by {int(ulp.max())} ulp"
        a = ab[t].cpu()
        assert torch.equal(a[..., [0, 1, 2, 8, 9]], rab[t][..., [0, 1, 2, 8, 9]]), f"{name} task {t}: anno_box offsets / z / velocity differ"
        assert (a[..., 3:8] - rab[t][..., 3:8]).abs().max().item() <= 1e-6, f"{name} task {t}: anno_box log-dims / sin / cos"


@pytest.mark.parametrize("batch", list(BATCHES))
@pytest.mark.parametrize("geom", GEOMS)
def test_targets_match_oracle(geom, batch):
    G = CO.GEOMETRIES[geom]
    boxes, labels = CO.synth_batch(11 + list(BATCHES).index(batch), geom, BATCHES[batch])
    ref = CO.targets([CO.gravity(b) for b in boxes], labels, G['tasks'], G['train_cfg'])
    _check_targets(f"{geom}/{batch}", _native_targets(geom, boxes, labels), ref)


@pytest.mark.parametrize("geom", GEOMS)
def test_targets_match_reference_golden(geom):
    z = np.load(GOLDEN)
    G = CO.GEOMETRIES[geom]
    sizes = z[f"{geom}/sizes"].tolist()
    allb, alll = torch.from_numpy(z[f"{geom}/boxes"]), torch.from_numpy(z[f"{geom}/labels"])
    offs = np.cumsum([0] + sizes)
    boxes = [allb[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    labels = [alll[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    W, H = CO.feature_map_size(G['train_cfg'])
    ref = ([], [], [], [])
    for t, ncls in enumerate(G['tasks']):
        hm = torch.zeros(len(sizes) * ncls * H * W)
        hm[torch.from_numpy(z[f"{geom}/{t}/hm_index"])] = torch.from_numpy(z[f"{geom}/{t}/hm_value"])
        ref[0].append(hm.view(len(sizes), ncls, H, W))
        for i, k in enumerate(("anno_box", "ind", "mask")):
            ref[i + 1].append(torch.from_numpy(z[f"{geom}/{t}/{k}"]))
    _check_targets(f"{geom}/golden", _native_targets(geom, boxes, labels), ref)


def _loss_case(geom, seed, batch=(60, 25)):
    G = CO.GEOMETRIES[geom]
    boxes, labels = CO.synth_batch(seed, geom, list(batch))
    hm, ab, ind, mask = CO.targets([CO.gravity(b) for b in boxes], labels, G['tasks'], G['train_cfg'])
    preds = CO.synth_preds(seed, geom, len(batch))
    return G, hm, ab, ind, mask, preds


def _near_clamp(logits64):
    s = logits64.sigmoid()
    return ((s - 1e-4).abs() <= 1e-6) | ((s - (1 - 1e-4)).abs() <= 1e-6)


@pytest.mark.parametrize("geom", GEOMS)
def test_focal_loss_forward_backward(geom):
    from sst_b200 import ops
    G, hm, _, _, _, preds = _loss_case(geom, 5)
    for t, target in enumerate(hm):
        x = preds[t][0]['heatmap']
        x64 = x.double().requires_grad_(True)
        ref, num_pos = CO.focal_loss(x64, target.double(), 1.0)
        ref.backward()
        xg = x.to(dev).requires_grad_(True)
        loss, npos = ops.gaussian_focal_loss(xg, target.to(dev))
        loss.backward()
        assert npos.item() == num_pos, f"task {t}: num_pos {npos.item()} != {num_pos}"
        err = abs(loss.item() - ref.item()) / abs(ref.item())
        assert err <= 1e-4, f"task {t}: focal loss rel err {err:.2e}"
        # the reference's own fp32 torch composition meets the same bound
        p = CO.clip_sigmoid(x.to(dev))
        tf = target.to(dev)
        comp = (CO.gaussian_focal_loss(p, tf).sum() / max(float(tf.eq(1).sum()), 1)).item()
        assert abs(comp - ref.item()) / abs(ref.item()) <= 1e-4
        keep = ~_near_clamp(x.double())
        gerr = (xg.grad.cpu().double() - x64.grad)[keep].abs().max().item()
        assert gerr <= 1e-4 * x64.grad.abs().max().item(), f"task {t}: focal gradient err {gerr:.2e}"


@pytest.mark.parametrize("geom", GEOMS)
def test_l1_loss_forward_backward(geom):
    from sst_b200 import ops
    G, _, ab, ind, mask, preds = _loss_case(geom, 6)
    cw = G['train_cfg']['code_weights']
    for t in range(len(ab)):
        p = {k: v for k, v in preds[t][0].items() if k != 'heatmap'}
        p64 = {k: v.double().requires_grad_(True) for k, v in p.items()}
        ref = CO.l1_loss(p64, ab[t], ind[t], mask[t], cw, G['loss_bbox_weight'])
        ref.backward()
        pg = {k: v.to(dev).requires_grad_(True) for k, v in p.items()}
        loss = ops.centerpoint_l1_loss(pg, ab[t].to(dev), ind[t].to(dev), mask[t].to(dev), cw, G['loss_bbox_weight'])
        loss.backward()
        err = abs(loss.item() - ref.item()) / abs(ref.item())
        assert err <= 1e-4, f"task {t}: L1 loss rel err {err:.2e}"
        for k in p:
            gerr = (pg[k].grad.cpu().double() - p64[k].grad).abs().max().item()
            assert gerr <= 1e-4 * p64[k].grad.abs().max().item() + 1e-30, f"task {t} {k}: gradient err {gerr:.2e}"


def test_l1_shared_centre_cells_sum_in_slot_order():
    """several objects on one cell: the gradient there is the sum of theirs, and two runs are bit-identical"""
    from sst_b200 import ops
    G = CO.GEOMETRIES["waymo"]
    pc, vs = G['train_cfg']['point_cloud_range'], G['train_cfg']['voxel_size']
    raw = torch.tensor([[pc[0] + (9.1 + 0.1 * k) * vs[0], pc[1] + 9.5 * vs[1], 0.0, 2.0 + k, 4.0, 1.5, 0.3 * k] for k in range(5)] +
                       [[pc[0] + 30.5 * vs[0], pc[1] + 9.5 * vs[1], 0.0, 2.0, 4.0, 1.5, 0.0]])
    labels = torch.tensor([0, 1, 0, 2, 0, 1])
    hm, ab, ind, mask = CO.targets([CO.gravity(raw)], [labels], G['tasks'], G['train_cfg'])
    assert int(mask[0].sum()) == 6 and int(torch.unique(ind[0][mask[0].bool()]).numel()) == 2
    preds = CO.synth_preds(3, "waymo", 1)[0][0]
    p = {k: v for k, v in preds.items() if k != 'heatmap'}
    p64 = {k: v.double().requires_grad_(True) for k, v in p.items()}
    CO.l1_loss(p64, ab[0], ind[0], mask[0], G['train_cfg']['code_weights'], 2.0).backward()
    grads = []
    for _ in range(2):
        pg = {k: v.to(dev).requires_grad_(True) for k, v in p.items()}
        ops.centerpoint_l1_loss(pg, ab[0].to(dev), ind[0].to(dev), mask[0].to(dev), G['train_cfg']['code_weights'], 2.0).backward()
        grads.append({k: v.grad.clone() for k, v in pg.items()})
    for k in p:
        assert torch.equal(grads[0][k], grads[1][k])
        assert (grads[0][k].cpu().double() - p64[k].grad).abs().max().item() <= 1e-6 * p64[k].grad.abs().max().item() + 1e-30


@pytest.mark.parametrize("geom", GEOMS)
def test_center_head_loss_and_backward(geom):
    """CenterHead(**cfg).loss through DCNSeparateHead: losses against the oracle, and the gradient at the head input against the oracle's
    float64 loss gradient pushed back through the same head (relative L2)"""
    import sst_b200  # noqa: F401
    from sst_b200.registry import MODELS
    G = CO.GEOMETRIES[geom]
    torch.manual_seed(0)
    cfg = CO.head_cfg(geom, in_channels=16, share_conv_channel=16, dcn=True)
    head = MODELS.build(cfg).to(dev).train()
    W, H = CO.feature_map_size(G['train_cfg'])
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 16, H, W, generator=g).to(dev).requires_grad_(True)
    raw, labels = CO.synth_batch(8, geom, [60, 25])
    preds = head([x])
    losses = head.loss([b.to(dev) for b in raw], [l.to(dev) for l in labels], preds)
    total = sum(losses.values())
    total.backward(retain_graph=True)
    hm, ab, ind, mask = CO.targets([CO.gravity(b) for b in raw], labels, G['tasks'], G['train_cfg'])
    leaves, ref_total = [], 0.0
    for t, pd in enumerate(preds):
        p64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in pd[0].items()}
        lh, _ = CO.focal_loss(p64['heatmap'], hm[t].double())
        lb = CO.l1_loss(p64, ab[t], ind[t], mask[t], G['train_cfg']['code_weights'], G['loss_bbox_weight'])
        for name, ref in ((f"task{t}.loss_heatmap", lh), (f"task{t}.loss_bbox", lb)):
            err = abs(losses[name].item() - ref.item()) / abs(ref.item())
            assert err <= 1e-4, f"{name}: rel err {err:.2e}"
        ref_total = ref_total + lh + lb
        leaves += [(pd[0][k], p64[k]) for k in p64]
    ref_total.backward()
    gx = torch.autograd.grad([a for a, _ in leaves], x, [b.grad.float().to(dev) for _, b in leaves])[0]
    rel = ((x.grad - gx).norm() / gx.norm()).item()
    assert rel <= 1e-4, f"gradient at the head input: relative L2 {rel:.2e}"


def _run_all(geom, raw, labels, preds):
    """targets + loss forward + backward on device tensors"""
    import sst_b200  # noqa: F401
    from sst_b200.centerhead_modules import CenterHead
    head = CenterHead(**{k: v for k, v in CO.head_cfg(geom).items() if k != 'type'})
    leaves = [{k: v.detach().clone().requires_grad_(True) for k, v in pd.items()} for pd in preds]
    targets = head.get_targets(raw, labels)
    losses = head.loss(raw, labels, [[p] for p in leaves])
    sum(losses.values()).backward()
    return targets, losses, leaves


@pytest.mark.parametrize("geom", GEOMS)
def test_deterministic_and_no_host_sync(geom):
    raw, labels = CO.synth_batch(21, geom, [300, 40])
    raw, labels = [b.to(dev) for b in raw], [l.to(dev) for l in labels]
    preds = [{k: v.to(dev) for k, v in pd[0].items()} for pd in CO.synth_preds(21, geom, 2)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = _run_all(geom, raw, labels, preds)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    b = _run_all(geom, raw, labels, preds)
    for u, v in zip(a[0], b[0]):
        for s, w in zip(u, v):
            assert torch.equal(s, w)
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), k
    for pa, pb in zip(a[2], b[2]):
        for k in pa:
            assert torch.equal(pa[k].grad, pb[k].grad), k


def test_errors():
    from sst_b200 import ops
    from sst_b200._lib import SSTB200Error
    G = CO.GEOMETRIES["waymo"]
    cfg = G['train_cfg']
    boxes = torch.zeros(4, 7)
    labels = torch.zeros(4, dtype=torch.long)
    args = ([4], G['tasks'], cfg['point_cloud_range'][:2], cfg['voxel_size'][:2], 1, (468, 468), 0.1, 2, 500)
    with pytest.raises(SSTB200Error):
        ops.centerpoint_targets(boxes, labels, *args)                                                 # CPU
    with pytest.raises(SSTB200Error):
        ops.centerpoint_targets(boxes.double().to(dev), labels.to(dev), *args)                        # dtype
    with pytest.raises(SSTB200Error):
        ops.centerpoint_targets(torch.zeros(4, 8, device=dev), labels.to(dev), *args)                 # box_dim
    x, t = torch.zeros(2, 3, 8, 8), torch.zeros(2, 3, 8, 8)
    with pytest.raises(SSTB200Error):
        ops.gaussian_focal_loss(x, t)                                                                 # CPU
    with pytest.raises(SSTB200Error):
        ops.gaussian_focal_loss(x.double().to(dev), t.double().to(dev))                               # dtype
    with pytest.raises(SSTB200Error):
        ops.gaussian_focal_loss(x.to(dev), torch.zeros(2, 3, 8, 9, device=dev))                       # shape
    p = {k: torch.zeros(2, c, 8, 8, device=dev) for k, c in ops.CENTERPOINT_HEADS}
    ab, ind, mask = torch.zeros(2, 5, 10, device=dev), torch.zeros(2, 5, dtype=torch.long, device=dev), torch.zeros(2, 5, dtype=torch.uint8,
                                                                                                                    device=dev)
    ops.centerpoint_l1_loss(p, ab, ind, mask, [1.0] * 10)
    with pytest.raises(SSTB200Error):
        ops.centerpoint_l1_loss(dict(p, dim=torch.zeros(2, 3, 8, 9, device=dev)), ab, ind, mask, [1.0] * 10)   # head / map sizes
    with pytest.raises(SSTB200Error):
        ops.centerpoint_l1_loss({k: v.cpu() for k, v in p.items()}, ab, ind, mask, [1.0] * 10)                # CPU
    with pytest.raises(SSTB200Error):
        ops.centerpoint_l1_loss(p, ab[:, :4], ind, mask, [1.0] * 10)                                          # anno_box / ind
    h = torch.zeros(2, 3, 8, 8, device=dev)
    with pytest.raises(SSTB200Error):
        ops.gaussian_focal_loss(h, torch.zeros(2, 3, 8, 8, dtype=torch.int32, device=dev))


def _sparse_preds(seed, geom, batch, n):
    """heatmap logits -12 except at n well-separated cells per sample with distinct logits; small boxes there, a few of them overlapping"""
    G = CO.GEOMETRIES[geom]
    W, H = CO.feature_map_size(G['train_cfg'])
    g = torch.Generator().manual_seed(seed)
    preds = CO.synth_preds(seed, geom, batch, scale=0.3)
    logit = 0.0
    for pd in preds:
        p = pd[0]
        p['heatmap'].fill_(-12.0)
        p['dim'] = torch.randn(p['dim'].shape, generator=g) * 0.2 - 1.0
        for b in range(batch):
            cells = torch.randperm((H // 4) * (W // 4), generator=g)[:n]
            for k, cell in enumerate(cells.tolist()):
                y, x = 4 * (cell // (W // 4)), 4 * (cell % (W // 4))
                c = k % p['heatmap'].shape[1]
                logit += 1e-3
                p['heatmap'][b, c, y, x] = -1.5 + logit
                if k % 5 == 0:                                    # a neighbour on the next cell: an overlapping box
                    logit += 1e-3
                    p['heatmap'][b, c, y, min(x + 1, W - 1)] = -1.5 + logit
    return preds


@pytest.mark.parametrize("geom", GEOMS)
def test_get_bboxes_matches_oracle(geom):
    import sst_b200  # noqa: F401
    from sst_b200.centerhead_modules import CenterHead
    G = CO.GEOMETRIES[geom]
    cfg = CO.head_cfg(geom)
    preds = _sparse_preds(31, geom, 2, 60)
    ref = CO.get_bboxes(preds, G['tasks'], G['bbox_coder'], G['test_cfg'])
    # the comparison is well-defined: no BEV IoU among a task's candidates lies within 1e-4 of nms_thr
    for pd in preds:
        for c in CO.decode(pd[0]['heatmap'].sigmoid(), pd[0]['rot'][:, 0:1], pd[0]['rot'][:, 1:2], pd[0]['height'], pd[0]['dim'].exp(),
                           pd[0]['vel'], pd[0]['reg'], G['bbox_coder']):
            keep = c['scores'] >= G['test_cfg']['score_threshold']
            bev = CO.bev_xyxyr(c['bboxes'][keep])
            assert IO.drop_near_threshold(bev, [G['test_cfg']['nms_thr']]).numel() == bev.shape[0]
    head = CenterHead(**{k: v for k, v in cfg.items() if k != 'type'})
    got = head.get_bboxes([[{k: v.to(dev) for k, v in pd[0].items()}] for pd in preds], [dict() for _ in range(2)])
    for (gb, gs, gl), (rb, rs, rl) in zip(got, ref):
        assert gb.shape == rb.shape and rb.shape[0] > 0
        assert torch.equal(gl.cpu(), rl)
        assert (gs.cpu() - rs).abs().max().item() <= 1e-6
        assert (gb.cpu() - rb).abs().max().item() <= 1e-4
    head.test_cfg = dict(head.test_cfg, nms_type='circle')
    with pytest.raises(NotImplementedError):
        head.get_bboxes([[{k: v.to(dev) for k, v in pd[0].items()}] for pd in preds], None)
