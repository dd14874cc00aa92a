"""GPU: FSD's second stage (sst_b200/csrc/roi_head.cu) against oracle/roi_head_oracle.py at the edges where its three kernel groups could
go wrong: the 3-D IoU, the assignment and sampling (rs_assign_sample_kernel), the targets (rs_targets_kernel) and the losses (rl_*).

Routes and edges
  IoU        B samples of one GT each, one assigner, pos = neg, num >= P and pos_fraction 1, so every proposal comes back with its IoU to
             its sample's GT: rotated boxes near the origin and 75 m away, sub-metre boxes, identical boxes, z ranges that touch, nest or
             are disjoint, zero width, length or height (exactly 0, never NaN), proposal widths 7 / 9 and GT widths 7 / 9 / 10.
  thresholds yaw-0 boxes with dyadic corners, whose kernel IoU RO.iou3d_fp32_axis reproduces bit for bit; the proposal height is swept
             over consecutive fp32 values until the IoU is fl32(t) and one ulp either side, for pos (0.45 and 0.35, which fl32 rounds
             down), neg, min_pos and both piece bounds (0.55 and 0.1, which fl32 rounds up).  The expected rows come from the oracle fed
             the fp32 IoUs and fp32-rounded thresholds, so that every compare is the kernel's fp32 compare, as torch makes it.  The soft
             label's `>` / `!<` at fl32(0.8, 0.65, 0.2, 0.15) and one ulp either side, bit for bit.
  routes     exact rows against RO.assign_and_sample on dyadic boxes through the C ABI, output rows pre-filled with a sentinel (rows
             below each count written, rows from the count up to num untouched): proposals per sample 1, 31, 32, 33, 511, 512, 513,
             1024, 1025, 4096 (4097 refused); GTs 0, 1, 511, 512, 513, 4096 (4097 refused); B = 1 and B = 40 of mixed sizes with
             1-proposal and GT-free samples; the ignore band, min_pos < pos, min_pos = 0, pos_fraction 0 and 1, 1, 2 and 3 pieces with
             the carry-over, the nneg <= nexp path, a piece with exactly `want` members, keys quantised to four values, duplicate GTs and
             proposals, proposal labels -1 and K with per_class on and off.
  low-qual   rotated, overlapping GT crowds 70 m out with min_pos < pos: the low-quality pass recomputes each IoU and compares it with
             the per-GT maximum with ==, so both computations must agree bit for bit; hundreds of proposals are re-targeted or promoted.
  refusals   4 IoU pieces, a negative fraction and non-last fractions past 1 (benign inputs: fewer negatives than num).
  targets    R = 1, 255, 256, 257 and 70001; roi and GT yaws -2 pi, -pi, 0, pi, 2 pi and their fp32 neighbours; relative yaws at
             pi / 2 and 3 pi / 2 +- k ulp and at the +-pi / 2 clamp; a label outside the classes (NaN soft label, reg_mask 1); roi width 9
             and GT width 10; outputs pre-filled with NaN and 0xFF through the C ABI, every element rewritten.
  losses     the loss grid n = 1, 255, 256, 257, 2047, 2048, 2049, 16384 S - 1, 16384 S, 16384 S + 1 and 65536 S + 5 (S = SM count);
             cls_stride 3 and pred_stride 9 through the C ABI, bit-identical to contiguous inputs; corner_class -1 and 0, no corner loss,
             code weights with a 0; SmoothL1 at |d| = beta and one ulp either side (both branches agree there to
             within u in value and gradient, so this pins the continuity of the two branches, not which one |d| = beta takes); the
             corner loss at pred = 0 with pos_gt == roi (loss and gradient exactly 0), with the GT shifted up by exactly 1 (every
             distance 1, where the Huber branches meet) and with a predicted corner at the GT's centre (equidistant from a GT corner and
             its flipped twin: torch.min's tie splits the gradient in half); +-inf, NaN and +-100 logits; upstream gradients 0, 0.5 and 2^16,
             one per loss; gradient buffers pre-filled with NaN and 0xFF; two-run bit identity and no host sync on the capped grid.

Error model (u = 2^-24, every bound per element)
  IoU        |iou - iou64| <= IOU_C u (1 + R / m): R the largest |coordinate| of the pair's corners, m the smaller BEV extent of the two
             boxes (the fp32 corners x -+ w / 2 each round by u R, the clip and shoelace by a few u of the area).
  targets    |t - t64| <= TG_C u |t64| + TG_ABS: one rounding of a double result, plus the double error of its cancellations.
  cls grad   |g - g64| <= CLS_C u (s + |y|) |scale| + FLT_MIN |scale|, s = sigmoid(x): s and y are non-negative, their difference
             carries the rounding of s.
  box grad   |g - g64| <= BOX_C u (|g_l1| + |g_corner|) + exactly 0 where both float64 terms are 0.
  losses     |l - l64| <= LOSS_C u (sum of the terms' magnitudes) + u |l64|.
  yaw        the kernel (double, contracted) and the oracle (double, torch) may pick different branches of the canonical yaw only where
             the double relative yaw lies within YAW_BAND of pi / 2 or 3 pi / 2; no fp32 input pair came within 1e-9 of a branch point.

Bounds, with the worst values seen on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the file runs in about 50 s there):
  IOU_C     8      IoU, units of u (1 + R / m)                 5.7 (identical rotated boxes; 1.3 at 75 m)
  TG_C      2      targets, u relative                         1.0 (the final rounding to fp32)
  TG_ABS    1e-12  targets, absolute                           2.5e-14 (targets below 2^-20)
  CLS_C     8      classification gradient, units of u         5.1
  BOX_C     8      box gradient, units of u                    2.3
  LOSS_C    8      losses, units of u                          0.7
  YAW_BAND  1e-12  radians                                     no row fell inside it"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import roi_head_oracle as RO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
IOU_C = 8.0
TG_C = 2.0
TG_ABS = 1e-12
CLS_C = 8.0
BOX_C = 8.0
LOSS_C = 8.0
YAW_BAND = 1e-12
NAN = float("nan")
INF = float("inf")
ERR_ARG, ERR_UNSUPPORTED = -2, -3
SENT_I, SENT_F = -777, -3.25


def _ops():
    from sst_b200 import ops
    return ops


def _L():
    from sst_b200 import _lib as L
    return L


def f32(x):
    return float(np.float32(x))


def ulps(x, k):
    """the fp32 value k ulps from fl32(x)"""
    v = np.float32(x)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return float(v)


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count if torch.cuda.is_available() else 132


# ---------------------------------------------------------------------------------------------------------------------------------------
# assignment and sampling through the C ABI, with sentinel-filled outputs
# ---------------------------------------------------------------------------------------------------------------------------------------
def _cfg(assigners, per_class, num, pos_fraction, fr, th):
    return _ops().RoiSampleConfig([a[0] for a in assigners], [a[1] for a in assigners], [a[2] for a in assigners], per_class, num,
                                  pos_fraction, fr, th)


def _assign_c(samples, cfg, keys, expect_rc=0):
    """samples: (props, plab, gt, gl) per sample -> per sample (inds, iou fp32, gt_rows, labels, num_pos), sample-local; asserts the
    rows below each count are written and the rows from the count up to num keep their sentinel"""
    L, ops = _L(), _ops()
    props = torch.cat([s[0] for s in samples]).float().to(DEV).contiguous()
    plab = torch.cat([s[1] for s in samples]).long().to(DEV).contiguous()
    gts = [s[2] for s in samples]
    gw = next((g.shape[1] for g in gts if len(g)), 7)
    gt = torch.cat([g if len(g) else torch.zeros((0, gw)) for g in gts]).float().to(DEV).contiguous()
    gl = torch.cat([s[3] for s in samples]).long().to(DEV).contiguous()
    k = keys.float().to(DEV).contiguous()
    B, num = len(samples), cfg.num
    out_i = torch.full((B * num,), SENT_I, dtype=torch.int64, device=DEV)
    out_f = torch.full((B * num,), SENT_F, dtype=torch.float32, device=DEV)
    out_g, out_l = out_i.clone(), out_i.clone()
    counts = torch.full((B, 2), -1, dtype=torch.int32, device=DEV)
    poff, goff = ops._offsets([len(s[0]) for s in samples]), ops._offsets([len(g) for g in gts])
    c = L.ctx(DEV)
    rc = L.lib().sstb200_roi_assign_sample(c, C.byref(cfg.struct), L.ptr(props), props.shape[1], L.ptr(plab), L.ptr(k),
                                           L.arr(C.c_int32, poff), L.ptr(gt) if gt.numel() else None, gw,
                                           L.ptr(gl) if gl.numel() else None, L.arr(C.c_int32, goff), B, L.ptr(out_i), L.ptr(out_f),
                                           L.ptr(out_g), L.ptr(out_l), L.ptr(counts))
    assert rc == expect_rc, (rc, L.lib().sstb200_last_error(c))
    if rc:
        return None
    torch.cuda.synchronize()
    cnt = counts.cpu().tolist()
    oi, of, og, ol = out_i.cpu(), out_f.cpu(), out_g.cpu(), out_l.cpu()
    res = []
    for b, (npos, n) in enumerate(cnt):
        assert 0 <= npos <= n <= num, (b, npos, n)
        w, rest = slice(b * num, b * num + n), slice(b * num + n, (b + 1) * num)
        assert (oi[w] != SENT_I).all() and (og[w] != SENT_I).all() and (ol[w] != SENT_I).all(), f"sample {b}: a row below the count unwritten"
        assert (oi[rest] == SENT_I).all() and (of[rest] == SENT_F).all() and (og[rest] == SENT_I).all() and (ol[rest] == SENT_I).all(), \
            f"sample {b}: a row past the count written"
        rows = og[w]
        res.append((oi[w] - poff[b], of[w], torch.where(rows >= 0, rows - goff[b], rows), ol[w], npos))
    return res


def _expect(samples, keys, assigners, per_class, num, pf, fr, th, fp32=True):
    """the oracle's rows per sample; fp32: the kernel's own IoUs (dyadic yaw-0 boxes) and fp32-rounded thresholds"""
    out, at = [], 0
    if fp32:
        assigners = [tuple(f32(v) for v in a) for a in assigners]
        th = [f32(v) for v in th]
    for p, l, g, gl in samples:
        kk = keys[at:at + len(p)]
        out.append(RO.assign_and_sample(p, l, kk, g[:, :7], gl, assigners, per_class, num, pf, fr, th,
                                        iou=RO.iou3d_fp32_axis if fp32 else RO.iou3d))
        at += len(p)
    return out


def _compare(got, want, iou_exact=True):
    for b, (g, w) in enumerate(zip(got, want)):
        assert g[4] == w[4], f"sample {b}: {g[4]} positives, the oracle {w[4]}"
        assert torch.equal(g[0], w[0]), f"sample {b}: sampled proposals differ"
        assert torch.equal(g[2], w[2]), f"sample {b}: GT rows differ"
        assert torch.equal(g[3], w[3]), f"sample {b}: labels differ"
        if iou_exact:
            assert torch.equal(g[1].double(), w[1]), f"sample {b}: IoUs differ"


def _dyadic_sample(gen, n_props, n_gt, K=3, spread=12.0, dup_gt=0, dup_props=0, bad_labels=0.0):
    """yaw-0 boxes on a 1/8 grid: GTs spread over [-spread, spread]^2, proposals jittered around them (and a fifth far away)"""
    q = lambda t: torch.round(t * 8) / 8  # noqa: E731
    gl = torch.randint(0, K, (n_gt,), generator=gen)
    gt = torch.zeros((n_gt, 7))
    gt[:, :2] = q((torch.rand(n_gt, 2, generator=gen) * 2 - 1) * spread)
    gt[:, 2] = q(torch.rand(n_gt, generator=gen) - 1)
    gt[:, 3:6] = q(torch.tensor([1.0, 2.0, 1.0]) + torch.rand(n_gt, 3, generator=gen) * torch.tensor([2.0, 3.0, 1.0]))
    if dup_gt and n_gt:
        gt[-dup_gt:], gl[-dup_gt:] = gt[:dup_gt], gl[:dup_gt]
    props = torch.zeros((n_props, 7))
    if n_gt:
        k = torch.randint(0, n_gt, (n_props,), generator=gen)
        props[:] = gt[k]
        props[:, :3] += q(torch.randn(n_props, 3, generator=gen) * torch.tensor([0.6, 0.6, 0.2]))
        props[:, 3:6] = q(props[:, 3:6] * (1 + 0.2 * torch.randn(n_props, 3, generator=gen)).clamp(0.5, 1.5)).clamp(min=0.25)
        plab = torch.where(torch.rand(n_props, generator=gen) < 0.85, gl[k], torch.randint(0, K, (n_props,), generator=gen))
    else:
        plab = torch.randint(0, K, (n_props,), generator=gen)
    far = torch.rand(n_props, generator=gen) < 0.2
    props[far, :2] = q((torch.rand(int(far.sum()), 2, generator=gen) * 2 - 1) * spread)
    props[~(props[:, 3:6] > 0).all(1), 3:6] = 1.0
    if dup_props and n_props > dup_props:
        props[-dup_props:], plab[-dup_props:] = props[:dup_props], plab[:dup_props]
    if bad_labels:
        bad = torch.rand(n_props, generator=gen) < bad_labels
        plab[bad] = torch.where(torch.rand(int(bad.sum()), generator=gen) < 0.5, -1, K)
    return props, plab, gt, gl


FSD = [(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)]
ROUTES = {   # name: (specs [(n_props, n_gt)], assigners, per_class, num, pos_fraction, fractions, thresholds, extra)
    "P1": ([(1, 1)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "P31_32_33": ([(31, 4), (32, 4), (33, 4)], FSD, True, 16, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "P511_512_513": ([(511, 40), (512, 40), (513, 40)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "P1024_1025": ([(1024, 80), (1025, 80)], FSD, True, 512, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "P4096": ([(4096, 120)], FSD, False, 1024, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "G0_1": ([(300, 0), (300, 1)], FSD, True, 128, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "G511_512_513": ([(700, 511), (700, 512), (700, 513)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], dict(spread=40.0)),
    "G4096": ([(4096, 4096)], FSD, False, 2048, 0.55, [0.8, 0.2], [0.55, 0.1], dict(spread=80.0)),
    "B40_mixed": (None, FSD, True, 128, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "ignore_band": ([(600, 60), (400, 30)], [(0.6, 0.3, 0.6), (0.5, 0.2, 0.5), (0.5, 0.25, 0.5)], True, 256, 0.55, [0.8, 0.2],
                    [0.55, 0.1], {}),
    "min_pos_below_pos": ([(600, 60), (400, 30)], [(0.7, 0.7, 0.2), (0.6, 0.6, 0.1), (0.6, 0.4, 0.3)], True, 256, 0.55, [0.8, 0.2],
                          [0.55, 0.1], {}),
    "min_pos_zero": ([(600, 60), (400, 30), (50, 3)], [(0.45, 0.45, 0.0), (0.35, 0.35, 0.0), (0.35, 0.35, 0.0)], True, 256, 0.55,
                     [0.8, 0.2], [0.55, 0.1], {}),
    "pos_fraction_0": ([(600, 60)], FSD, True, 128, 0.0, [0.8, 0.2], [0.55, 0.1], {}),
    "pos_fraction_1": ([(600, 60)], FSD, True, 128, 1.0, [0.8, 0.2], [0.55, 0.1], {}),
    "one_piece": ([(600, 60), (300, 20)], FSD, True, 128, 0.3, [1.0], [0.55], {}),
    "three_pieces": ([(900, 60), (600, 20)], FSD, True, 200, 0.25, [0.5, 0.3, 0.2], [0.55, 0.3, 0.05], {}),
    "three_pieces_carry": ([(900, 60), (600, 20)], FSD, True, 200, 0.25, [0.4, 0.5, 0.1], [0.95, 0.9, 0.02], {}),
    "nneg_le_nexp": ([(60, 10), (5, 2), (1, 0)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], {}),
    "key_ties": ([(800, 60), (600, 40)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], dict(ties=True)),
    "duplicates": ([(800, 60), (600, 40)], [(0.7, 0.7, 0.2), (0.6, 0.6, 0.1), (0.6, 0.4, 0.3)], True, 256, 0.55, [0.8, 0.2],
                   [0.55, 0.1], dict(dup_gt=15, dup_props=150)),
    "bad_labels_per_class": ([(600, 60), (300, 20)], FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1], dict(bad_labels=0.2)),
    "bad_labels_one_assigner": ([(600, 60), (300, 20)], FSD, False, 256, 0.55, [0.8, 0.2], [0.55, 0.1], dict(bad_labels=0.2)),
}


@pytest.mark.parametrize("name", list(ROUTES))
def test_assign_sample_routes(name):
    specs, assigners, per_class, num, pf, fr, th, extra = ROUTES[name]
    gen = torch.Generator().manual_seed(100 + list(ROUTES).index(name))
    if specs is None:
        specs = [(int(np.random.RandomState(b).choice([1, 2, 50, 300, 600])), int(np.random.RandomState(50 + b).choice([0, 1, 5, 30])))
                 for b in range(40)]
    if not per_class:
        assigners = assigners[:1]
    kw = {k: v for k, v in extra.items() if k != "ties"}
    samples = [_dyadic_sample(gen, n, g, **kw) for n, g in specs]
    P = sum(n for n, _ in specs)
    keys = torch.rand(P, generator=gen)
    if extra.get("ties"):
        keys = torch.floor(keys * 4) / 4
    got = _assign_c(samples, _cfg(assigners, per_class, num, pf, fr, th), keys)
    want = _expect(samples, keys, assigners, per_class, num, pf, fr, th)
    _compare(got, want)
    npos = [w[4] for w in want]
    print(f"{name}: rows {[len(w[0]) for w in want][:8]}, positives {npos[:8]}")
    if name in ("ignore_band", "min_pos_below_pos", "duplicates", "min_pos_zero"):
        assert sum(npos) > 0


def test_piece_with_exactly_want_members():
    """no positives, num 10: piece 0 ([0.1, 0.55)) holds exactly int(10 * 0.8) = 8 negatives, the last piece the other 20"""
    gt = torch.tensor([[0, 0, 0, 4, 4, 2, 0]], dtype=torch.float32)
    near = gt.repeat(8, 1)
    near[:, 0] = 2.0 + torch.arange(8) / 8            # IoU (4 - s) / (4 + s) in [0.16, 0.34]
    far = gt.repeat(20, 1)
    far[:, 0] = 40.0 + torch.arange(20) * 8
    props = torch.cat([far[:10], near, far[10:]])
    samples = [(props, torch.zeros(28, dtype=torch.int64), gt, torch.zeros(1, dtype=torch.int64))]
    for seed in range(4):
        keys = torch.rand(28, generator=torch.Generator().manual_seed(seed))
        got = _assign_c(samples, _cfg(FSD[:1], False, 10, 0.55, [0.8, 0.2], [0.55, 0.1]), keys)
        want = _expect(samples, keys, FSD[:1], False, 10, 0.55, [0.8, 0.2], [0.55, 0.1])
        _compare(got, want)
        assert set(range(10, 18)) <= set(got[0][0].tolist()) and len(got[0][0]) == 10


def test_refusals():
    """more than 4096 proposals or GTs in a sample, 4 IoU pieces, a negative fraction, non-last fractions past 1.  The piece settings
    come with fewer negatives than num, so that a kernel that took them would still stay within its rows."""
    gen = torch.Generator().manual_seed(9)
    s = _dyadic_sample(gen, 50, 5)
    keys = torch.rand(4097, generator=gen)
    _assign_c([_dyadic_sample(gen, 4097, 5)], _cfg(FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1]), keys, ERR_UNSUPPORTED)
    _assign_c([_dyadic_sample(gen, 20, 4097, spread=80.0)], _cfg(FSD, True, 256, 0.55, [0.8, 0.2], [0.55, 0.1]), keys[:20],
              ERR_UNSUPPORTED)
    _assign_c([s], _cfg(FSD, True, 256, 0.55, [0.3, 0.3, 0.3, 0.1], [0.55, 0.45, 0.3, 0.1]), keys[:50], ERR_UNSUPPORTED)
    _assign_c([s], _cfg(FSD, True, 256, 0.55, [0.5, -0.1, 0.6], [0.55, 0.3, 0.1]), keys[:50], ERR_ARG)
    _assign_c([s], _cfg(FSD, True, 256, 0.55, [0.7, 0.4, 0.1], [0.55, 0.3, 0.1]), keys[:50], ERR_ARG)
    # the largest accepted sizes still run
    _assign_c([_dyadic_sample(gen, 4096, 1)], _cfg(FSD, True, 64, 0.55, [0.8, 0.2], [0.55, 0.1]), keys[:4096])


# ---------------------------------------------------------------------------------------------------------------------------------------
# thresholds at equality
# ---------------------------------------------------------------------------------------------------------------------------------------
def _pair_at(v, x0=0.0):
    """(gt, prop) yaw-0 boxes whose kernel IoU is exactly the fp32 value v: the proposal, shifted by s along x and pl long in y, has its
    height swept over consecutive fp32 values (its z range covers the GT's, so the overlap height stays the GT's 2); several (s, pl)
    are tried, as one sweep may step over a value"""
    L = 4.0
    gt = torch.tensor([[x0, 0, 0, L, 4, 2, 0]], dtype=torch.float32)
    for s in (1.0, 0.5, 1.5, 0.25, 0.75, 1.25, 2.0):
        for pl in (4.0, 6.0, 8.0, 5.0):
            ov = (L - s) * 4 * 2
            h0 = np.float32((ov / v - L * 8 + ov) / (L * pl))
            if not h0 >= 2:
                continue
            hs = [h0]
            a = b = h0
            for _ in range(200):
                a, b = np.nextafter(a, np.float32(-np.inf)), np.nextafter(b, np.float32(np.inf))
                hs += [a, b]
            props = torch.tensor([[x0 + s, 0, 0, L, pl, float(h), 0] for h in hs], dtype=torch.float32)
            iou = RO.iou3d_fp32_axis(gt, props)[0]
            hit = torch.nonzero(iou == torch.tensor(v, dtype=torch.float32)).view(-1)
            if len(hit):
                return gt, props[int(hit[0])][None]
    raise AssertionError(f"no proposal gives IoU {v!r}")


def _threshold_sample(values, others=(), x0=0.0, exact_best=True):
    """one GT with one proposal per IoU value (and an identical proposal, IoU 1, so that the GT's best proposal is not among them)"""
    props = []
    for v in values:
        gt, p = _pair_at(v, x0)
        props.append(p)
    if exact_best:
        props.append(gt.clone())
    props = torch.cat(props + list(others))
    return props, torch.zeros(len(props), dtype=torch.int64), gt, torch.zeros(1, dtype=torch.int64)


def _thr_run(samples, assigners, num, pf, fr, th, per_class=False, seed=0):
    P = sum(len(s[0]) for s in samples)
    keys = torch.rand(P, generator=torch.Generator().manual_seed(seed))
    got = _assign_c(samples, _cfg(assigners, per_class, num, pf, fr, th), keys)
    want = _expect(samples, keys, assigners, per_class, num, pf, fr, th)
    _compare(got, want)
    return got


def _gi_of(res, n):
    """proposal -> 1 + GT row for positives, 0 for sampled negatives, -1 for rows not sampled"""
    inds, _, rows, _, _ = res
    out = torch.full((n,), -1, dtype=torch.int64)
    out[inds] = torch.where(rows >= 0, rows + 1, torch.zeros_like(rows))
    return out


@pytest.mark.parametrize("t", [0.45, 0.35, 0.55])
def test_pos_threshold_at_equality(t):
    """mo >= pos at fl32(t) and one ulp either side; neg = pos, so the one below is negative"""
    vals = [ulps(t, -1), f32(t), ulps(t, 1)]
    s = _threshold_sample(vals)
    got = _thr_run([s], [(t, t, t)], 64, 1.0, [0.8, 0.2], [0.55, 0.1])
    assert torch.equal(RO.iou3d_fp32_axis(s[2], s[0])[0][:3], torch.tensor(vals, dtype=torch.float32))
    assert _gi_of(got[0], 4).tolist() == [0, 1, 1, 1]


@pytest.mark.parametrize("t", [0.45, 0.35, 0.1])
def test_neg_threshold_at_equality(t):
    """mo < neg with an ignore band (pos 0.9): below fl32(t) negative, at and above it ignored"""
    s = _threshold_sample([ulps(t, -1), f32(t), ulps(t, 1)])
    got = _thr_run([s], [(0.9, t, 0.9)], 64, 1.0, [0.8, 0.2], [0.55, 0.1])
    assert _gi_of(got[0], 4).tolist() == [0, -1, -1, 1]


@pytest.mark.parametrize("t", [0.45, 0.35, 0.1])
def test_min_pos_at_equality(t):
    """m >= min_pos: three GTs 32 m apart, each with a single proposal at fl32(t) - 1 ulp, fl32(t), + 1 ulp; pos 0.9 and neg 0.05, so
    only the low-quality match can make them positive"""
    samples = []
    props, gts = [], []
    for j, v in enumerate([ulps(t, -1), f32(t), ulps(t, 1)]):
        g, p = _pair_at(v, x0=32.0 * j)
        props.append(p), gts.append(g)
    samples = [(torch.cat(props), torch.zeros(3, dtype=torch.int64), torch.cat(gts), torch.zeros(3, dtype=torch.int64))]
    got = _thr_run(samples, [(0.9, 0.05, t)], 64, 1.0, [0.8, 0.2], [0.55, 0.1])
    assert _gi_of(got[0], 3).tolist() == [-1, 2, 3]


def test_piece_bounds_at_equality():
    """negatives at 0.55 and 0.1 (fl32 rounds both up) and one ulp either side, pieces [0.1, 0.55) and [0, 0.1): 24 samples of the same
    boxes under different keys, num 3 (one positive, two negatives, one from each piece)"""
    vals = [ulps(0.55, -1), f32(0.55), ulps(0.55, 1), ulps(0.1, -1), f32(0.1), ulps(0.1, 1), 0.3, 0.05]
    base = _threshold_sample(vals)
    samples = [base] * 24
    got = _thr_run(samples, [(0.9, 0.9, 0.95)], 3, 0.34, [0.5, 0.5], [0.55, 0.1], seed=3)
    chosen = torch.zeros(len(vals) + 1)
    for r in got:
        chosen[r[0]] += 1
    # 0.55 and above lie in no piece; the rest are drawn by their keys
    assert chosen[1] == 0 and chosen[2] == 0 and chosen[len(vals)] == 24 and chosen.sum() == 3 * 24


def test_soft_label_thresholds_at_equality():
    """get_multi_class_soft_label: iou > pos -> 1, !(iou < neg) -> (iou - neg) / (pos - neg), else 0, with fp32 compares and an fp32
    divisor formed in double: bit for bit at fl32(pos), fl32(neg) and one ulp either side, for every class"""
    ops = _ops()
    pos, neg = (0.8, 0.65, 0.65), (0.2, 0.15, 0.15)
    ious, labs = [], []
    for c in range(3):
        for t in (pos[c], neg[c]):
            for k in (-1, 0, 1):
                ious.append(ulps(t, k))
                labs.append(c)
    R = len(ious)
    iou = torch.tensor(ious, dtype=torch.float32)
    lab = torch.tensor(labs)
    rois = torch.tensor([[0, 0, 0, 2, 4, 1.5, 0.1]] * R, dtype=torch.float32)
    soft, _, _, _ = ops.roi_head_targets(rois.to(DEV), iou.to(DEV), torch.arange(R).to(DEV), lab.to(DEV), rois.to(DEV), pos, neg)
    want = torch.zeros(R, dtype=torch.float32)
    for r in range(R):
        c = labs[r]
        p32, n32 = np.float32(pos[c]), np.float32(neg[c])
        v = np.float32(ious[r])
        want[r] = 1.0 if v > p32 else (float(np.float32(v - n32) / np.float32(pos[c] - neg[c])) if not v < n32 else 0.0)
    assert _bits(soft.cpu(), want), (soft.cpu(), want)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 3-D IoU element by element
# ---------------------------------------------------------------------------------------------------------------------------------------
def _iou_case(name, gen):
    """(gts [B, 7], props [B, n, 7]): one GT per sample and n proposals around it"""
    B, n = 16, 64
    gt = torch.zeros((B, 7))
    centre = {"far": 75.0}.get(name, 0.0)
    ang = torch.rand(B, generator=gen) * 2 * math.pi
    gt[:, 0], gt[:, 1] = centre * torch.cos(ang), centre * torch.sin(ang)
    gt[:, 2] = torch.rand(B, generator=gen) - 1
    size = torch.tensor([0.4, 0.6, 0.5]) if name == "submetre" else torch.tensor([2.0, 4.5, 1.6])
    gt[:, 3:6] = size * (0.7 + 0.6 * torch.rand(B, 3, generator=gen))
    gt[:, 6] = (torch.rand(B, generator=gen) * 2 - 1) * math.pi
    p = gt[:, None, :].repeat(1, n, 1)
    if name == "identical":
        pass
    else:
        p[..., :2] += torch.randn(B, n, 2, generator=gen) * size[:2].max() * 0.4
        p[..., 2] += torch.randn(B, n, generator=gen) * 0.3
        p[..., 3:6] *= (1 + 0.2 * torch.randn(B, n, 3, generator=gen)).clamp(0.5, 1.5)
        p[..., 6] += torch.randn(B, n, generator=gen) * 0.5
    if name == "z_edges":
        h = gt[:, None, 5]
        k = torch.arange(n) % 4
        p[..., 2] = torch.where(k == 0, gt[:, None, 2] + h, p[..., 2])                                # touches the top
        p[..., 2] = torch.where(k == 1, gt[:, None, 2] - p[..., 5], p[..., 2])                        # touches the bottom
        nest = k == 2
        p[..., 5] = torch.where(nest, h * 0.5, p[..., 5])
        p[..., 2] = torch.where(nest, gt[:, None, 2] + h * 0.25, p[..., 2])                           # nested
        p[..., 2] = torch.where(k == 3, gt[:, None, 2] + h + 1.0, p[..., 2])                          # disjoint
    if name == "zero_volume":
        k = torch.arange(n) % 4
        for c in range(3):
            p[..., 3 + c] = torch.where(k == c, torch.zeros_like(p[..., 3 + c]), p[..., 3 + c])
        gt[::4, 3] = 0.0                                                                              # zero-width GTs too
    return gt, p


@pytest.mark.parametrize("name,pw,gw", [("origin", 7, 7), ("far", 7, 9), ("submetre", 9, 10), ("identical", 7, 7), ("z_edges", 9, 7),
                                        ("zero_volume", 7, 10), ("far_submetre", 9, 9)])
def test_iou_elementwise(name, pw, gw):
    gen = torch.Generator().manual_seed(len(name) * 7 + pw + gw)
    if name == "far_submetre":
        gt, p = _iou_case("submetre", gen)
        gt[:, :2] += 75.0 / math.sqrt(2)
        p[..., :2] += 75.0 / math.sqrt(2)
    else:
        gt, p = _iou_case(name, gen)
    B, n = p.shape[:2]
    gtw = torch.cat([gt, torch.randn(B, gw - 7, generator=gen)], 1) if gw > 7 else gt
    pp = torch.cat([p, torch.randn(B, n, pw - 7, generator=gen)], 2) if pw > 7 else p
    samples = [(pp[b].float(), torch.zeros(n, dtype=torch.int64), gtw[b:b + 1].float(), torch.zeros(1, dtype=torch.int64)) for b in range(B)]
    keys = torch.rand(B * n, generator=gen)
    got = _assign_c(samples, _cfg([(0.5, 0.5, 0.5)], False, n, 1.0, [0.8, 0.2], [0.55, 0.1]), keys)
    worst = 0.0
    for b, r in enumerate(got):
        assert len(r[0]) == n
        iou = torch.empty(n, dtype=torch.float32)
        iou[r[0]] = r[1]
        ref = RO.iou3d(gt[b:b + 1].float(), p[b].float())[0]
        assert not torch.isnan(iou).any(), f"{name}: NaN IoU"
        g32, p32 = gt[b:b + 1].float().double(), p[b].float().double()
        zero = (p32[:, 3:6] == 0).any(1) | bool((g32[0, 3:6] == 0).any())
        assert (iou[zero] == 0).all(), f"{name}: a zero-volume box with IoU {iou[zero].abs().max()}"
        ext = lambda t: torch.sqrt(t[:, 3] ** 2 + t[:, 4] ** 2) / 2  # noqa: E731
        R = torch.max(g32[0, :2].abs().max() + ext(g32)[0], p32[:, :2].abs().max(1).values + ext(p32))
        m = torch.min(torch.min(g32[0, 3:5]).expand(n), p32[:, 3:5].min(1).values)
        ok = ~zero
        bound = IOU_C * U * (1 + R[ok] / m[ok])
        err = (iou[ok].double() - ref[ok]).abs()
        assert (err <= bound).all(), f"{name}: IoU off by {float((err / bound).max()):.3g} of the bound"
        if err.numel():
            worst = max(worst, float((err / bound).max()))
        if name == "z_edges":
            k = torch.arange(n) % 4
            assert (iou[(k == 0) | (k == 3)] == 0).all()   # touching from above (the kernel's zt is torch's fp32 z + h) and apart
    print(f"IoU {name}: worst {worst:.3f} of the bound")


# ---------------------------------------------------------------------------------------------------------------------------------------
# the low-quality match on rotated crowds far from the origin
# ---------------------------------------------------------------------------------------------------------------------------------------
def _crowd(seed, n_gt=200, n_props=1500, margin=1e-4, thrs=(0.7, 0.3, 0.1)):
    g = torch.Generator().manual_seed(seed)
    ang = float(torch.rand(1, generator=g)) * 2 * math.pi
    cx, cy = 70 * math.cos(ang), 70 * math.sin(ang)
    gt = torch.zeros((n_gt, 7))
    gt[:, 0] = cx + (torch.rand(n_gt, generator=g) * 2 - 1) * 15
    gt[:, 1] = cy + (torch.rand(n_gt, generator=g) * 2 - 1) * 15
    gt[:, 2] = torch.rand(n_gt, generator=g) * 0.4 - 1
    gt[:, 3:6] = torch.tensor([2.0, 4.5, 1.6]) * (0.8 + 0.4 * torch.rand(n_gt, 3, generator=g))
    gt[:, 6] = (torch.rand(n_gt, generator=g) * 2 - 1) * math.pi
    k = torch.randint(0, n_gt, (n_props,), generator=g)
    p = gt[k].clone()
    p[:, :2] += torch.randn(n_props, 2, generator=g) * 1.0
    p[:, 2] += torch.randn(n_props, generator=g) * 0.2
    p[:, 3:6] *= (1 + 0.2 * torch.randn(n_props, 3, generator=g)).clamp(0.6, 1.4)
    p[:, 6] += torch.randn(n_props, generator=g) * 0.4
    gt, p = gt.float(), p.float()
    # keep the float64 decisions away from fp32's reach: no IoU near a threshold, no near-tie for a GT's best proposal or a
    # proposal's best GT
    for _ in range(6):
        ov = RO.iou3d(gt, p)
        bad = torch.zeros(len(p), dtype=torch.bool)
        for t in thrs:
            bad |= ((ov - t).abs() < margin).any(0)
        top2 = ov.topk(2, 0).values if len(gt) > 1 else None
        if top2 is not None:
            bad |= (top2[0] > 0) & (top2[0] - top2[1] < margin)
        srt = ov.sort(1, descending=True).values
        near_best = (ov > 0) & (ov < ov.max(1, keepdim=True).values) & (ov > ov.max(1, keepdim=True).values - margin)
        bad |= near_best.any(0)
        gbad = (srt[:, 0] - thrs[2]).abs() < margin
        if not bad.any() and not gbad.any():
            break
        p = p[~bad]
        gt = gt[~gbad]
    return gt, p


def test_low_quality_match_on_rotated_crowds():
    """min_pos 0.1 < pos 0.7: a GT's best proposal goes to that GT even when its own best GT is another one, or its IoU is below pos.
    The kernel finds it by recomputing the IoU and comparing it with the per-GT maximum with ==."""
    samples, thr = [], (0.7, 0.3, 0.1)
    for b in range(4):
        gt, p = _crowd(40 + b, thrs=thr)
        samples.append((p, torch.zeros(len(p), dtype=torch.int64), gt, torch.zeros(len(gt), dtype=torch.int64)))
    P = sum(len(s[0]) for s in samples)
    keys = torch.rand(P, generator=torch.Generator().manual_seed(1))
    num = max(len(s[0]) for s in samples)
    got = _assign_c(samples, _cfg([thr], False, num, 1.0, [0.8, 0.2], [0.55, 0.1]), keys)
    want = _expect(samples, keys, [thr], False, num, 1.0, [0.8, 0.2], [0.55, 0.1], fp32=False)
    _compare(got, want, iou_exact=False)
    moved = 0
    for (p, _, gt, _), w in zip(samples, want):
        ov = RO.iou3d(gt, p)
        mo, arg = ov.max(0)
        plain = torch.where(mo >= thr[0], arg + 1, torch.where(mo < thr[1], torch.zeros_like(arg), torch.full_like(arg, -1)))
        final = torch.full((len(p),), -1, dtype=torch.int64)
        final[w[0]] = torch.where(w[2] >= 0, w[2] + 1, torch.zeros_like(w[2]))
        moved += int((final != plain).sum())
    print(f"low-quality: {moved} proposals re-targeted or promoted over {len(samples)} crowds")
    assert moved >= 300


# ---------------------------------------------------------------------------------------------------------------------------------------
# targets
# ---------------------------------------------------------------------------------------------------------------------------------------
POS, NEG = (0.8, 0.65, 0.65), (0.2, 0.15, 0.15)


def _targets_inputs(seed, R, rw=7, gw=7, yaws=None):
    g = torch.Generator().manual_seed(seed)
    rois = torch.zeros((R, rw))
    rois[:, :2] = torch.randn(R, 2, generator=g) * 30
    rois[:, 2] = torch.randn(R, generator=g) * 0.3
    rois[:, 3:6] = torch.tensor([2.0, 4.5, 1.6]) * (0.5 + torch.rand(R, 3, generator=g))
    rois[:, 6] = (torch.rand(R, generator=g) * 4 - 2) * math.pi
    if rw > 7:
        rois[:, 7:] = torch.randn(R, rw - 7, generator=g)
    gt = torch.zeros((R, gw))
    gt[:, :7] = rois[:, :7]
    gt[:, :3] += torch.randn(R, 3, generator=g) * 0.5
    gt[:, 3:6] *= (1 + 0.2 * torch.randn(R, 3, generator=g)).clamp(0.5, 1.5)
    gt[:, 6] += torch.randn(R, generator=g) * 2
    if gw > 7:
        gt[:, 7:] = torch.randn(R, gw - 7, generator=g)
    if yaws is not None:
        rois[:len(yaws[0]), 6] = torch.tensor(yaws[0])
        gt[:len(yaws[1]), 6] = torch.tensor(yaws[1])
    rows = torch.where(torch.rand(R, generator=g) < 0.7, torch.arange(R), torch.full((R,), -1))
    lab = torch.where(rows >= 0, torch.randint(0, 3, (R,), generator=g), torch.full((R,), -1))
    iou = torch.rand(R, generator=g)
    return rois.float(), gt.float(), rows, lab, iou.float()


def _targets_check(name, rois, gt, rows, lab, iou, K=3):
    ops = _ops()
    soft, reg_mask, bt, pg = ops.roi_head_targets(rois.to(DEV), iou.to(DEV), rows.to(DEV), lab.to(DEV), gt.to(DEV), POS[:K], NEG[:K])
    soft, reg_mask, bt, pg = soft.cpu(), reg_mask.cpu(), bt.cpu(), pg.cpu()
    pos = rows >= 0
    assert torch.equal(reg_mask, pos.long())
    assert (soft[~pos] == 0).all() and (bt[~pos] == 0).all() and (pg[~pos] == 0).all()
    assert torch.equal(pg[pos], gt[rows[pos], :7])
    inside = pos & (lab >= 0) & (lab < K)
    assert torch.isnan(soft[pos & ~inside]).all(), f"{name}: a label outside the classes must give a NaN soft label"
    # soft labels: fp32 compares, bit for bit
    li = lab[inside]
    p32, n32 = torch.tensor(POS[:K], dtype=torch.float32)[li], torch.tensor(NEG[:K], dtype=torch.float32)[li]
    span = torch.tensor([f32(a - b) for a, b in zip(POS[:K], NEG[:K])], dtype=torch.float32)[li]
    v = iou[inside]
    want = torch.where(v > p32, torch.ones_like(v), torch.where(v < n32, torch.zeros_like(v), (v - n32) / span))
    assert _bits(soft[inside], want), f"{name}: soft labels differ"
    # box targets against the float64 oracle
    if not pos.any():
        return 0.0
    ref_lab = torch.where(inside, lab, torch.zeros_like(lab))[pos]
    _, bt64 = RO.targets(rois[pos], iou[pos].double(), gt[rows[pos]], ref_lab, POS[:K], NEG[:K])
    got = bt[pos].double()
    # the canonical yaw: the double relative yaw of each row, and its distance from the branch points
    ry = torch.remainder(rois[pos, 6].double(), 2 * math.pi)
    yl = torch.remainder(gt[rows[pos], 6].double() - ry, 2 * math.pi)
    near = torch.min((yl - math.pi / 2).abs(), (yl - 1.5 * math.pi).abs()) <= YAW_BAND
    ok = torch.ones_like(got, dtype=torch.bool)
    ok[near, 6] = False
    err = (got - bt64).abs()
    bound = TG_C * U * bt64.abs() + TG_ABS
    assert (err[ok] <= bound[ok]).all(), f"{name}: box targets off by {float((err / bound)[ok].max()):.3g} of the bound"
    small = ok & (bt64.abs() < 2.0 ** -20)
    if small.any():
        print(f"{name}: worst absolute error of targets below 2^-20: {float(err[small].max()):.3g}")
    if near.any():
        print(f"{name}: {int(near.sum())} rows inside the undecided yaw band")
    return float((err / bound)[ok].max())


@pytest.mark.parametrize("R", [1, 255, 256, 257, 70001])
def test_targets_row_counts(R):
    w = _targets_check(f"R={R}", *_targets_inputs(R, R))
    print(f"targets R={R}: worst {w:.3f} of the bound")


def test_targets_yaw_edges():
    """roi and GT yaws at -2 pi, -pi, 0, pi, 2 pi and their fp32 neighbours against each other; relative yaws at pi / 2 and 3 pi / 2
    +- 1..4 ulp of the GT yaw; relative yaws past the +-pi / 2 clamp"""
    base = [-2 * math.pi, -math.pi, 0.0, math.pi, 2 * math.pi]
    ys = sorted({ulps(v, k) for v in base for k in (-1, 0, 1)})
    ry = [a for a in ys for _ in ys]
    gy = [b for _ in ys for b in ys]
    for r in (0.3, -1.2, 2.5):
        for branch in (0.5 * math.pi, 1.5 * math.pi, -0.5 * math.pi):
            for k in range(-4, 5):
                ry.append(r)
                gy.append(ulps(r + branch, k))
    for r in (0.0, 1.0):
        for d in (0.49 * math.pi, 0.51 * math.pi, 1.49 * math.pi, 1.51 * math.pi, 0.9 * math.pi, 1.1 * math.pi):
            ry.append(r)
            gy.append(r + d)
    R = len(ry)
    rois, gt, rows, lab, iou = _targets_inputs(77, R, yaws=(ry, gy))
    rows, lab = torch.arange(R), torch.randint(0, 3, (R,), generator=torch.Generator().manual_seed(0))
    w = _targets_check("yaw edges", rois, gt, rows, lab, iou)
    print(f"targets yaw edges: worst {w:.3f} of the bound")


def test_targets_widths_and_labels_outside_the_classes():
    rois, gt, rows, lab, iou = _targets_inputs(5, 3001, rw=9, gw=10)
    lab = torch.where((rows >= 0) & (torch.arange(3001) % 7 == 0), torch.full_like(lab, 3), lab)
    _targets_check("rw 9 gw 10, label 3", rois, gt, rows, lab, iou)


@pytest.mark.parametrize("fill", ["nan", "ff"])
def test_targets_dirty_outputs_c_abi(fill):
    L, ops = _L(), _ops()
    rois, gt, rows, lab, iou = _targets_inputs(6, 4099, rw=9, gw=9)
    d = [t.to(DEV).contiguous() for t in (rois, iou, rows, lab, gt)]
    ref = ops.roi_head_targets(*d[:4], d[4], POS, NEG)
    outs = [torch.empty_like(t) for t in ref]
    for t in outs:
        if fill == "nan" and t.is_floating_point():
            t.fill_(NAN)
        else:
            t.view(torch.uint8).fill_(0xFF)
    c = L.ctx(DEV)
    L.check(c, L.lib().sstb200_roi_head_targets(c, L.ptr(d[0]), 9, L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), 4099, L.ptr(d[4]), 9, 3,
                                                L.arr(C.c_double, list(POS)), L.arr(C.c_double, list(NEG)), *[L.ptr(t) for t in outs]))
    torch.cuda.synchronize()
    for a, b in zip(outs, ref):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------------------------------------------------------------------
class Loss:
    """synthetic RoI loss inputs: rois, row-aligned targets (from the native targets kernel), logits and predictions"""

    def __init__(self, seed, R, npos_frac=0.3, empty=0.2, car=0.5, max_pos=None):
        g = torch.Generator().manual_seed(seed)
        self.R = R
        rois = torch.zeros((R, 7))
        rois[:, :2] = torch.randn(R, 2, generator=g) * 20
        rois[:, 2] = torch.randn(R, generator=g) * 0.3
        rois[:, 3:6] = torch.tensor([2.0, 4.5, 1.6]) * (1 + 0.2 * torch.rand(R, 3, generator=g))
        rois[:, 6] = (torch.rand(R, generator=g) * 2 - 1) * math.pi
        gt = rois.clone()
        gt[:, :3] += torch.randn(R, 3, generator=g) * 0.3
        gt[:, 3:6] *= 1 + 0.1 * torch.randn(R, 3, generator=g)
        gt[:, 6] += 0.3 * torch.randn(R, generator=g) + (torch.rand(R, generator=g) < 0.2).float() * math.pi
        pos = torch.rand(R, generator=g) < npos_frac
        if max_pos is not None:
            pos &= torch.arange(R) < max_pos * 3
        self.rows = torch.where(pos, torch.arange(R), torch.full((R,), -1))
        lab = torch.where(torch.rand(R, generator=g) < car, 0, torch.randint(1, 3, (R,), generator=g))
        self.lab = torch.where(pos, lab, torch.full_like(lab, -1))
        self.iou = torch.rand(R, generator=g)
        self.nonempty = torch.rand(R, generator=g) >= empty
        self.x = (torch.randn(R, 1, generator=g) * 2).float()
        self.p = (torch.randn(R, 7, generator=g) * 0.3).float()
        self.rois, self.gt = rois.float(), gt.float()
        self.kw = dict(w_cls=1.0, w_bbox=2.0, smooth_l1=False, beta=1.0, code_weights=None, with_corner=True, corner_class=0, w_corner=1.0)
        self.up = torch.tensor([1.0, 0.7, 1.3])
        self.targets()

    def targets(self):
        ops = _ops()
        t = ops.roi_head_targets(self.rois.to(DEV), self.iou.to(DEV), self.rows.to(DEV), self.lab.to(DEV), self.gt.to(DEV), POS, NEG)
        self.soft, self.reg_mask, self.bt, self.pg = [a.cpu() for a in t]

    def cfg(self):
        k = self.kw
        return _ops().RoiLossConfig(k["w_cls"], k["w_bbox"], k["smooth_l1"], k["beta"], k["with_corner"], k["corner_class"],
                                    k["w_corner"], k["code_weights"])

    def avg(self):
        npos = float(((self.reg_mask > 0) & self.nonempty).sum())
        return torch.tensor([float(self.R)]), torch.tensor([npos])

    def run(self, x=None, p=None):
        ops = _ops()
        x = (self.x if x is None else x).to(DEV).requires_grad_(True)
        p = (self.p if p is None else p).to(DEV).requires_grad_(True)
        ca, ra = self.avg()
        losses = ops.roi_head_loss(x, p, self.nonempty.to(DEV), self.soft.to(DEV), self.reg_mask.to(DEV), self.bt.to(DEV), self.pg.to(DEV),
                                   self.lab.to(DEV), self.rois.to(DEV), ca.to(DEV), ra.to(DEV), self.cfg())
        losses.backward(self.up.to(DEV))
        return losses.detach().cpu(), x.grad.cpu(), p.grad.cpu()

    def ref(self, x=None, p=None):
        """float64 losses and the gradients of each term separately"""
        x64 = (self.x if x is None else x).double().requires_grad_(True)
        p64 = (self.p if p is None else p).double().requires_grad_(True)
        kw = dict(self.kw)
        ca, ra = self.avg()
        kw["cls_avg"] = float(ca)
        kw["reg_avg"] = float(ra) if float(ra) > 0 else None
        out = RO.losses(x64, p64, self.nonempty, self.soft, self.reg_mask, self.bt, self.pg, self.lab, self.rois, kw)
        vals = [out['loss_rcnn_cls'], out['loss_rcnn_bbox'], out['loss_rcnn_corner']]
        gx = torch.autograd.grad(vals[0] * float(self.up[0]), x64, allow_unused=True, retain_graph=True)[0]
        gb = torch.autograd.grad(vals[1] * float(self.up[1]), p64, allow_unused=True, retain_graph=True)[0]
        gk = torch.autograd.grad(vals[2] * float(self.up[2]), p64, allow_unused=True, retain_graph=True)[0]
        z = torch.zeros_like(p64)
        return [float(v) for v in vals], gx if gx is not None else torch.zeros_like(x64), gb if gb is not None else z, \
            gk if gk is not None else z


def _loss_check(name, lo, x=None, p=None, nan_x=None):
    losses, gx, gp = lo.run(x, p)
    vals, rx, rb, rk = lo.ref(x, p)
    xx = (lo.x if x is None else x).double()[:, 0]
    # classification gradient
    ne = lo.nonempty
    scale = float(lo.up[0]) * lo.kw["w_cls"] / lo.R
    s = torch.sigmoid(xx)
    y = lo.soft.double()
    gxv = gx[:, 0].double()
    want_nan = torch.isnan(xx) & ne if nan_x is None else nan_x
    assert torch.equal(torch.isnan(gxv), want_nan), f"{name}: NaN classification gradients at the wrong rows"
    ok = ~want_nan & torch.isfinite(xx)
    bound = CLS_C * U * (s + y.abs()) * abs(scale) + FLT_MIN * abs(scale)
    err = (gxv - rx[:, 0])[ok].abs()
    assert (err <= bound[ok]).all(), f"{name}: classification gradient off by {float((err / bound[ok]).max()):.3g}"
    assert (gxv[~ne] == 0).all(), f"{name}: an empty RoI with a classification gradient"
    wc = CLS_C * float((err / bound[ok]).max()) if err.numel() else 0.0
    # box gradient: L1 / SmoothL1 plus corner
    ref = rb + rk
    gpd = gp.double()
    both0 = (rb == 0) & (rk == 0)
    assert (gpd[both0] == 0).all(), f"{name}: {int((gpd[both0] != 0).sum())} box gradients nonzero where the reference's are 0"
    bb = BOX_C * U * (rb.abs() + rk.abs()) + 1e-300
    e = (gpd - ref).abs()
    assert (e <= bb).all(), f"{name}: box gradient off by {float((e / bb).max()):.3g} of the bound"
    wb = BOX_C * float((e / bb).max())
    wl = 0.0
    # losses
    if not math.isnan(vals[0]):
        terms = (torch.clamp(xx, min=0) + xx.abs() * y + torch.log1p(torch.exp(-xx.abs()))) * ne.double()
        unit = lo.kw["w_cls"] * float(terms[ok].sum()) / lo.R
        el = abs(float(losses[0]) - vals[0])
        assert el <= LOSS_C * U * unit + U * abs(vals[0]), f"{name}: cls loss {float(losses[0])} vs {vals[0]}"
        wl = max(wl, max(el - U * abs(vals[0]), 0.0) / (U * unit) if unit > 0 else 0.0)
    for q in (1, 2):
        el = abs(float(losses[q]) - vals[q])
        assert el <= LOSS_C * U * abs(vals[q]) + 1e-30, f"{name}: loss {q} {float(losses[q])} vs {vals[q]}"
        wl = max(wl, el / (U * abs(vals[q])) if vals[q] != 0 else 0.0)
    print(f"{name}: worst cls gradient {wc:.2f} u, box gradient {wb:.2f} u, loss {wl:.2f} u")
    return wc, wb


def _grid_sizes():
    N = 16384 * _sms()
    return [1, 255, 256, 257, 2047, 2048, 2049, N - 1, N, N + 1, 4 * N + 5]


GRID_IDS = ["1", "255", "256", "257", "2047", "2048", "2049", "16384S-1", "16384S", "16384S+1", "65536S+5"]
CAPPED = {"16384S-1", "16384S", "16384S+1", "65536S+5"}


@pytest.mark.parametrize("k", range(11), ids=GRID_IDS)
def test_loss_grid(k):
    n = _grid_sizes()[k]
    lo = Loss(300 + k, n, max_pos=3000 if n > 100000 else None)
    lo.up = torch.tensor([0.5, 2.0 ** 16, 0.0]) if k % 2 else torch.tensor([2.0, 0.5, 1.0])
    wc, wb = _loss_check(f"n={n}", lo)
    if GRID_IDS[k] in CAPPED:
        a, b = lo.run(), lo.run()
        assert all(_bits(u, v) for u, v in zip(a, b)), "two runs differ"


LOSS_CASES = {
    "corner_all_classes": dict(corner_class=-1),
    "corner_car": dict(corner_class=0),
    "no_corner": dict(with_corner=False),
    "code_weights_zero": dict(code_weights=[1.0, 0.5, 2.0, 0.0, 1.0, 0.25, 3.0]),
    "smooth_l1": dict(smooth_l1=True, beta=1.0 / 9.0, code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.5]),
}


@pytest.mark.parametrize("case", list(LOSS_CASES))
def test_loss_settings(case):
    lo = Loss(400 + list(LOSS_CASES).index(case), 5003)
    lo.kw.update(LOSS_CASES[case])
    lo.up = torch.tensor([0.5, 2.0, 0.25])
    wc, wb = _loss_check(case, lo)


def test_smooth_l1_at_beta():
    """|d| = beta exactly and one ulp either side: a zero target makes d exact"""
    lo = Loss(500, 3001, npos_frac=0.6)
    lo.kw.update(smooth_l1=True, beta=0.125, with_corner=False)
    pos = lo.reg_mask > 0
    lo.bt[pos] = 0.0
    vals = np.array([0.125, ulps(0.125, -1), ulps(0.125, 1)], dtype=np.float32)
    v = torch.from_numpy(np.resize(vals, (int(pos.sum()) * 7,)).reshape(-1, 7))
    v = v * torch.where(torch.rand(v.shape, generator=torch.Generator().manual_seed(1)) > 0.5, 1.0, -1.0)
    p = lo.p.clone()
    p[pos] = v.float()
    _loss_check("SmoothL1 at beta", lo, p=p)


def _corner_rows(seed, R, kind):
    """R positive, non-empty car rows, pred = 0, dyadic RoIs.  kind 'zero': pos_gt == roi (yaw >= 0, so that the yaw target is exactly
    0); 'z1': the GT moved up by exactly 1; 'tie': yaw-0 RoIs and GTs, the GT centred on the RoI's (-w / 2, -l / 2) corner, so that
    this corner (bottom and top) is equidistant from the GT corner and its flipped twin"""
    lo = Loss(seed, R, npos_frac=1.0, empty=0.0, car=1.0)
    g = torch.Generator().manual_seed(seed)
    lo.rois[:, :6] = torch.round(lo.rois[:, :6] * 64) / 64
    lo.gt = lo.rois.clone()
    if kind == "zero":
        lo.rois[:, 6] = lo.rois[:, 6].abs()
        lo.gt = lo.rois.clone()
    elif kind == "z1":
        lo.gt[:, 2] += 1.0
    else:
        lo.rois[:, 6] = 0.0
        lo.gt[:, 0] = lo.rois[:, 0] - lo.rois[:, 3] / 2
        lo.gt[:, 1] = lo.rois[:, 1] - lo.rois[:, 4] / 2
        lo.gt[:, 3:6] = torch.round(lo.rois[:, 3:6] * (0.7 + 0.6 * torch.rand(R, 3, generator=g)) * 64) / 64
        lo.gt[:, 6] = 0.0
    lo.kw.update(corner_class=-1, exact_flip=True)
    lo.up = torch.tensor([1.0, 0.5, 2.0])
    lo.targets()
    return lo, torch.zeros_like(lo.p)


def test_corner_loss_edges():
    """pred = 0 with pos_gt == roi: corner loss exactly 0 and every gradient exactly 0 (every corner distance is 0, where the gradient
    must take torch.norm's 0 rather than 0 / 0); the GT moved up by exactly 1: every distance 1, where the Huber branches meet, so the
    corner loss is exactly 0.5; a predicted corner at the GT's centre: a tie of the two distances, whose gradient torch.min splits in
    half, against the float64 reference with the flipped corners formed exactly"""
    lo, p = _corner_rows(600, 1001, "zero")
    losses, _, gp = lo.run(p=p)
    assert float(losses[2]) == 0.0 and not gp.any(), "a perfect prediction must give corner loss 0 and gradient 0"
    _loss_check("corner d = 0", lo, p=p)
    lo, p = _corner_rows(601, 1001, "z1")
    losses, _, _ = lo.run(p=p)
    assert float(losses[2]) == 0.5, float(losses[2])
    _loss_check("corner d = 1", lo, p=p)
    lo, p = _corner_rows(602, 1001, "tie")
    # the tie holds exactly in float64: the RoI corner at the GT centre is as far from the GT corner as from its reflection
    pc = RO.corners(lo.rois.double())
    gc = RO.corners(lo.gt.double())
    fc = torch.cat([2 * lo.gt.double()[:, None, :2] - gc[..., :2], gc[..., 2:]], -1)
    d1, d2 = (pc - gc).norm(dim=2), (pc - fc).norm(dim=2)
    assert int((d1 == d2).sum(1).min()) >= 2, "every row needs its two tied corners"
    _loss_check("corner tie", lo, p=p)


def test_nan_inf_and_saturated_logits():
    """+-100 logits against the float64 reference; +inf: loss inf where the soft label is below 1 (NaN at 1, 0 * inf), gradient
    scale (1 - y); -inf: loss inf where y > 0 (NaN at 0), gradient -scale y; a NaN logit: NaN loss, NaN gradient on its own row only"""
    lo = Loss(700, 4001)
    x = lo.x.clone()
    x[::5] = 100.0
    x[1::5] = -100.0
    _loss_check("+-100 logits", lo, x=x)
    ne = lo.nonempty
    for v in (INF, -INF):
        x = lo.x.clone()
        x[::3] = v
        losses, gx, _ = lo.run(x=x)
        sc = float(lo.up[0]) / lo.R
        y = lo.soft
        rows = torch.zeros(lo.R, dtype=torch.bool)
        rows[::3] = True
        want = (1 - y) * sc if v > 0 else -y * sc
        r = rows & ne
        assert torch.allclose(gx[r, 0].double(), want[r].double(), rtol=8 * U, atol=FLT_MIN), f"gradient at {v} logits"
        y0 = ((y[r] == 1.0).any() if v > 0 else (y[r] == 0.0).any())
        assert math.isnan(float(losses[0])) if y0 else float(losses[0]) == INF
    x = lo.x.clone()
    i = int(torch.nonzero(ne)[5])
    x[i] = NAN
    losses, gx, gp = lo.run(x=x)
    assert math.isnan(float(losses[0])) and torch.isfinite(losses[1:]).all()
    want = torch.zeros(lo.R, dtype=torch.bool)
    want[i] = True
    assert torch.equal(torch.isnan(gx[:, 0]), want) and not torch.isnan(gp).any()


def _loss_c_abi(lo, x, xs, p, ps, gx=None, gp=None):
    """forward + backward through the C ABI with row strides xs / ps; returns (losses, grad_cls, grad_pred)"""
    L = _L()
    d = dict(ne=lo.nonempty.to(torch.uint8).to(DEV), soft=lo.soft.to(DEV), rm=lo.reg_mask.to(DEV), bt=lo.bt.to(DEV), pg=lo.pg.to(DEV),
             lab=lo.lab.to(DEV), rois=lo.rois.to(DEV))
    ca, ra = [t.to(DEV) for t in lo.avg()]
    st = lo.cfg().struct
    losses = torch.empty(3, device=DEV)
    counts = torch.empty(2, device=DEV)
    c = L.ctx(DEV)
    common = [L.ptr(d["ne"]), L.ptr(d["soft"]), L.ptr(d["rm"]), L.ptr(d["bt"]), L.ptr(d["pg"]), L.ptr(d["lab"]), L.ptr(d["rois"]), 7, lo.R,
              L.ptr(ca), L.ptr(ra)]
    L.check(c, L.lib().sstb200_roi_head_loss_forward(c, C.byref(st), L.ptr(x), xs, L.ptr(p), ps, *common, L.ptr(losses), L.ptr(counts)))
    gx = torch.empty(lo.R, device=DEV) if gx is None else gx
    gp = torch.empty(lo.R, 7, device=DEV) if gp is None else gp
    up = lo.up.to(DEV)
    L.check(c, L.lib().sstb200_roi_head_loss_backward(c, C.byref(st), L.ptr(x), xs, L.ptr(p), ps, *common, L.ptr(counts), L.ptr(up),
                                                      L.ptr(gx), L.ptr(gp)))
    torch.cuda.synchronize()
    return losses.cpu(), gx.cpu(), gp.cpu()


def test_strided_rows_c_abi():
    """cls_score with row stride 3 and bbox_pred with row stride 9 give the contiguous call's results bit for bit"""
    lo = Loss(800, 6007)
    xb = torch.randn(lo.R, 3).float()
    xb[:, 1] = lo.x[:, 0]
    pb = torch.randn(lo.R, 9).float()
    pb[:, 2:9] = lo.p
    xb, pb = xb.to(DEV), pb.to(DEV)
    a = _loss_c_abi(lo, xb[:, 1:], 3, pb[:, 2:], 9)
    b = _loss_c_abi(lo, lo.x.to(DEV).contiguous(), 1, lo.p.to(DEV).contiguous(), 7)
    assert all(_bits(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("fill", ["nan", "ff"])
def test_loss_dirty_gradient_buffers_c_abi(fill):
    lo = Loss(900, 5001, empty=0.3)
    lo.up = torch.tensor([0.5, 2.0, 0.0])
    x, p = lo.x.to(DEV).contiguous(), lo.p.to(DEV).contiguous()
    gx, gp = torch.empty(lo.R, device=DEV), torch.empty(lo.R, 7, device=DEV)
    for t in (gx, gp):
        if fill == "nan":
            t.fill_(NAN)
        else:
            t.view(torch.uint8).fill_(0xFF)
    a = _loss_c_abi(lo, x, 1, p, 7, gx, gp)
    b = _loss_c_abi(lo, x, 1, p, 7)
    assert all(_bits(u, v) for u, v in zip(a, b))


def test_loss_no_host_sync_on_the_capped_grid():
    ops = _ops()
    lo = Loss(1000, 16384 * _sms() + 1, max_pos=2000)
    ca, ra = [t.to(DEV) for t in lo.avg()]
    ins = [lo.nonempty.to(DEV), lo.soft.to(DEV), lo.reg_mask.to(DEV), lo.bt.to(DEV), lo.pg.to(DEV), lo.lab.to(DEV), lo.rois.to(DEV)]
    cfg = lo.cfg()
    up = lo.up.to(DEV)

    def step():
        x, p = lo.x.to(DEV).requires_grad_(True), lo.p.to(DEV).requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ops.roi_head_loss(x, p, *ins, ca, ra, cfg).backward(up)
        finally:
            torch.cuda.set_sync_debug_mode("default")

    step()
    step()
    torch.cuda.synchronize()
