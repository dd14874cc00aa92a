"""GPU: the loss kernels of Anchor3DHead (sst_b200/csrc/anchor3d.cu), VoteSegHead (voteseg.cu) and SparseClusterHeadV2 / FSDV2Head
(cluster_head.cu, code sizes 8 and 10) against the float64 / CPU oracles (oracle/anchor3d_oracle.py, voteseg_oracle.py,
cluster_head_oracle.py, fsdv2_head_oracle.py), element by element, at the grid, layout and saturation edges where they could go wrong.
The three heads share heads.cuh's sig, sigmoid_focal(_grad), abs_grad, loss_grid and sum_partials, so one error model covers them.

Routes and edges
  grid      every loss pass is a grid-strided loop of 256-thread blocks, clamp(ceil(n / 2048), 1, 8 S) of them (S = the device's SM count),
            and one block adds the per-block double partials in a fixed order (more than 256 of them on the capped grid, so each thread
            adds several): n = 1, 255, 256, 257, 2047, 2048, 2049, 16384 S - 1, 16384 S, 16384 S + 1 and 65536 S + 5 (more than 8
            elements per thread) for Anchor3D's focal pass (n = B A C H W), its box / direction pass (n = B A H W), VoteSeg at C = 1 (n
            points) and the cluster heads at T = 1, C = 1 (n clusters).  On the capped grid two runs are bit-identical and no loss, forward
            or backward, syncs with the host.
  Anchor3D  A != C, H != W, B = 1 and 3 with A = 1, C = 1 and H = 1 among them; labels that vary per anchor, so that a swapped anchor /
            class or cell / slot index fails; labels -1 and C, zero label weights; upstream gradients 0.5, 2^16 and 0, a different one per
            loss; code weights (1, 0.5, 2, 0, 1, 0.25, 3); a sample with no positive inside num_total_pos; direction logits +-100 apart;
            yaw predictions equal to their target bit for bit, 2 pi away (exact in fp32) and 1 to 8 ulp away.
  VoteSeg   sigmoid focal at C = 1 and 3 with the runtime-gamma powf path at gamma 1, 1.5 and 2; softmax at C = 11, 27 and 64 (65 is
            refused); logit_scale 1.7, class weights with a 0, logit and vote rows wider than their C and 3 C columns; rows where one logit
            leads by 100 or more and rows of equal logits; invalid labels; NaN votes with valid points and with none (the latter read by
            vs_vote_nonfinite_kernel's own grid over N 3 C, the NaN in its last element).
  clusters  T = 1, 3, 6 (the Argoverse 2 groups) and 8 (9 is refused), C_t up to 64 (65 is refused); code 8 and code 10 with velocity
            weights 0 / 1 and the vel mean over 2 num_pos; per-group loss weights, per-task cls_avg / reg_avg, tasks with num_pos = 0,
            label -1 rows (NaN targets) and label C rows; an upstream gradient per (task, quantity); SmoothL1 at |d| = beta exactly and one
            ulp either side.
  special   a NaN logit reaches its own loss and gradient only (its row's under softmax); a NaN box or vote coordinate gives a NaN loss and
            a zero gradient, a NaN yaw a NaN gradient, as torch; +-inf logits follow the kernels' closed form: on the label's side loss 0
            and gradient 0, on the other loss inf and gradient NaN (mmdet's Python path gives NaN for both; include/sstb200.h says so).
  dirty     every backward's gradient buffers pre-filled with NaN and then 0xFF through the C ABI: every element is rewritten, the zero
            rows off the positives included.

Error model (u = 2^-24, every bound per element, each constant set from the worst value seen with margin)
  focal gradient   |g - g64| <= FOCAL_C u |g64| + FLT_MIN |scale|: every factor (q, s, softplus, gamma s softplus + q) is non-negative,
                   so nothing cancels and a relative bound holds at every logit; the FLT_MIN term covers underflow.  g64 is
                   oracle.voteseg_oracle.sigmoid_focal64, the same function as the oracles' focal terms with s and q both formed from
                   exp(-|x|) (tied to the oracles' autograd gradient below |x| = 15, where 1 - p still keeps its digits in float64).
  losses           focal and L1 losses are sums of non-negative terms added in double: LOSS_C u relative.  Anchor3D's yaw term can cancel,
                   so loss_bbox is held to LOSS_C u times its terms' sizes (|sin p cos t| + |cos p sin t| for the yaw).
  cross-entropy    |g_c - g64_c| <= (CE_C u ((C + 2)(p_c + [c = y]) + p_c |x_c - max x|) + FLT_MIN) |w|: the p_c |x_c - max x|
                   term is the rounding of x_c - max pushed through exp, the FLT_MIN term exp's underflow where one logit leads by 87 or
                   more; the loss within CE_LOSS_C u of the rows' summed first-order error w (|max| + |log se| + |x_y| + nll).
  L1 / SmoothL1    the fp32 difference of two fp32 values keeps its sign and is 0 only on equality, so the gradient is within L1_C u of
                   float64's (relative), and exactly 0 where the reference's is (d = 0, d NaN, off the positives).
  yaw              inside a band where the float64 |sin(p - t)| <= YAW_BAND u (|sp ct| + |cp st|) either sign (or 0) is allowed; outside
                   it the sign must agree and the value lie within YAW_C u (|cp ct| + |sp st|) |scale|; exactly 0 where p == t.
  VoteSeg's logits are compared after the kernel's fp32 product with logit_scale (a rounded __fmul_rn, as torch's fp32 x * scale).

Bounds, with the worst values seen on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the file runs in about 70 s there, most of it
in the float64 oracles at n = 65536 S + 5):
  FOCAL_C   24     focal gradient, u of |g64|                                   14.7 (cluster heads; 14.6 VoteSeg, 14.0 Anchor3D)
  LOSS_C    6      focal / L1 / box loss, u of the terms' sum                    2.6 (cluster focal loss at n = 1)
  CE_C      2      cross-entropy gradient, in units of its bound                 1.02 (Anchor3D direction, logits 100 apart)
  CE_LOSS_C 1      cross-entropy loss, u of the rows' first-order error          0.18
  L1_C      4      L1 / SmoothL1 gradient, u relative                            2.4 (SmoothL1's quadratic branch)
  YAW_BAND  8      undecided band of the yaw sign, u of the terms                (held: no sign disagreed outside it)
  YAW_C     8      yaw gradient, u of the terms                                  4.9"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import anchor3d_oracle as AO
from oracle import cluster_head_oracle as CO
from oracle import fsdv2_head_oracle as FO
from oracle import voteseg_oracle as VO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
FOCAL_C = 24.0
LOSS_C = 6.0
CE_C = 2.0
CE_LOSS_C = 1.0
L1_C = 4.0
YAW_BAND = 8.0
YAW_C = 8.0
INF = float("inf")
NAN = float("nan")


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count if torch.cuda.is_available() else 132


def _grid_sizes():
    N = 16384 * _sms()
    return [1, 255, 256, 257, 2047, 2048, 2049, N - 1, N, N + 1, 4 * N + 5]


GRID_IDS = ["1", "255", "256", "257", "2047", "2048", "2049", "16384S-1", "16384S", "16384S+1", "65536S+5"]
CAPPED = {"16384S-1", "16384S", "16384S+1", "65536S+5"}


# ---------------------------------------------------------------------------------------------------------------------------------------
# shared checks: each returns its worst error in units of its bound
# ---------------------------------------------------------------------------------------------------------------------------------------
def _bits(a, b):
    """bit-identical fp32 tensors (NaN included)"""
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _focal_grad(name, got, x64, t, scale, alpha, gamma, nan_rows=None, ref=None):
    """got: the kernel's gradient; x64: the logits as the kernel reads them; t: bool targets; scale: the float64 multiplier of each
    element's d loss / d x (broadcastable); nan_rows: elements the kernel must make NaN besides NaN logits; ref: the oracle's autograd
    gradient, tied to sigmoid_focal64 where 1 - p keeps its digits"""
    got = got.detach().cpu().double()
    scale = torch.as_tensor(scale, dtype=torch.float64).expand_as(x64)
    _, g = VO.sigmoid_focal64(x64, t, alpha, gamma)
    g = g * scale
    want_nan = torch.isnan(x64) | (torch.zeros_like(t) if nan_rows is None else nan_rows)
    assert torch.equal(torch.isnan(got), want_nan), f"{name}: NaN at {int((torch.isnan(got) != want_nan).sum())} wrong elements"
    ok = ~want_nan & torch.isfinite(x64)
    if ref is not None:
        tie = ok & (x64.abs() < 15)
        assert ((ref[tie] - g[tie]).abs() <= 1e-8 * g[tie].abs() + 1e-300).all(), f"{name}: sigmoid_focal64 departs from the oracle"
    err = (got - g).abs()[ok]
    bound = FOCAL_C * U * g.abs()[ok] + FLT_MIN * scale.abs()[ok]
    bad = err > bound
    assert not bad.any(), (f"{name}: {int(bad.sum())} focal gradients off, worst {float((err / bound)[bad].max()):.3g} of the bound at "
                           f"x = {float(x64[ok][bad][(err / bound)[bad].argmax()]):.6g}")
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _rel(name, got, ref, c, what="gradient"):
    """elementwise |got - ref| <= c u |ref|, NaN where ref is NaN and exactly 0 where ref is 0"""
    got = got.detach().cpu().double()
    ref = ref.detach().double()
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), f"{name}: NaN {what} at {int((torch.isnan(got) != torch.isnan(ref)).sum())}"
    ok = ~torch.isnan(ref)
    zero = ok & (ref == 0)
    assert (got[zero] == 0).all(), f"{name}: {int((got[zero] != 0).sum())} {what} elements nonzero where the reference is 0"
    nz = ok & (ref != 0)
    r = (got[nz] - ref[nz]).abs() / (ref[nz].abs() * U)
    worst = float(r.max()) if r.numel() else 0.0
    assert worst <= c, f"{name}: {what} off by {worst:.3g} u (bound {c})"
    return worst / c


def _loss(name, got, ref, unit, c=LOSS_C):
    """|got - ref| <= c u unit (+ the final fp32 rounding), NaN where ref is NaN"""
    got, ref = float(got), float(ref)
    if math.isnan(ref):
        assert math.isnan(got), f"{name}: loss {got}, the reference's is NaN"
        return 0.0
    bound = c * U * unit + U * abs(ref)
    err = abs(got - ref)
    assert err <= bound or got == ref, f"{name}: loss {got} against {ref}: {err / max(bound, 1e-300):.3g} of the bound"
    return err / bound if bound > 0 else 0.0


def _ce_grad(name, got, z64, y, w, ref):
    """softmax cross-entropy gradient of rows z64 [R, C] with labels y [R] and row weights w [R] against the oracle's ref"""
    got = got.detach().cpu().double()
    assert not torch.isnan(got).any(), f"{name}: NaN cross-entropy gradients"
    Cn = z64.shape[1]
    p = torch.softmax(z64, 1)
    m = z64.max(1, keepdim=True).values
    oh = torch.nn.functional.one_hot(y, Cn).double()
    bound = (CE_C * U * ((Cn + 2) * (p + oh) + p * (z64 - m).abs()) + FLT_MIN) * w.abs()[:, None]
    err = (got - ref).abs()
    bad = err > bound
    assert not bad.any(), f"{name}: {int(bad.sum())} cross-entropy gradients off, worst {float((err / bound)[bad].max()):.3g}"
    r = (err / bound)[bound > 0]
    return float(r.max()) if r.numel() else 0.0


def _ce_unit(z64, y, w):
    """the rows' summed first-order error of w (logsumexp(z) - z_y), in units of u"""
    m = z64.max(1).values
    se = torch.exp(z64 - m[:, None]).sum(1)
    zy = z64.gather(1, y[:, None])[:, 0]
    nll = m + torch.log(se) - zy
    return float((w.abs() * (m.abs() + torch.log(se).abs() + zy.abs() + nll.abs())).sum())


# ---------------------------------------------------------------------------------------------------------------------------------------
# Anchor3DHead
# ---------------------------------------------------------------------------------------------------------------------------------------
CW = [1.0, 0.5, 2.0, 0.0, 1.0, 0.25, 3.0]


class Anchor:
    """synthetic Anchor3D loss inputs on a [B, A, C, H, W] map: labels [B, H W A] in slot order (H W A) and the per-element views of
    them in the kernels' [B, A C | A 7 | A 2, H, W] layouts"""

    def __init__(self, seed, B, A, Cn, H, W, scale=6.0, pos=0.4, empty=None, lw_zero=0.1):
        g = torch.Generator().manual_seed(seed)
        self.B, self.A, self.C, self.H, self.W = B, A, Cn, H, W
        n = H * W * A
        pick = torch.rand(B, n, generator=g)
        lab = torch.randint(0, Cn, (B, n), generator=g)
        lab[pick > pos] = Cn
        lab[pick > 0.93] = -1
        if empty is not None:
            lab[empty][lab[empty] >= 0] = Cn
        self.labels = lab
        self.lw = (torch.rand(B, n, generator=g) > lw_zero).float()
        self.cls = (torch.randn(B, A * Cn, H, W, generator=g) * scale).float()
        self.reg = torch.randn(B, A * 7, H, W, generator=g).float()
        self.dir = (torch.randn(B, A * 2, H, W, generator=g) * 3).float()
        self.bt = torch.randn(B, n, 7, generator=g).float()
        self.bw = (torch.rand(B, n, 7, generator=g) > 0.1).float()
        self.dt = torch.randint(0, 2, (B, n), generator=g)
        self.dw = (torch.rand(B, n, generator=g) > 0.1).float()
        npos = ((lab >= 0) & (lab < Cn)).sum(1)
        self.ntp = int(npos.clamp(min=1).sum())

    # slot-order [B, H W A, ...] -> the kernels' [B, A K, H, W] element layout
    def grid(self, t, K=1):
        B, A, H, W = self.B, self.A, self.H, self.W
        t = t.reshape(B, H, W, A, K)
        return t.permute(0, 3, 4, 1, 2).reshape(B, A * K, H, W)

    def focal_targets(self):
        L4 = self.labels.reshape(self.B, self.H, self.W, self.A, 1)
        t = L4 == torch.arange(self.C).view(1, 1, 1, 1, self.C)
        return self.grid(t, self.C), self.grid(self.lw[..., None].expand(-1, -1, self.C).contiguous(), self.C)

    def pos(self):
        return (self.labels >= 0) & (self.labels < self.C)

    def device(self):
        return [t.to(DEV) for t in (self.labels, self.lw, self.bt, self.bw, self.dt, self.dw)] + \
            [torch.tensor(self.ntp, dtype=torch.int64, device=DEV)]


def _anchor_focal(an, upstream=1.0, loss_weight=1.0, cls=None):
    from sst_b200 import ops
    cls = an.cls if cls is None else cls
    lab, lw, *_, ntp = an.device()
    xg = cls.to(DEV).requires_grad_(True)
    loss = ops.anchor_focal_loss(xg, lab, lw, ntp, an.C, loss_weight)
    loss.backward(torch.tensor(upstream, device=DEV))
    return loss.item(), xg.grad


def _anchor_focal_check(name, an, upstream=1.0, loss_weight=1.5, cls=None, expect_nan_loss=False):
    cls = an.cls if cls is None else cls
    loss, grad = _anchor_focal(an, upstream, loss_weight, cls)
    x64 = cls.double().requires_grad_(True)
    lab = an.labels.clone()
    lab[lab < 0] = an.C                      # a label of -1 is no class, as the background C (one_hot refuses -1)
    ref = AO.focal_loss(x64, lab, an.lw, an.ntp, an.C, loss_weight)
    ref.backward(torch.tensor(upstream, dtype=torch.float64))
    t, lwe = an.focal_targets()
    scale = upstream * loss_weight / an.ntp * lwe.double()
    wg = _focal_grad(name, grad, cls.double(), t, scale, 0.25, 2.0, ref=x64.grad)
    if expect_nan_loss:
        assert math.isnan(loss), f"{name}: loss {loss} with a NaN logit"
        return wg, 0.0
    terms, _ = VO.sigmoid_focal64(cls.double(), t, 0.25, 2.0)
    wl = _loss(name, loss, ref.item(), loss_weight * float((terms * lwe).sum()) / an.ntp)
    return wg, wl


def _anchor_reg(an, up, reg=None, dr=None, w_bbox=0.75, w_dir=0.2):
    from sst_b200 import ops
    reg = an.reg if reg is None else reg
    dr = an.dir if dr is None else dr
    lab, lw, bt, bw, dt, dw, ntp = an.device()
    rg, dg = reg.to(DEV).requires_grad_(True), dr.to(DEV).requires_grad_(True)
    lb, ld = ops.anchor_reg_dir_loss(rg, dg, lab, bt, bw, dt, dw, ntp, an.C, CW, w_bbox, w_dir)
    torch.autograd.backward([lb, ld], [torch.tensor(up[0], device=DEV), torch.tensor(up[1], device=DEV)])
    return (lb.item(), ld.item()), (rg.grad, dg.grad)


def _anchor_reg_check(name, an, up=(0.5, 65536.0), reg=None, dr=None, w_bbox=0.75, w_dir=0.2):
    reg = an.reg if reg is None else reg
    dr = an.dir if dr is None else dr
    (lb, ld), (gr, gd) = _anchor_reg(an, up, reg, dr, w_bbox, w_dir)
    r64, d64 = reg.double().requires_grad_(True), dr.double().requires_grad_(True)
    # the targets in float64 too (their fp32 values exactly): the oracle then forms add_sin_difference's two products in float64 alone,
    # and a yaw equal to its target gives exactly 0, as torch's fp32 products do
    rb, rd = AO.reg_dir_loss(r64, d64, an.labels, an.bt.double(), an.bw, an.dt, an.dw, an.ntp, an.C, CW, w_bbox, w_dir)
    torch.autograd.backward([rb, rd], [torch.tensor(up[0], dtype=torch.float64), torch.tensor(up[1], dtype=torch.float64)])
    B, A, H, W = an.B, an.A, an.H, an.W
    pos = an.grid(an.pos()[..., None].float()).bool()                          # [B, A, H, W]
    gr = gr.cpu().double().reshape(B, A, 7, H, W)
    ref_r = r64.grad.reshape(B, A, 7, H, W)
    worst = {}
    worst["box"] = _rel(f"{name} box", gr[:, :, :6], ref_r[:, :, :6], L1_C)
    # yaw: undecided band, else the sign and YAW_C u of the terms
    p = reg.double().reshape(B, A, 7, H, W)[:, :, 6]
    t = an.grid(an.bt[..., 6:7].double())
    sp, cp, st, ct = torch.sin(p), torch.cos(p), torch.sin(t), torch.cos(t)
    sc = abs(up[0] * w_bbox / an.ntp) * an.grid(an.bw[..., 6:7].double()) * CW[6]
    band = (sp * ct - cp * st).abs() <= YAW_BAND * U * ((sp * ct).abs() + (cp * st).abs())
    g6, r6 = gr[:, :, 6], ref_r[:, :, 6]
    assert torch.equal(torch.isnan(g6), torch.isnan(r6)), f"{name}: NaN yaw gradients differ"
    ok = ~torch.isnan(r6)
    bound = YAW_C * U * ((cp * ct).abs() + (sp * st).abs()) * sc
    assert (g6[~pos] == 0).all(), f"{name}: yaw gradient off the positives"
    same = ok & pos & (p.float() == t.float())
    assert (g6[same] == 0).all(), f"{name}: {int((g6[same] != 0).sum())} yaw gradients nonzero where the yaw equals its target"
    out = ok & pos & ~band
    e = (g6 - r6).abs()
    bad = out & (e > bound)
    assert not bad.any(), f"{name}: {int(bad.sum())} yaw gradients off outside the band, worst {float((e / bound)[bad].max()):.3g}"
    inb = ok & pos & band & ~same
    alt = torch.minimum(e, (g6 + r6).abs())
    assert ((alt <= bound) | (g6 == 0))[inb].all(), f"{name}: in-band yaw gradients neither +-the reference nor 0"
    r = (e / bound)[out & (bound > 0)]
    worst["yaw"] = float(r.max()) if r.numel() else 0.0
    # direction cross-entropy over the positives
    gd = gd.cpu().double().reshape(B, A, 2, H, W).permute(0, 1, 3, 4, 2)
    assert (gd[~pos] == 0).all(), f"{name}: direction gradient off the positives"
    gd = gd[pos]
    rgd = d64.grad.reshape(B, A, 2, H, W).permute(0, 1, 3, 4, 2)
    z = dr.double().reshape(B, A, 2, H, W).permute(0, 1, 3, 4, 2)[pos]
    y = an.grid(an.dt[..., None]).reshape(B, A, H, W)[pos]
    wrow = up[1] * w_dir / an.ntp * an.grid(an.dw[..., None].double()).reshape(B, A, H, W)[pos]
    worst["dir"] = _ce_grad(f"{name} dir", gd, z, y, wrow, rgd[pos]) if pos.any() else 0.0
    # losses
    if pos.any():
        bw = an.grid(an.bw.double(), 7).reshape(B, A, 7, H, W) * torch.tensor(CW, dtype=torch.float64).view(1, 1, 7, 1, 1)
        d = (reg.double() - an.grid(an.bt.double(), 7)).reshape(B, A, 7, H, W)
        terms = (d[:, :, :6].abs() * bw[:, :, :6]).sum(2) + ((sp * ct).abs() + (cp * st).abs()) * bw[:, :, 6]
        unit_b = w_bbox * float(torch.nan_to_num(terms[pos], nan=0.0).sum()) / an.ntp
        wrow_l = w_dir / an.ntp * an.grid(an.dw[..., None].double()).reshape(B, A, H, W)[pos]
        worst["loss_bbox"] = _loss(f"{name} loss_bbox", lb, rb.item(), unit_b)
        worst["loss_dir"] = _loss(f"{name} loss_dir", ld, rd.item(), _ce_unit(z, y, wrow_l), CE_LOSS_C)
    else:
        assert lb == 0.0 and ld == 0.0
    return worst


ANCHOR_SHAPES = {      # B, A, C, H, W
    "B1_A6_C3_17x29": (1, 6, 3, 17, 29),
    "B3_A2_C5_29x17": (3, 2, 5, 29, 17),
    "B3_A1_C4_1x53": (3, 1, 4, 1, 53),
    "B1_A5_C1_13x7": (1, 5, 1, 13, 7),
    "B3_A3_C2_40x9": (3, 3, 2, 40, 9),
}
UPSTREAMS = [(0.5, 65536.0, 0.0), (65536.0, 0.0, 0.5), (0.0, 0.5, 65536.0)]


@pytest.mark.parametrize("shape", list(ANCHOR_SHAPES))
def test_anchor_layouts(shape):
    """per-anchor labels on maps with A != C and H != W: a swapped anchor / class or cell / slot index fails element by element; the
    upstream gradients differ per loss (0.5, 2^16, 0 in turn); sample 1 (when B = 3) has no positive"""
    B, A, Cn, H, W = ANCHOR_SHAPES[shape]
    k = list(ANCHOR_SHAPES).index(shape)
    an = Anchor(100 + k, B, A, Cn, H, W, empty=1 if B == 3 else None)
    ups = UPSTREAMS[k % 3]
    wf, wl = _anchor_focal_check(shape, an, upstream=ups[0])
    w = _anchor_reg_check(shape, an, up=ups[1:])
    print(f"anchor {shape}: focal gradient {wf:.3f}, loss {wl:.3f}, " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


@pytest.mark.parametrize("k", range(11), ids=GRID_IDS)
def test_anchor_grid(k):
    n = _grid_sizes()[k]
    an = Anchor(200 + k, 1, 1, 1, 1, n, pos=0.3)
    wf, wl = _anchor_focal_check(f"focal n={n}", an, upstream=0.5)
    w = _anchor_reg_check(f"reg n={n}", an, up=(2.0, 0.5))
    if GRID_IDS[k] in CAPPED:
        a = [_anchor_focal(an, 0.5), _anchor_focal(an, 0.5)]
        b = [_anchor_reg(an, (2.0, 0.5)), _anchor_reg(an, (2.0, 0.5))]
        assert a[0][0] == a[1][0] and torch.equal(a[0][1], a[1][1]), "focal: two runs differ"
        assert b[0][0] == b[1][0] and all(torch.equal(x, y) for x, y in zip(b[0][1], b[1][1])), "reg / dir: two runs differ"
    print(f"anchor grid n={n}: focal gradient {wf:.3f}, loss {wl:.3f}, " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


def test_anchor_saturated_logits_and_dir_margins():
    """focal logits on a fine sweep out to +-60 for both targets, direction logits +-100 apart"""
    an = Anchor(300, 1, 2, 3, 31, 37)
    x = torch.linspace(-60, 60, an.cls.numel()).float()
    an.cls = x[torch.randperm(x.numel(), generator=torch.Generator().manual_seed(1))].reshape(an.cls.shape)
    sgn = torch.where(torch.rand(an.dir.shape[0], an.A, 1, an.H, an.W, generator=torch.Generator().manual_seed(2)) > 0.5, 1.0, -1.0)
    an.dir = (an.dir.reshape(1, an.A, 2, an.H, an.W) + torch.cat([50 * sgn, -50 * sgn], 2)).reshape(an.dir.shape).float()
    wf, wl = _anchor_focal_check("saturated", an, upstream=65536.0)
    w = _anchor_reg_check("dir +-100", an, up=(1.0, 65536.0))
    print(f"anchor saturated: focal gradient {wf:.3f}, loss {wl:.3f}, dir {w['dir']:.3f}, loss_dir {w['loss_dir']:.3f}")


def _yaw_edges(an):
    """yaw predictions set against their targets at the positives: equal bit for bit, t + 2 pi exact in fp32, and 1 to 8 ulp away"""
    B, A, H, W = an.B, an.A, an.H, an.W
    g = torch.Generator().manual_seed(9)
    kinds = torch.randint(0, 4, (B, H * W * A), generator=g)
    ulps = torch.randint(1, 9, (B, H * W * A), generator=g) * torch.where(torch.rand(B, H * W * A, generator=g) > 0.5, 1, -1)
    t = an.bt[..., 6].numpy()
    p = t.copy()
    two_pi = np.float32(2 * np.pi)
    k = kinds.numpy()
    shifted = (t.astype(np.float32) + two_pi).astype(np.float32)
    exact = (shifted.astype(np.float64) - t.astype(np.float64)) == np.float64(two_pi)
    p = np.where((k == 1) & exact, shifted, p)
    bits = t.view(np.int32) + ulps.numpy().astype(np.int32)
    p = np.where(k == 2, bits.view(np.float32), p)
    p = np.where(k == 3, an.bt[..., 6].numpy() + np.float32(0.7), p).astype(np.float32)
    reg = an.reg.reshape(B, A, 7, H, W).clone()
    reg[:, :, 6] = an.grid(torch.from_numpy(p)[..., None]).reshape(B, A, H, W)
    return reg.reshape(an.reg.shape), int(((k == 1) & exact).sum()), int((k == 0).sum())


def test_anchor_yaw_equal_to_target():
    """a yaw equal to its target gets gradient 0 (a contracted sp ct - cp st leaves one product's rounding residual and a full-size
    gradient of either sign); 2 pi away falls in the undecided band"""
    an = Anchor(400, 3, 2, 3, 23, 19, pos=0.9)
    reg, n2pi, neq = _yaw_edges(an)
    assert n2pi > 50 and neq > 50
    w = _anchor_reg_check("yaw edges", an, up=(1.0, 1.0), reg=reg)
    print("anchor yaw edges: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


def test_anchor_nan_box_and_yaw():
    """a NaN box coordinate: loss_bbox NaN and gradient 0 there (torch.abs' gradient at NaN); a NaN yaw: NaN gradient; a NaN logit: NaN
    at that element only"""
    an = Anchor(500, 1, 2, 3, 11, 13, pos=0.8)
    pos = torch.nonzero(an.pos()[0])[:, 0]
    reg = an.reg.reshape(1, 2, 7, 11, 13).clone()
    for j, ch in ((0, 0), (1, 3), (2, 5)):
        hw, a = divmod(int(pos[j]), 2)
        reg[0, a, ch, hw // 13, hw % 13] = NAN
    yaw_hw, yaw_a = divmod(int(pos[3]), 2)
    reg[0, yaw_a, 6, yaw_hw // 13, yaw_hw % 13] = NAN
    reg = reg.reshape(an.reg.shape)
    (lb, ld), (gr, gd) = _anchor_reg(an, (1.0, 1.0), reg=reg)
    assert math.isnan(lb) and not math.isnan(ld)
    g = gr.cpu().reshape(1, 2, 7, 11, 13)
    for j, ch in ((0, 0), (1, 3), (2, 5)):
        hw, a = divmod(int(pos[j]), 2)
        assert g[0, a, ch, hw // 13, hw % 13].item() == 0.0, f"NaN box coordinate {ch}: gradient {g[0, a, ch, hw // 13, hw % 13].item()}"
    assert int(torch.isnan(g).sum()) == 1 and math.isnan(g[0, yaw_a, 6, yaw_hw // 13, yaw_hw % 13].item())
    _anchor_reg_check("NaN box / yaw", an, up=(1.0, 1.0), reg=reg)
    cls = an.cls.clone()
    cls[0, 4, 3, 5] = NAN
    cls[0, 0, 10, 12] = NAN
    _anchor_focal_check("NaN logit", an, cls=cls, expect_nan_loss=True)


def test_anchor_infinite_logits():
    """+-inf on the label's side: loss 0, gradient 0; on the other side: loss inf, gradient NaN"""
    an = Anchor(600, 1, 2, 2, 5, 7, pos=0.5)
    t, _ = an.focal_targets()
    an.lw.fill_(1.0)
    right = torch.where(t, INF, -INF)
    sel = torch.rand(an.cls.shape, generator=torch.Generator().manual_seed(3)) < 0.2
    cls = torch.where(sel, right, an.cls).float()
    loss, grad = _anchor_focal(an, 1.0, 1.0, cls)
    finite = torch.where(sel, torch.where(t, 1e3, -1e3), an.cls).double()
    x64 = finite.clone().requires_grad_(True)
    lab = an.labels.clone()
    lab[lab < 0] = an.C
    ref = AO.focal_loss(x64, lab, an.lw, an.ntp, an.C, 1.0)
    ref.backward()
    assert (grad.cpu()[sel] == 0).all()
    _focal_grad("inf right side", grad, finite, t, 1.0 / an.ntp, 0.25, 2.0)
    _loss("inf right side", loss, ref.item(), float(VO.sigmoid_focal64(finite, t, 0.25, 2.0)[0].sum()) / an.ntp)
    wrong = torch.where(sel, -right, an.cls).float()
    loss, grad = _anchor_focal(an, 1.0, 1.0, wrong)
    assert loss == INF, f"wrong-side inf: loss {loss}"
    assert torch.equal(torch.isnan(grad.cpu()), sel), "wrong-side inf: NaN gradients elsewhere than the infinite logits"


# ---------------------------------------------------------------------------------------------------------------------------------------
# VoteSegHead
# ---------------------------------------------------------------------------------------------------------------------------------------
LOGIT_SCALE = float(np.float32(1.7))      # the fp32 value the kernel multiplies by


class Vote:
    def __init__(self, seed, N, Cn, softmax, xs_pad=0, vs_pad=0, scale=6.0, invalid=0.0):
        g = torch.Generator().manual_seed(seed)
        self.N, self.C, self.softmax = N, Cn, softmax
        hi = Cn if softmax else Cn + 1
        self.labels = torch.randint(0, hi, (N,), generator=g)
        if invalid:
            bad = torch.rand(N, generator=g) < invalid
            self.labels[bad] = torch.where(torch.rand(N, generator=g) > 0.5, -1, hi)[bad]
        self.mask = (torch.rand(N, generator=g) < 0.6) & (self.labels >= 0) & (self.labels < Cn)
        self.vt = torch.where(self.mask[:, None], torch.randn(N, 3, generator=g), torch.zeros(N, 3)).float()
        x = torch.randn(N, Cn + xs_pad, generator=g) * scale
        if softmax and N >= 8:
            r = torch.randperm(N, generator=g)
            lead = r[: N // 8]
            x[lead, torch.randint(0, Cn, (lead.numel(),), generator=g)] += 100 + 20 * torch.rand(lead.numel(), generator=g)
            x[r[N // 8: N // 4], :Cn] = 2.5                 # rows of equal logits
        self.xbuf = x.float()
        self.vbuf = torch.randn(N, 3 * Cn + vs_pad, generator=g).float()
        self.cw = [float(v) for v in (torch.rand(Cn, generator=g) * 2)]
        self.cw[0] = 0.0

    @property
    def x(self):
        return self.xbuf[:, :self.C]

    @property
    def v(self):
        return self.vbuf[:, :3 * self.C]

    def cfg(self, gamma=2.0, alpha=0.25):
        from sst_b200 import ops
        return ops.VoteSegLossConfig(self.C, not self.softmax, gamma=gamma, alpha=alpha,
                                     class_weight=self.cw if self.softmax else None, logit_scale=LOGIT_SCALE, loss_weight=1.25,
                                     loss_weight_vote=0.75)

    def run(self, cfg, up=(0.5, 65536.0), x=None, v=None):
        """ops.voteseg_loss on the strided views of the row buffers -> (seg, vote), (grad x, grad v)"""
        from sst_b200 import ops
        xb = (self.xbuf if x is None else x).to(DEV).requires_grad_(True)
        vb = (self.vbuf if v is None else v).to(DEV).requires_grad_(True)
        xv, vv = xb[:, :self.C], vb[:, :3 * self.C]
        assert xv.stride(0) == xb.shape[1] and vv.stride(0) == vb.shape[1]
        seg, vote, _ = ops.voteseg_loss(xv, vv, self.labels.to(DEV), self.vt.to(DEV), self.mask.to(DEV), cfg)
        torch.autograd.backward([seg, vote], [torch.tensor(up[0], device=DEV), torch.tensor(up[1], device=DEV)])
        gx, gv = xb.grad[:, :self.C], vb.grad[:, :3 * self.C]
        assert not xb.grad[:, self.C:].any() and not vb.grad[:, 3 * self.C:].any()
        return (seg.item(), vote.item()), (gx, gv)


def _vote_check(name, vo, gamma=2.0, up=(0.5, 65536.0), x=None, v=None):
    cfg = vo.cfg(gamma)
    (seg, vote), (gx, gv) = vo.run(cfg, up, x, v)
    x = (vo.xbuf if x is None else x)[:, :vo.C]
    v = (vo.vbuf if v is None else v)[:, :3 * vo.C]
    xr = (x * torch.tensor(LOGIT_SCALE, dtype=torch.float32)).double()      # the kernel's rounded fp32 product
    ok = (vo.labels >= 0) & (vo.labels < (vo.C if vo.softmax else vo.C + 1))
    lab = torch.where(ok, vo.labels, torch.zeros_like(vo.labels) if vo.softmax else torch.full_like(vo.labels, vo.C))
    x64, v64 = xr.clone().requires_grad_(True), v.double().requires_grad_(True)
    kw = dict(use_sigmoid=not vo.softmax, gamma=gamma, alpha=0.25, class_weight=vo.cw if vo.softmax else None, logit_scale=1.0,
              loss_weight=1.25, loss_weight_vote=0.75)
    rs, rv = VO.losses(x64, v64, lab, vo.vt, vo.mask, **kw)
    torch.autograd.backward([rs, rv], [torch.tensor(up[0], dtype=torch.float64), torch.tensor(up[1], dtype=torch.float64)])
    w = {}
    gx = gx.cpu().double()
    if not vo.softmax:
        t = lab[:, None] == torch.arange(vo.C)[None]
        sc = up[0] * 1.25 * LOGIT_SCALE / (vo.N * vo.C)
        w["seg_grad"] = _focal_grad(name, gx, xr, t, sc, 0.25, gamma, nan_rows=~ok[:, None].expand_as(t), ref=x64.grad * LOGIT_SCALE)
        terms, _ = VO.sigmoid_focal64(xr, t, 0.25, gamma)
        if ok.all():
            w["seg_loss"] = _loss(f"{name} seg", seg, rs.item(), 1.25 * float(terms.sum()) / (vo.N * vo.C))
    else:
        assert torch.equal(torch.isnan(gx).any(1), ~ok | torch.isnan(xr).any(1))
        rows = ok & ~torch.isnan(xr).any(1)
        wr = up[0] * 1.25 * LOGIT_SCALE / vo.N * torch.tensor(vo.cw, dtype=torch.float64)[lab]
        w["seg_grad"] = _ce_grad(name, gx[rows], xr[rows], lab[rows], wr[rows], (x64.grad * LOGIT_SCALE)[rows])
        if rows.all():
            w["seg_loss"] = _loss(f"{name} seg", seg, rs.item(),
                                  _ce_unit(xr, lab, 1.25 / vo.N * torch.tensor(vo.cw, dtype=torch.float64)[lab]), CE_LOSS_C)
    if not ok.all():
        assert math.isnan(seg), f"{name}: loss_sem_seg {seg} with invalid labels"
    w["vote_grad"] = _rel(f"{name} vote", gv, v64.grad, L1_C)
    nv = int(vo.mask.sum())
    if nv:
        d = v.double().reshape(vo.N, vo.C, 3)[vo.mask][torch.arange(nv), lab[vo.mask]] - vo.vt[vo.mask].double()
        w["vote_loss"] = _loss(f"{name} vote", vote, rv.item(), 0.75 * float(torch.nan_to_num(d.abs(), nan=0.0).sum()) / (3 * nv))
    return w


VOTE_CASES = {   # C, softmax, gamma, logit row padding, vote row padding
    "sigmoid_C1_g2": (1, False, 2.0, 0, 0),
    "sigmoid_C3_g1": (3, False, 1.0, 2, 5),
    "sigmoid_C3_g1.5": (3, False, 1.5, 0, 1),
    "sigmoid_C3_g2": (3, False, 2.0, 1, 0),
    "softmax_C11": (11, True, 2.0, 3, 7),
    "softmax_C27": (27, True, 2.0, 0, 0),
    "softmax_C64": (64, True, 2.0, 1, 2),
}


@pytest.mark.parametrize("case", list(VOTE_CASES))
def test_voteseg_classes_and_strides(case):
    Cn, sm, gamma, xp, vp = VOTE_CASES[case]
    vo = Vote(700 + list(VOTE_CASES).index(case), 20011, Cn, sm, xp, vp)
    w = _vote_check(case, vo, gamma)
    print(f"voteseg {case}: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


@pytest.mark.parametrize("k", range(11), ids=GRID_IDS)
def test_voteseg_grid(k):
    n = _grid_sizes()[k]
    vo = Vote(800 + k, n, 1, False)
    w = _vote_check(f"n={n}", vo, 2.0, up=(2.0, 0.5))
    if GRID_IDS[k] in CAPPED:
        cfg = vo.cfg()
        a, b = vo.run(cfg), vo.run(cfg)
        assert a[0] == b[0] and all(torch.equal(p, q) for p, q in zip(a[1], b[1])), "two runs differ"
    print(f"voteseg grid n={n}: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


def test_voteseg_invalid_labels_nan_and_inf_logits():
    for sm in (False, True):
        Cn = 11 if sm else 3
        vo = Vote(900 + sm, 5003, Cn, sm, invalid=0.01)
        _vote_check(f"invalid labels softmax={sm}", vo)
        vo = Vote(910 + sm, 5003, Cn, sm)
        x = vo.xbuf.clone()
        x[17, 0] = NAN
        x[4001, Cn - 1] = NAN
        (seg, vote), (gx, _) = vo.run(vo.cfg(), x=x)
        assert math.isnan(seg) and not math.isnan(vote)
        want = torch.zeros(vo.N, Cn, dtype=torch.bool)
        if sm:
            want[[17, 4001]] = True
        else:
            want[17, 0] = want[4001, Cn - 1] = True
        assert torch.equal(torch.isnan(gx.cpu()), want), f"softmax={sm}: a NaN logit reaches other gradients"
    # +-inf sigmoid logits: loss 0 and gradient 0 on the label's side, inf and NaN on the other
    vo = Vote(920, 3001, 3, False)
    t = vo.labels[:, None] == torch.arange(3)[None]
    sel = torch.rand(3001, 3, generator=torch.Generator().manual_seed(4)) < 0.1
    right = torch.where(t, INF, -INF)
    x = torch.where(sel, right / LOGIT_SCALE, vo.x).float()
    (seg, _), (gx, _) = vo.run(vo.cfg(), x=x)
    assert math.isfinite(seg) and (gx.cpu()[sel] == 0).all() and not torch.isnan(gx).any()
    x = torch.where(sel, -right, vo.x).float()
    (seg, _), (gx, _) = vo.run(vo.cfg(), x=x)
    assert seg == INF and torch.equal(torch.isnan(gx.cpu()), sel)


def test_voteseg_nan_votes():
    vo = Vote(930, 4099, 3, False)
    i = int(torch.nonzero(vo.mask)[0])
    j = int(torch.nonzero(vo.mask)[1])
    v = vo.vbuf.clone()
    v[i, 3 * int(vo.labels[i]) + 1] = NAN                 # read: loss NaN, gradient 0 there
    v[j, (3 * int(vo.labels[j]) + 3) % 9] = NAN          # another class's channel: never read
    w = _vote_check("NaN votes", vo, v=v)
    (_, vote), (_, gv) = vo.run(vo.cfg(), v=v)
    assert math.isnan(vote) and not torch.isnan(gv).any() and gv[i, 3 * int(vo.labels[i]) + 1].item() == 0.0
    print("voteseg NaN votes: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))
    # no valid point: vote_preds.sum() * 0 -> NaN when any vote is not finite, read by its own grid over N 3 C (the last element here)
    n = 16384 * _sms() + 1
    vo = Vote(940, n, 1, False, scale=2.0)
    vo.mask[:] = False
    vo.vt.zero_()
    v = vo.vbuf.clone()
    (_, vote), (_, gv) = vo.run(vo.cfg(), v=v)
    assert vote == 0.0 and not gv.any()
    v[-1, -1] = NAN
    (_, vote), (_, gv) = vo.run(vo.cfg(), v=v)
    assert math.isnan(vote) and not gv.any()


def test_voteseg_refuses_65_classes():
    from sst_b200 import _lib as L
    vo = Vote(950, 64, 65, True)
    with pytest.raises(L.SSTB200Error, match="at most 64"):
        vo.run(vo.cfg())


# ---------------------------------------------------------------------------------------------------------------------------------------
# SparseClusterHeadV2 / FSDV2Head
# ---------------------------------------------------------------------------------------------------------------------------------------
LW = dict(loss_weight_cls=1.5, loss_weight_center=0.5, loss_weight_size=0.75, loss_weight_rot=0.2)


class Cluster:
    def __init__(self, seed, M, classes, code=8, smooth=False, beta=0.1, gamma=2.0, no_pos=(), scale=6.0):
        g = torch.Generator().manual_seed(seed)
        self.M, self.classes, self.code, self.T = M, list(classes), code, len(classes)
        self.kw = dict(gamma=gamma, alpha=0.25, smooth_l1=smooth, beta=float(np.float32(beta)), **LW)
        if code == 10:
            self.kw["loss_weight_vel"] = 0.3
        tc = 11 if code == 10 else 8
        self.labels, self.tg, self.x, self.r = [], [], [], []
        for t, Cn in enumerate(classes):
            pick = torch.rand(M, generator=g)
            lab = torch.randint(0, Cn, (M,), generator=g)
            lab[pick > 0.5] = Cn
            lab[pick > 0.97] = -1
            if t in no_pos:
                lab[lab >= 0] = Cn
            tg = torch.randn(M, tc, generator=g)
            if code == 10:
                tg[:, 10] = (torch.rand(M, generator=g) > 0.3).float()
            tg[lab == Cn] = 0.0
            tg[lab < 0] = NAN
            self.labels.append(lab)
            self.tg.append(tg.float())
            self.x.append((torch.randn(M, Cn, generator=g) * scale).float())
            self.r.append(torch.randn(M, code, generator=g).float())
        self.num_pos = torch.tensor([int(((lb >= 0) & (lb < Cn)).sum()) for lb, Cn in zip(self.labels, classes)])
        self.cls_avg = (torch.rand(self.T, generator=g) * 50 + 1).float()
        self.reg_avg = (torch.rand(self.T, generator=g) * 30 + 1).float()
        self.up = (torch.rand(self.T, 5 if code == 10 else 4, generator=g) * 4 + 0.25).float()

    def cfg(self):
        from sst_b200 import ops
        return ops.ClusterHeadLossConfig(**self.kw)

    def run(self, x=None):
        from sst_b200 import ops
        xs = [a.to(DEV).requires_grad_(True) for a in (self.x if x is None else x)]
        rs = [a.to(DEV).requires_grad_(True) for a in self.r]
        losses = ops.cluster_head_loss(xs, rs, [a.to(DEV) for a in self.labels], [a.to(DEV) for a in self.tg], self.num_pos.to(DEV),
                                       self.cls_avg.to(DEV), self.reg_avg.to(DEV), self.cfg())
        losses.backward(self.up.to(DEV))
        return losses.detach().cpu(), [a.grad for a in xs], [a.grad for a in rs]


def _cluster_check(name, cl, x=None):
    xin = cl.x if x is None else x
    losses, gx, gr = cl.run(x)
    x64 = [a.double().requires_grad_(True) for a in xin]
    r64 = [a.double().requires_grad_(True) for a in cl.r]
    if cl.code == 10:
        ref = FO.losses(x64, r64, cl.labels, cl.tg, cl.num_pos, cl.cls_avg, cl.reg_avg, **cl.kw)
    else:
        ref = CO.losses(x64, r64, cl.labels, cl.tg, cl.num_pos, cl.cls_avg, cl.reg_avg, **cl.kw)
    ref.backward(cl.up.double())
    w = {"cls_grad": 0.0, "reg_grad": 0.0, "cls_loss": 0.0, "reg_loss": 0.0}
    for t, Cn in enumerate(cl.classes):
        lab = cl.labels[t]
        tt = lab[:, None] == torch.arange(Cn)[None]
        sc = float(cl.up[t, 0]) * LW["loss_weight_cls"] / float(cl.cls_avg[t])
        nan_rows = (lab < 0)[:, None].expand_as(tt)
        w["cls_grad"] = max(w["cls_grad"], _focal_grad(f"{name} task {t} cls", gx[t], xin[t].double(), tt, sc, 0.25, cl.kw["gamma"],
                                                       nan_rows=nan_rows, ref=x64[t].grad))
        w["reg_grad"] = max(w["reg_grad"], _rel(f"{name} task {t} reg", gr[t], r64[t].grad, L1_C))
        if int(cl.num_pos[t]) == 0:
            assert not gr[t].any() and (losses[t, 1:] == 0).all()
        if (lab < 0).any():
            assert math.isnan(float(losses[t, 0]))
        else:
            terms, _ = VO.sigmoid_focal64(xin[t].double(), tt, 0.25, cl.kw["gamma"])
            unit = LW["loss_weight_cls"] * float(terms.sum()) / float(cl.cls_avg[t])
            w["cls_loss"] = max(w["cls_loss"], _loss(f"{name} task {t} cls", losses[t, 0], ref[t, 0].item(), unit))
        for q in range(1, losses.shape[1]):
            w["reg_loss"] = max(w["reg_loss"], _loss(f"{name} task {t} q{q}", losses[t, q], ref[t, q].item(), abs(ref[t, q].item())))
    return w


CLUSTER_CASES = {    # classes per task, code size, SmoothL1, gamma, tasks without positives
    "T1_C1_code8": ([1], 8, False, 2.0, ()),
    "T3_code8_smooth": ([1, 2, 3], 8, True, 2.0, (1,)),
    "T6_argo_smooth_g1": ([4, 5, 4, 5, 4, 4], 8, True, 1.0, (3,)),
    "T8_C64_code8": ([64, 1, 7, 2, 33, 3, 5, 9], 8, False, 2.0, (2, 6)),
    "T3_code10": ([1, 2, 2], 10, False, 2.0, (2,)),
    "T6_code10_smooth": ([1, 2, 2, 1, 2, 2], 10, True, 2.0, (0,)),
}


@pytest.mark.parametrize("case", list(CLUSTER_CASES))
def test_cluster_tasks_and_codes(case):
    classes, code, smooth, gamma, no_pos = CLUSTER_CASES[case]
    cl = Cluster(1000 + list(CLUSTER_CASES).index(case), 3001, classes, code, smooth, 0.1, gamma, no_pos)
    w = _cluster_check(case, cl)
    print(f"cluster {case}: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


@pytest.mark.parametrize("k", range(11), ids=GRID_IDS)
def test_cluster_grid(k):
    n = _grid_sizes()[k]
    cl = Cluster(1100 + k, n, [1], 10 if k % 2 else 8)
    w = _cluster_check(f"n={n}", cl)
    if GRID_IDS[k] in CAPPED:
        a, b = cl.run(), cl.run()
        assert _bits(a[0], b[0]) and all(_bits(p, q) for p, q in zip(a[1] + a[2], b[1] + b[2])), "two runs differ"
    print(f"cluster grid n={n}: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


def test_cluster_smooth_l1_at_beta():
    """|d| = beta exactly and one ulp either side, with a zero target so that d is exact"""
    beta = 0.1
    b32 = np.float32(beta)
    vals = np.array([b32, np.nextafter(b32, np.float32(0)), np.nextafter(b32, np.float32(1))], dtype=np.float32)
    cl = Cluster(1200, 600, [2, 1], 10, True, beta)
    for t in range(2):
        pos = (cl.labels[t] >= 0) & (cl.labels[t] < cl.classes[t])
        cl.tg[t][pos, :10] = 0.0
        v = torch.from_numpy(np.resize(vals, (int(pos.sum()) * 10,)).reshape(-1, 10))
        v = v * torch.where(torch.rand(v.shape, generator=torch.Generator().manual_seed(t)) > 0.5, 1.0, -1.0)
        cl.r[t][pos] = v.float()
    w = _cluster_check("SmoothL1 at beta", cl)
    print("cluster SmoothL1 at beta: " + ", ".join(f"{a} {b:.3f}" for a, b in w.items()))


def test_cluster_nan_and_inf_logits_and_refusals():
    from sst_b200 import _lib as L
    cl = Cluster(1300, 2001, [3, 2], 8)
    x = [a.clone() for a in cl.x]
    x[0][5, 1] = NAN
    x[1][1999, 0] = NAN
    losses, gx, _ = cl.run(x)
    for t, (i, c) in enumerate(((5, 1), (1999, 0))):
        assert math.isnan(float(losses[t, 0]))
        want = (cl.labels[t] < 0)[:, None].expand_as(x[t]).clone()
        want[i, c] = True
        assert torch.equal(torch.isnan(gx[t].cpu()), want), f"task {t}: a NaN logit reaches other gradients"
    for t in range(2):
        cl.labels[t][cl.labels[t] < 0] = cl.classes[t]
        cl.tg[t] = torch.nan_to_num(cl.tg[t], nan=0.0)
    tts = [cl.labels[t][:, None] == torch.arange(c)[None] for t, c in enumerate(cl.classes)]
    sel = [torch.rand(a.shape, generator=torch.Generator().manual_seed(5 + t)) < 0.1 for t, a in enumerate(cl.x)]
    right = [torch.where(sel[t], torch.where(tts[t], INF, -INF), cl.x[t]).float() for t in range(2)]
    losses, gx, _ = cl.run(right)
    assert torch.isfinite(losses).all() and all((g.cpu()[s] == 0).all() and not torch.isnan(g).any() for g, s in zip(gx, sel))
    wrong = [torch.where(sel[t], torch.where(tts[t], -INF, INF), cl.x[t]).float() for t in range(2)]
    losses, gx, _ = cl.run(wrong)
    assert (losses[:, 0] == INF).all() and all(torch.equal(torch.isnan(g.cpu()), s) for g, s in zip(gx, sel))
    with pytest.raises(L.SSTB200Error, match="at most 8"):
        Cluster(1301, 64, [1] * 9).run()
    with pytest.raises(L.SSTB200Error, match="at most 64"):
        Cluster(1302, 64, [65]).run()


# ---------------------------------------------------------------------------------------------------------------------------------------
# every backward rewrites dirty gradient buffers; no loss syncs with the host on the capped grid
# ---------------------------------------------------------------------------------------------------------------------------------------
def _fill(ts, fill):
    for t in ts:
        if fill == "nan":
            t.fill_(NAN)
        else:
            t.view(torch.uint8).fill_(0xFF)


@pytest.mark.parametrize("fill", ["nan", "ff"])
def test_dirty_gradient_buffers_c_abi(fill):
    from sst_b200 import _lib as L
    from sst_b200 import ops
    c = L.ctx(DEV)
    # Anchor3D: the positives' channels and the zero channels off them
    an = Anchor(1400, 3, 2, 3, 9, 11, empty=1)
    lab, lw, bt, bw, dt, dw, ntp = an.device()
    _, ref_f = _anchor_focal(an, 0.5, 1.5)
    (_, _), (ref_r, ref_d) = _anchor_reg(an, (0.5, 2.0))
    x, r, d = an.cls.to(DEV), an.reg.to(DEV), an.dir.to(DEV)
    gf, gr, gd = torch.empty_like(x), torch.empty_like(r), torch.empty_like(d)
    _fill([gf, gr, gd], fill)
    dims = (an.B, an.A, an.C, an.H, an.W)
    L.check(c, L.lib().sstb200_anchor_focal_loss_backward(c, L.ptr(x), *dims, L.ptr(lab), L.ptr(lw), L.ptr(ntp), 1.5,
                                                          L.ptr(torch.tensor([0.5], device=DEV)), L.ptr(gf)))
    gl = torch.tensor([0.5, 2.0], device=DEV)
    L.check(c, L.lib().sstb200_anchor_reg_dir_loss_backward(c, L.ptr(r), L.ptr(d), an.B, an.A, an.C, an.H, an.W, L.ptr(lab), L.ptr(bt),
                                                            L.ptr(bw), L.ptr(dt), L.ptr(dw), L.arr(C.c_float, CW), L.ptr(ntp), 0.75, 0.2,
                                                            L.ptr(gl), L.ptr(gr), L.ptr(gd)))
    torch.cuda.synchronize()
    assert all(_bits(a, b) for a, b in ((gf, ref_f), (gr, ref_r), (gd, ref_d)))
    # VoteSeg (strided rows)
    vo = Vote(1401, 3001, 3, False, 1, 2)
    cfg = vo.cfg()
    _, (ref_x, ref_v) = vo.run(cfg, (0.5, 2.0))
    xb, vb = vo.xbuf.to(DEV), vo.vbuf.to(DEV)
    labd, vtd, md = vo.labels.to(DEV), vo.vt.to(DEV), vo.mask.to(DEV).view(torch.uint8)
    losses = torch.empty(2, device=DEV)
    nvalid = torch.empty((), dtype=torch.int64, device=DEV)
    counts = torch.empty(1, dtype=torch.int64, device=DEV)
    st, keep = cfg.struct()
    L.check(c, L.lib().sstb200_voteseg_loss_forward(c, C.byref(st), L.ptr(xb), xb.stride(0), L.ptr(vb), vb.stride(0), vo.N, L.ptr(labd),
                                                    L.ptr(vtd), L.ptr(md), L.ptr(losses), L.ptr(nvalid), L.ptr(counts)))
    gx, gv = torch.empty(vo.N, 3, device=DEV), torch.empty(vo.N, 9, device=DEV)
    _fill([gx, gv], fill)
    L.check(c, L.lib().sstb200_voteseg_loss_backward(c, C.byref(st), L.ptr(xb), xb.stride(0), L.ptr(vb), vb.stride(0), vo.N, L.ptr(labd),
                                                     L.ptr(vtd), L.ptr(md), L.ptr(nvalid), L.ptr(torch.tensor([0.5, 2.0], device=DEV)),
                                                     L.ptr(gx), L.ptr(gv)))
    torch.cuda.synchronize()
    assert _bits(gx, ref_x) and _bits(gv, ref_v)
    del keep
    # cluster heads, code 8 and 10
    for code in (8, 10):
        cl = Cluster(1402 + code, 2003, [2, 3, 1], code, no_pos=(1,))
        _, ref_x, ref_r = cl.run()
        xs, rs = [a.to(DEV) for a in cl.x], [a.to(DEV) for a in cl.r]
        labs, tgs = [a.to(DEV) for a in cl.labels], [a.to(DEV) for a in cl.tg]
        np_, ca, ra, up = cl.num_pos.to(DEV), cl.cls_avg.to(DEV), cl.reg_avg.to(DEV), cl.up.to(DEV).contiguous()
        gxs, grs = [torch.empty_like(a) for a in xs], [torch.empty_like(a) for a in rs]
        _fill(gxs + grs, fill)
        cfgc = cl.cfg()
        st = cfgc.struct_ex() if code == 10 else cfgc.struct()
        fn = L.lib().sstb200_cluster_head_loss_backward_ex if code == 10 else L.lib().sstb200_cluster_head_loss_backward
        L.check(c, fn(c, C.byref(st), cl.T, cl.M, ops._ptrs(xs), L.arr(C.c_int64, [a.stride(0) for a in xs]),
                      L.arr(C.c_int32, cl.classes), ops._ptrs(rs), L.arr(C.c_int64, [a.stride(0) for a in rs]), ops._ptrs(labs),
                      ops._ptrs(tgs), L.ptr(np_), L.ptr(ca), L.ptr(ra), L.ptr(up), ops._ptrs(gxs), ops._ptrs(grs)))
        torch.cuda.synchronize()
        for a, b in zip(gxs + grs, list(ref_x) + list(ref_r)):
            assert _bits(a, b), f"code {code}: a gradient element differs from a clean call"


def test_no_host_sync_on_the_capped_grid():
    from sst_b200 import ops
    n = 16384 * _sms() + 1
    an = Anchor(1500, 1, 1, 1, 1, n)
    vo = Vote(1501, n, 1, False)
    cl = Cluster(1502, n, [1], 10)
    lab, lw, bt, bw, dt, dw, ntp = an.device()
    xs = [an.cls.to(DEV).requires_grad_(True), an.reg.to(DEV).requires_grad_(True), an.dir.to(DEV).requires_grad_(True),
          vo.x.to(DEV).requires_grad_(True), vo.v.to(DEV).requires_grad_(True), cl.x[0].to(DEV).requires_grad_(True),
          cl.r[0].to(DEV).requires_grad_(True)]
    vargs = [vo.labels.to(DEV), vo.vt.to(DEV), vo.mask.to(DEV)]
    cargs = [[cl.labels[0].to(DEV)], [cl.tg[0].to(DEV)], cl.num_pos.to(DEV), cl.cls_avg.to(DEV), cl.reg_avg.to(DEV)]
    vcfg, ccfg = vo.cfg(), cl.cfg()
    ups = [torch.ones((), device=DEV) for _ in range(5)] + [cl.up.to(DEV)]

    def step():
        lc = ops.anchor_focal_loss(xs[0], lab, lw, ntp, 1, 1.0)
        lb, ld = ops.anchor_reg_dir_loss(xs[1], xs[2], lab, bt, bw, dt, dw, ntp, 1, CW, 1.0, 1.0)
        seg, vote, _ = ops.voteseg_loss(xs[3], xs[4], *vargs, vcfg)
        lcl = ops.cluster_head_loss([xs[5]], [xs[6]], *cargs, ccfg)
        torch.autograd.backward([lc, lb, ld, seg, vote, lcl], ups)

    step()                      # the first call binds the library and builds its context
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
