"""GPU: FSD's SIR layer (csrc/sir.cu, sir_bf16.cu, sir_train.cu) against float64 on every route, tile edge and dirty workspace.

sstb200_sir_layer_forward_ex / _forward_train / _backward run one of three routes that share nothing past the group CSR:
    fp32 eval   sir_rel_gate_kernel (warp per point), gemm_rows_kernel (128 x 64 tiles, K step 16), add_norm_kernel and
                segmax_sorted_kernel (64-row CSR chunks, atomicMax on the float bits at chunk edges)
    fp32 train  the same forward with its state, then sirb_ln_act_bwd_kernel, sirb_dw_kernel (64 x 64 tiles, 16-row steps, an fp64
                flush every 64 rows, row splits) and sirb_rel_bwd_kernel
    bf16 eval   sir_a_kernel / sir_b_kernel: persistent wgmma kernels over 128-point tiles in CSR order, grid min(tiles, SMs), ids
                prefetched one tile ahead, warp_segmax_ord (one pass per distinct group in a warp), KP = 128 or 192
The cases put group edges on CSR positions 31|32, 63|64, 127|128 and 128|129, run 32 distinct groups per warp, one group over
three tiles, the group_csr switch at G = 4096 | 4097, CSR given and built in the call, point counts on both sides of the 64-row
chunk and 128-row tile and up to a third pass of the persistent loop, and a G larger than the ids used (empty groups must pool
to exactly 0, as torch_scatter gives).  Every width the routes accept is run, and the ones they refuse must raise.

Each eval case first runs a "poison twin" on the same context (weights and features x 1e4, another G), then the real call twice
into outputs prefilled with a sentinel that has 16 guard rows past N and past G: the guard rows must keep it and the two calls
must agree bit for bit.

Error metric: a max-norm check beside a PER-ROW bound
    max_c |got - ref|  <=  tol * max_c mag  (+ max_c dev on the bf16 route)
where mag is the float64 magnitude propagated through the layer: a Linear gives |X| |W|^T, a LayerNorm |gamma| rstd64 (mag + max
over the row of mag) + |beta|, an activation multiplies by its Lipschitz bound, the gating gives |x| mag_rel, pooling takes the
group max of mag, and layer 1 takes [mag_p0 || mag_g0[inv]].  dev carries the bf16 route's tanh GELU (<= 5e-4 + 2^-12 |x| from
the erf form, MUFU.TANH included) through the same maps without the |beta| term.  That propagation is worst-case: each
Linear + LayerNorm multiplies the slack by about 2 sqrt(K), so after five layers mag exceeds the values by 1e5..1e6 and the
tolerances come from measurement on an H100 80GB HBM3 (700 W): worst err / mag over every case here 1.3e-9 on the fp32
routes (4.4e-10 without the shift cases) and 2.4e-7 on bf16, against tolerances of 5e-9 and 1e-6.  The max-norm check is 1e-4 (fp32) and 1e-2 (bf16; 3e-2 for
cin < 16, 2.1e-2 measured at cin 3).

Gradients (training route) against float64 autograd, per row of grad_feats and grad_f_cluster and per output channel of every
parameter gradient:  err <= GRAD_TOL (|ref row|_inf + 1e-3 |ref|_inf).  The inputs are built so that no (group, channel) has its
two largest float64 values within 1e-4 relative of each other (_separate_ties moves each runner-up point into a group of its
own and the property is asserted): otherwise an fp32 / float64 arg-max flip moves whole gradient terms.  GRAD_TOL = 1e-3; the
worst measured err / (|ref row|_inf + 1e-3 |ref|_inf) on the same H100 is 4.1e-4, for LayerNorm parameter gradients, and it is
the same at 64 rows as at 150 000: the fp32 partial sums of those gradients do not limit them.

Shift cases: a common part about 1000 times the spread of the rel-MLP's last pre-LayerNorm outputs (cin 8, 84, 127, 133) or an
offset of about 1024 in both VFE layers' pre-LayerNorm rows (forward on all three routes; the gradients of that layer are
cancelling sums of terms ~1000 x their result, which fp32 cannot pin to float64).  The shared part enters through weights that are exact in bf16, so
the shifted layer computes the same function as the unshifted one; its bound is the unshifted layer's bound plus the fp32
tolerance of the shifted layer's own magnitude.  With the bf16 rel-MLP LayerNorm's variance taken over all KP columns less
(KP - cin) mean^2 (the form before this test), the cin 8, 84 and 133 cases fail their max-norm check at 1.14, 1.6e-2 and
2.2e-2; cin 127 (one pad column) passes.  The max-norm for shift cases is 1e-2 on both routes, since the fp32 route rounds the
shared part at fp32 precision (1.5e-3 measured).
"""
import copy
import ctypes as C
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

NZ = [20.0, 20.0, 4.0]
EPS = 1e-3
SCALER = 10.0
# mag is a worst-case (triangle-inequality) magnitude: through five stacked Linear + LayerNorm layers it exceeds the values by
# 1e5..1e6, so the per-row tolerances are set from measurement (worst err / mag on an H100: fp32 1.3e-9, bf16 2.4e-7)
ROW_TOL = {"fp32": 5e-9, "bf16": 1e-6}
MAX_TOL = {"fp32": 1e-4, "bf16": 1e-2}
MAX_TOL_NARROW_BF16 = 3e-2  # cin < 16: layer 0 has rank <= cin, no averaging over K (2.1e-2 measured at cin 3)
MAX_TOL_SHIFT = 1e-2  # the fp32 route rounds a shared part ~1000 x the spread at fp32 precision (1.5e-3 measured)
DEV_UNIT = 5e-3  # the tanh GELU's deviation enters mag in units of bf16 rounding
GRAD_TOL = 1e-3  # worst measured 4.1e-4 (a LayerNorm bias gradient; the same at 64 and 150 000 rows)
TIE_REL = 1e-4
LIP = {"relu": 1.0, "gelu": 1.13}  # max |GELU'| = 1.1289
SENTINEL = 1e30
GUARD = 16
POISON = 1e4


# ----------------------------------------------------------------------------------------------------------------------
# layer, inputs and group layouts
# ----------------------------------------------------------------------------------------------------------------------
def _layer(cin, feats=(128, 128), rel_dims=(16, 32), rel_in=3, act="gelu", seed=0):
    """SIRLayer (LN, max) with LayerNorm weights 1 + N(0, 0.2) and biases N(0, 0.2); rel_dims are the hidden widths (cin is added)"""
    from sst_b200.sir_modules import SIRLayer
    torch.manual_seed(seed)
    m = SIRLayer(in_channels=cin, feat_channels=list(feats), rel_mlp_hidden_dims=list(rel_dims), rel_mlp_in_channel=rel_in,
                 norm_cfg=dict(type="LN", eps=EPS), mode="max", return_point_feats=True, rel_dist_scaler=SCALER, xyz_normalizer=NZ,
                 act=act)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if n_.endswith(".1.weight") or "norm.weight" in n_ else 0.0))
    return m.eval()


def _inputs(N, cin, rel_in, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, generator=g)
    x[:, :3] *= 10
    return x, torch.randn(N, rel_in, generator=g) * 2


def _random_counts(seed, total, lo, hi):
    g = np.random.default_rng(seed)
    out = []
    while sum(out) < total:
        out.append(int(g.integers(lo, hi + 1)))
    out[-1] -= sum(out) - total
    return out


@functools.lru_cache(maxsize=None)
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n(spec):
    """point counts: ints, or tile counts in terms of the SM count (the bf16 grid is min(tiles, SMs))"""
    if isinstance(spec, int):
        return spec
    return {"S128": 128 * _sms(), "S128+1": 128 * _sms() + 1, "2S128+37": 2 * 128 * _sms() + 37}[spec]


EDGE = [3, 29, 1, 31, 63, 1, 1]  # CSR group ends at 3, 32, 33, 64, 127, 128, 129
assert np.cumsum(EDGE).tolist() == [3, 32, 33, 64, 127, 128, 129]
SPAN3 = [1, 300, 1, 1, 2, 1, 90, 1, 1, 40]  # CSR positions 1..300: one group over tiles 0, 1 and 2


def _counts(layout, N, seed):
    """points per group in group-id (CSR) order; zeros are empty groups"""
    if layout == "one":
        return [N]
    if layout == "distinct":
        return [1] * N
    if layout == "random":  # sizes 0..12: empty groups between occupied ones
        return _random_counts(seed, N, 0, 12)
    if layout == "edges":
        return EDGE + _random_counts(seed, N - sum(EDGE), 1, 9)
    if layout == "span3":
        return SPAN3 + _random_counts(seed, N - sum(SPAN3), 1, 4)
    if layout in ("g4096", "g4097"):  # with the 3 trailing empty groups _groups adds, G = 4096 | 4097
        ng = int(layout[1:]) - 3
        return [1 + (i * 7919 + seed) % 3 for i in range(ng)]
    raise ValueError(layout)


def _groups(counts, seed, extra=3):
    """inv [N] int64 in random point order (CSR order differs from point order) and G = len(counts) + extra trailing empty groups"""
    g = torch.Generator().manual_seed(seed)
    inv = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    inv = inv[torch.randperm(inv.numel(), generator=g)]
    return inv.contiguous(), len(counts) + extra


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference and magnitudes
# ----------------------------------------------------------------------------------------------------------------------
def _w64(m, grad=False):
    return {"x." + k: v.detach().double().cpu().clone().requires_grad_(grad) for k, v in m.state_dict().items()}


def _reference(m, x, fcl, inv, G, shortcut):
    return O.sir_layer_forward(x.double(), inv, G, fcl.double(), _w64(m), "x.", len(m.rel_dims), m.num_vfe, NZ, EPS, m.act, SCALER,
                               with_shortcut=shortcut)


def _pool(v, inv, G):
    return torch.zeros((G, v.shape[1]), dtype=v.dtype).scatter_reduce(0, inv[:, None].expand_as(v), v, "amax", include_self=False)


def _magnitudes(m, x, fcl, inv, G, shortcut, tanh_gelu):
    """(mag_point, mag_group, dev_point, dev_group) in float64, and the post-activation rows of each VFE layer"""
    w = _w64(m)
    x, f = x.double(), fcl.double() / SCALER
    lip = LIP[m.act]
    act = F.gelu if m.act == "gelu" else F.relu
    gelu_dev = tanh_gelu and m.act == "gelu"

    def layer(h, mg, dv, W, gam, bet):
        t, mg, dv = h @ W.T, mg @ W.abs().T, dv @ W.abs().T
        mu = t.mean(1, keepdim=True)
        r = 1.0 / torch.sqrt(((t - mu) ** 2).mean(1, keepdim=True) + EPS)
        y = (t - mu) * r * gam + bet
        mg = gam.abs() * r * (mg + mg.amax(1, keepdim=True)) + bet.abs()
        dv = gam.abs() * r * (dv + dv.amax(1, keepdim=True))
        dv = lip * dv + ((5e-4 + 2.5e-4 * y.abs()) if gelu_dev else 0.0)
        return act(y), lip * mg, dv

    h, mg, dv = f, f.abs(), torch.zeros_like(f)
    for k in range(len(m.rel_dims)):
        h, mg, dv = layer(h, mg, dv, w[f"x.rel_mlp.{k}.0.weight"], w[f"x.rel_mlp.{k}.1.weight"], w[f"x.rel_mlp.{k}.1.bias"])
    xn = torch.cat([x[:, :3] / torch.tensor(NZ, dtype=torch.float64), x[:, 3:]], 1)
    h, mg, dv = xn * h, xn.abs() * mg, xn.abs() * dv
    mgs, dvs, posts = [], [], []
    for i in range(m.num_vfe):
        p = f"x.vfe_layers.{i}."
        h, mg, dv = layer(h, mg, dv, w[p + "linear.weight"], w[p + "norm.weight"], w[p + "norm.bias"])
        posts.append(h)
        gh, gm, gd = _pool(h, inv, G), _pool(mg, inv, G), _pool(dv, inv, G)
        mgs.append(gm)
        dvs.append(gd)
        h, mg, dv = torch.cat([h, gh[inv]], 1), torch.cat([mg, gm[inv]], 1), torch.cat([dv, gd[inv]], 1)
    C = m.feat_channels[-1]
    mg, dv = mg[:, :C], dv[:, :C]
    if shortcut and x.shape[1] - 3 == C:
        mg = mg + x[:, 3:].abs()
    return mg, torch.cat(mgs, 1), dv, torch.cat(dvs, 1), posts


def _row_check(got, ref, mag, tol, tol_max, what):
    """per-row bound tol * max_c mag and max-norm; returns the worst err / max_c mag"""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    if ref.numel() == 0:
        return 0.0
    err = (got - ref).abs().amax(1)
    b = tol * mag.amax(1)
    bad = torch.nonzero(err > b).flatten()
    if bad.numel():
        k = int(bad[torch.argmax(err[bad] / b[bad])])
        raise AssertionError(f"{what}: {bad.numel()} of {err.numel()} rows beyond the bound; worst row {k}: err {err[k].item():.3e} "
                             f"bound {b[k].item():.3e}")
    rel = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
    assert rel < tol_max, f"{what}: max-norm error {rel:.3e}"
    nz = b > 0
    return float((err[nz] / b[nz]).max()) * tol if bool(nz.any()) else 0.0


# ----------------------------------------------------------------------------------------------------------------------
# C entry points
# ----------------------------------------------------------------------------------------------------------------------
_PREC = {"fp32": 0, "bf16": 1}


def _struct(m, shortcut):
    s = m._struct()
    s.with_shortcut = int(shortcut)
    return s


def _eval_call(m, x, fcl, inv, G, precision, shortcut, csr=None):
    """sstb200_sir_layer_forward_ex into outputs with GUARD sentinel rows past N and G"""
    from sst_b200 import _lib as L
    N, dev = x.shape[0], x.device
    pbuf = torch.full((N + GUARD, m.feat_channels[-1]), SENTINEL, device=dev)
    gbuf = torch.full((G + GUARD, sum(m.feat_channels)), SENTINEL, device=dev)
    off, order = csr if csr is not None else (None, None)
    s = _struct(m, shortcut)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_sir_layer_forward_ex(c, C.byref(s), x.data_ptr(), 0, 0, 0, fcl.data_ptr(), inv.data_ptr(), N, G,
                                                     L.ptr(off), L.ptr(order), _PREC[precision], pbuf.data_ptr(), 0, gbuf.data_ptr()))
    torch.cuda.synchronize()
    return pbuf, gbuf


def _train_call(m, x, fcl, inv, G, shortcut, csr=None):
    """sstb200_sir_layer_forward_train into sentinel-guarded outputs"""
    from sst_b200 import _lib as L
    N, dev = x.shape[0], x.device
    pbuf = torch.full((N + GUARD, m.feat_channels[-1]), SENTINEL, device=dev)
    gbuf = torch.full((G + GUARD, sum(m.feat_channels)), SENTINEL, device=dev)
    off, order = csr if csr is not None else (None, None)
    s = _struct(m, shortcut)
    nbytes = L.lib().sstb200_sir_layer_train_state_bytes(C.byref(s), N, G)
    state = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_sir_layer_forward_train(c, C.byref(s), x.data_ptr(), fcl.data_ptr(), inv.data_ptr(), N, G, L.ptr(off),
                                                        L.ptr(order), pbuf.data_ptr(), gbuf.data_ptr(), state.data_ptr(), nbytes))
    torch.cuda.synchronize()
    return pbuf, gbuf


def _poison_twin(m):
    t = copy.deepcopy(m)
    with torch.no_grad():
        for p in t.parameters():
            p.mul_(POISON)
    return t


def _check_forward(cuda, m, x, fcl, inv, G, route, shortcut=False, csr=False, bound_model=None, max_tol=None):
    """poison twin, two calls (bit-identical), guard rows, exact zeros for empty groups, per-row bound against float64.
    bound_model: the layer whose magnitudes bound the error at the route's precision (shift cases); m's own at fp32 is added."""
    from sst_b200.sir_modules import group_csr
    precision = "bf16" if route == "bf16" else "fp32"
    call = (lambda mm, xx, GG, cc: _train_call(mm, xx, fcl_d, inv_d, GG, shortcut, cc)) if route == "train" else \
        (lambda mm, xx, GG, cc: _eval_call(mm, xx, fcl_d, inv_d, GG, precision, shortcut, cc))
    N = x.shape[0]
    m = m.to(cuda)
    x_d, fcl_d, inv_d = x.to(cuda).contiguous(), fcl.to(cuda).contiguous(), inv.to(cuda).contiguous()
    twin = _poison_twin(m)
    call(twin, x_d * POISON, G + 37, None)
    cs = group_csr(inv_d, G) if csr else None
    pa, ga = call(m, x_d, G, cs)
    pb, gb = call(m, x_d, G, cs)
    assert torch.equal(pa, pb) and torch.equal(ga, gb), "two identical calls differ"
    assert bool((pa[N:] == SENTINEL).all()), "point rows past N were written"
    assert bool((ga[G:] == SENTINEL).all()), "group rows past G were written"
    empty = torch.bincount(inv, minlength=G) == 0
    assert bool((ga[:G][empty.to(cuda)] == 0).all()), "an empty group's row is not exactly 0"
    pref, gref = _reference(m.cpu(), x, fcl, inv, G, shortcut)
    mp, mg, dp, dg, _ = _magnitudes(bound_model if bound_model is not None else m.cpu(), x, fcl, inv, G, shortcut, route == "bf16")
    tol = ROW_TOL[precision]
    mp, mg = mp + dp / DEV_UNIT, mg + dg / DEV_UNIT
    if bound_model is not None:
        mp2, mg2, _, _, _ = _magnitudes(m.cpu(), x, fcl, inv, G, shortcut, False)
        mp, mg = mp + ROW_TOL["fp32"] / tol * mp2, mg + ROW_TOL["fp32"] / tol * mg2
    if max_tol is None:
        max_tol = MAX_TOL_NARROW_BF16 if precision == "bf16" and m.in_channels < 16 else MAX_TOL[precision]
    rp = _row_check(pa[:N], pref, mp, tol, max_tol, f"{route} point")
    rg = _row_check(ga[:G], gref, mg, tol, max_tol, f"{route} group")
    print(f"[sir-edges] {route} N={N} G={G} worst err/mag: point {rp:.3g} group {rg:.3g}")
    return pa[:N], ga[:G]


# ----------------------------------------------------------------------------------------------------------------------
# gradients
# ----------------------------------------------------------------------------------------------------------------------
def _near_ties(post, inv, G, tie_rel):
    """rows that are the runner-up of a (group, channel) whose two largest values lie within TIE_REL of each other"""
    N, Cc = post.shape
    ix = inv[:, None].expand(-1, Cc)
    rows = torch.arange(N)[:, None].expand(-1, Cc)
    m1 = _pool(post, inv, G)
    first = torch.full((G, Cc), N, dtype=torch.long).scatter_reduce(0, ix, torch.where(post == m1[inv], rows, N), "amin")
    rest = torch.where(rows == first[inv], torch.tensor(-float("inf"), dtype=post.dtype), post)
    m2 = torch.full((G, Cc), -float("inf"), dtype=post.dtype).scatter_reduce(0, ix, rest, "amax")
    # exactly equal values (ReLU zeros, a channel held constant) are equal in fp32 as well, and both sides give the lowest row
    tie = torch.isfinite(m2) & (m1 != m2) & ((m1 - m2) <= tie_rel * torch.maximum(m1.abs(), m2.abs()))
    second = torch.full((G, Cc), N, dtype=torch.long).scatter_reduce(0, ix, torch.where(rest == m2[inv], rows, N), "amin")
    return torch.unique(second[tie])


def _separate_ties(m, x, fcl, inv, G):
    """move runner-up points of near-tied (group, channel) pairs into groups of their own until none is left (asserted)"""
    inv = inv.clone()
    for _ in range(20):
        *_, posts = _magnitudes(m, x, fcl, inv, G, False, False)
        moved = torch.unique(torch.cat([_near_ties(p, inv, G, TIE_REL) for p in posts]))
        if moved.numel() == 0:
            return inv, G
        inv[moved] = G + torch.arange(moved.numel())
        G += moved.numel()
    raise AssertionError("inputs with separated group maxima not found")


def _grad_check(got, ref, what, tol=GRAD_TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    if ref.dim() == 1:
        got, ref = got[:, None], ref[:, None]
    assert torch.isfinite(got).all(), f"{what}: non-finite gradient"
    err = (got - ref).abs().amax(1)
    b = tol * (ref.abs().amax(1) + 1e-3 * ref.abs().max())
    bad = torch.nonzero(err > b).flatten()
    if bad.numel():
        k = int(bad[torch.argmax(err[bad] / b[bad])])
        raise AssertionError(f"{what}: {bad.numel()} of {err.numel()} rows beyond the bound; worst row {k}: err {err[k].item():.3e} "
                             f"bound {b[k].item():.3e}")
    nz = b > 0
    return float((err[nz] / b[nz]).max()) * tol if bool(nz.any()) else 0.0


def _check_train(cuda, m, x, fcl, inv, G, shortcut=False, csr=False, seed=0, grad_tol=GRAD_TOL):
    """forward on the training route (guarded, poisoned, repeated), then the native backward twice (bit-identical) against
    float64 autograd through the oracle"""
    from sst_b200.sir_modules import SirLayerFunction, group_csr
    inv, G = _separate_ties(m, x, fcl, inv, G)
    _check_forward(cuda, m, x, fcl, inv, G, "train", shortcut, csr)
    g = torch.Generator().manual_seed(seed)
    w = _w64(m, grad=True)
    x_o, c_o = x.double().requires_grad_(True), fcl.double().requires_grad_(True)
    pf, gf = O.sir_layer_forward(x_o, inv, G, c_o, w, "x.", len(m.rel_dims), m.num_vfe, NZ, EPS, m.act, SCALER, with_shortcut=shortcut)
    up_p, up_g = torch.randn(pf.shape, generator=g), torch.randn(gf.shape, generator=g)
    ((pf * up_p.double()).sum() + (gf * up_g.double()).sum()).backward()
    m = m.to(cuda)
    inv_d = inv.to(cuda)
    cs = group_csr(inv_d, G) if csr else None
    runs = []
    for twin in (True, False, False):
        mm = _poison_twin(m) if twin else m
        params = [p.detach().clone().requires_grad_(True) for p in mm._train_params()]
        xg = (x.to(cuda) * (POISON if twin else 1.0)).requires_grad_(True)
        cg = fcl.to(cuda).requires_grad_(True)
        a, b = SirLayerFunction.apply(mm, shortcut, xg, cg, inv_d, G, cs, *params)
        ((a * up_p.to(cuda)).sum() + (b * up_g.to(cuda)).sum()).backward()
        torch.cuda.synchronize()
        if not twin:
            runs.append([xg.grad, cg.grad] + [p.grad for p in params])
    for u, v in zip(*runs):
        assert u is not None and torch.equal(u, v), "two identical backward calls differ"
    names = [n_ for n_, p in m.named_parameters()]
    order = {id(p): n_ for n_, p in m.named_parameters()}
    pnames = [order[id(p)] for p in m._train_params()]
    assert sorted(pnames) == sorted(names)
    worst = {"in_feats": _grad_check(runs[0][0], x_o.grad, "grad in_feats", grad_tol),
             "f_cluster": _grad_check(runs[0][1], c_o.grad, "grad f_cluster", grad_tol)}
    for n_, gr in zip(pnames, runs[0][2:]):
        worst[n_] = _grad_check(gr, w["x." + n_].grad, f"grad {n_}", grad_tol)
    k = max(worst, key=worst.get)
    print(f"[sir-edges] train grads N={x.shape[0]} G={G} worst err/scale {worst[k]:.3g} ({k})")


# ----------------------------------------------------------------------------------------------------------------------
# tests: layouts
# ----------------------------------------------------------------------------------------------------------------------
NS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, "S128", "S128+1", "2S128+37"]


@pytest.mark.parametrize("route", ["fp32", "bf16"])
@pytest.mark.parametrize("layout", ["one", "distinct", "random"])
@pytest.mark.parametrize("n", NS, ids=str)
def test_layouts(cuda, route, layout, n):
    """one group, N distinct groups (32 per warp) and random sizes with empty groups, at every tile / chunk edge"""
    N = _n(n)
    x, fcl = _inputs(N, 84, 3, seed=N)
    inv, G = _groups(_counts(layout, N, N), seed=N + 1)
    _check_forward(cuda, _layer(84, seed=1), x, fcl, inv, G, route, csr=(N % 2 == 1))


@pytest.mark.parametrize("route", ["fp32", "bf16", "train"])
@pytest.mark.parametrize("csr", [False, True], ids=["csr_built", "csr_given"])
@pytest.mark.parametrize("layout,n", [("edges", 700), ("span3", 900), ("g4096", 0), ("g4097", 0)])
def test_special_layouts(cuda, route, csr, layout, n):
    """group edges at CSR positions 31|32, 63|64, 127|128, 128|129; one group over three tiles between singletons; the group_csr
    small / large switch at G = 4096 | 4097"""
    counts = _counts(layout, n, 5)
    N = sum(counts)
    x, fcl = _inputs(N, 133, 3, seed=N)
    inv, G = _groups(counts, seed=7)
    m = _layer(133, seed=2)
    if route == "train":
        _check_train(cuda, m, x, fcl, inv, G, csr=csr, seed=3)
    else:
        _check_forward(cuda, m, x, fcl, inv, G, route, csr=csr)


# ----------------------------------------------------------------------------------------------------------------------
# tests: widths
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["relu", "gelu"])
@pytest.mark.parametrize("rel_in", [1, 3, 4])
@pytest.mark.parametrize("cin", [3, 8, 84, 127, 128, 129, 133, 155])
def test_bf16_widths(cuda, cin, rel_in, act):
    """every cin the tensor-core route takes (KP = 128 | 192; past 155 the in_feats tile no longer fits shared memory),
    rel_mlp_in_channel 1..4, ReLU and GELU"""
    counts = EDGE + _random_counts(cin, 300, 1, 9)
    x, fcl = _inputs(sum(counts), cin, rel_in, seed=cin + rel_in)
    inv, G = _groups(counts, seed=cin)
    _check_forward(cuda, _layer(cin, rel_in=rel_in, act=act, seed=cin), x, fcl, inv, G, "bf16")


@pytest.mark.parametrize("cin,rel_in", [(156, 3), (191, 3), (192, 3), (193, 3), (84, 5)])
def test_bf16_refuses(cuda, cin, rel_in):
    from sst_b200._lib import SSTB200Error
    x, fcl = _inputs(200, cin, rel_in, seed=0)
    inv, G = _groups([100, 100], seed=0)
    with pytest.raises(SSTB200Error):
        _eval_call(_layer(cin, rel_in=rel_in).to(cuda), x.to(cuda), fcl.to(cuda), inv.to(cuda), G, "bf16", False)
    # the context stays usable
    _check_forward(cuda, _layer(84), *_inputs(200, 84, 3, seed=0), inv, G, "bf16")


FEATS = [(a, b) for a in (32, 96, 128, 160, 256) for b in (32, 96, 128, 160, 256)] + [(a,) for a in (32, 96, 128, 160, 256)]
WIDTHS = ([("feats", f, 84, 3, (16, 32)) for f in FEATS] + [("cin", (128, 128), c, 3, (16, 32)) for c in (3, 35, 64, 65, 84, 133, 213, 256)]
          + [("rel_in", (128, 128), 84, r, (16, 32)) for r in (1, 3, 13, 32)]
          + [("num_rel", (128, 128), 84, 3, d) for d in ((), (16,), (16, 32), (16, 32, 64))])


@pytest.mark.parametrize("route", ["fp32", "train"])
@pytest.mark.parametrize("kind,feats,cin,rel_in,rel_dims", WIDTHS, ids=lambda v: str(v).replace(" ", ""))
def test_fp32_widths(cuda, route, kind, feats, cin, rel_in, rel_dims):
    """(C0, C1) over 32..256 and num_vfe = 1, cin 3..256, rel_mlp_in_channel 1..32 (13 is the RoI head's), 1..4 rel-MLP layers"""
    counts = EDGE + _random_counts(cin + len(feats), 1025 - sum(EDGE), 0, 20)
    x, fcl = _inputs(1025, cin, rel_in, seed=cin * 7 + rel_in)
    inv, G = _groups(counts, seed=cin)
    m = _layer(cin, feats=feats, rel_dims=rel_dims, rel_in=rel_in, seed=sum(feats) + cin)
    if route == "train":
        _check_train(cuda, m, x, fcl, inv, G, seed=cin)
    else:
        _check_forward(cuda, m, x, fcl, inv, G, route)


@pytest.mark.parametrize("route", ["fp32", "train", "bf16"])
@pytest.mark.parametrize("cin,feats", [(131, (128, 128)), (35, (32,)), (99, (96, 96))])
def test_shortcut(cuda, route, cin, feats):
    """with_shortcut where cin - 3 == C_last: point features + in_feats[:, 3:]"""
    if route == "bf16" and feats != (128, 128):
        pytest.skip("the tensor-core route is built for [128, 128] only")
    counts = _random_counts(cin, 900, 1, 30)
    x, fcl = _inputs(900, cin, 3, seed=cin)
    inv, G = _groups(counts, seed=cin)
    m = _layer(cin, feats=feats, seed=cin)
    if route == "train":
        _check_train(cuda, m, x, fcl, inv, G, shortcut=True, seed=cin)
    else:
        _check_forward(cuda, m, x, fcl, inv, G, route, shortcut=True)


@pytest.mark.parametrize("route", ["fp32", "train"])
@pytest.mark.parametrize("cin,feats", [(257, (128, 128)), (84, (48, 48))])
def test_fp32_refuses(cuda, route, cin, feats):
    from sst_b200._lib import SSTB200Error
    x, fcl = _inputs(200, cin, 3, seed=0)
    inv, G = _groups([100, 100], seed=0)
    m = _layer(cin, feats=feats).to(cuda)
    with pytest.raises(SSTB200Error):
        if route == "train":
            _train_call(m, x.to(cuda), fcl.to(cuda), inv.to(cuda), G, False)
        else:
            _eval_call(m, x.to(cuda), fcl.to(cuda), inv.to(cuda), G, "fp32", False)


# ----------------------------------------------------------------------------------------------------------------------
# tests: training row counts
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 15, 16, 17, 63, 64, 65, 1025, 150000])
def test_train_rows(cuda, N):
    """FSD widths (cin 133, [128, 128], rel-MLP 16-32, GELU) on both sides of the dW 16-row steps, the 64-row flush and the
    splits; K and M tails against 64 are in test_fp32_widths.  150 000 points is the FSD frame size."""
    counts = _random_counts(N, N, 0, 8) if N < 150000 else _random_counts(N, N, 400, 800)
    x, fcl = _inputs(N, 133, 3, seed=N)
    inv, G = _groups(counts, seed=N)
    _check_train(cuda, _layer(133, seed=4), x, fcl, inv, G, csr=N % 2 == 0, seed=N)


# ----------------------------------------------------------------------------------------------------------------------
# tests: shift cases
# ----------------------------------------------------------------------------------------------------------------------
def _rel3_shift_pair(cin, act="gelu", seed=0):
    """(base, shifted): the last rel-MLP layer's weights are k / 128 (k in -1..1, exact in bf16) and its inputs about 3 (a large
    rel_mlp.1 LayerNorm bias); the shifted layer adds 1 to every weight, a part shared by all cin outputs about 1000 times their
    spread.  LayerNorm removes it, so both compute the same function."""
    base = _layer(cin, act=act, seed=seed)
    g = torch.Generator().manual_seed(seed + 2)
    with torch.no_grad():
        base.rel_mlp[1][1].bias.add_(3.0)
        w = base.rel_mlp[2][0].weight
        w.copy_(torch.randint(-1, 2, w.shape, generator=g).float() / 128)
        w[:, 0] = 1.0 / 128  # no all-zero row
    shifted = copy.deepcopy(base)
    with torch.no_grad():
        shifted.rel_mlp[2][0].weight.add_(1.0)
    return base, shifted


@pytest.mark.parametrize("route", ["fp32", "bf16"])
@pytest.mark.parametrize("cin", [8, 84, 127, 133])
def test_rel3_shift(cuda, route, cin):
    base, shifted = _rel3_shift_pair(cin, seed=cin)
    counts = EDGE + _random_counts(cin, 600, 1, 9)
    x, fcl = _inputs(sum(counts), cin, 3, seed=cin)
    inv, G = _groups(counts, seed=cin)
    _check_forward(cuda, shifted, x, fcl, inv, G, route, bound_model=base, max_tol=MAX_TOL_SHIFT)


def _vfe_shift_pair(cin, seed=0):
    """(base, shifted, x): x0[:, 3] is about 1024 (in_feats[:, 3] over a constant rel-MLP gate) and p0[:, 0] is act(4); the base
    layer's weights on them are 0, the shifted layer's 1 and 256 (exact in bf16): an offset of about 1024 in every pre-LayerNorm
    row of both VFE layers"""
    base = _layer(cin, seed=seed)
    with torch.no_grad():
        base.rel_mlp[2][1].weight[3] = 0.0
        base.rel_mlp[2][1].bias[3] = 1.0
        base.vfe_layers[0].linear.weight[:, 3] = 0.0
        base.vfe_layers[0].norm.weight[0] = 0.0
        base.vfe_layers[0].norm.bias[0] = 4.0
        base.vfe_layers[1].linear.weight[:, 0] = 0.0
    shifted = copy.deepcopy(base)
    with torch.no_grad():
        shifted.vfe_layers[0].linear.weight[:, 3] = 1.0
        shifted.vfe_layers[1].linear.weight[:, 0] = 256.0
    return base, shifted


@pytest.mark.parametrize("route", ["fp32", "bf16", "train"])
def test_vfe_shift(cuda, route):
    base, shifted = _vfe_shift_pair(84, seed=6)
    counts = EDGE + _random_counts(6, 600, 1, 9)
    x, fcl = _inputs(sum(counts), 84, 3, seed=6)
    x[:, 3] = 1024.0 / float(F.gelu(torch.tensor(1.0))) * (1 + 0.01 * torch.randn(x.shape[0], generator=torch.Generator().manual_seed(6)))
    inv, G = _groups(counts, seed=6)
    # the training route's forward only: with x0[:, 3] ~ 1024 the gradients are cancelling sums of terms ~1000 x the result
    _check_forward(cuda, shifted, x, fcl, inv, G, route, bound_model=base, max_tol=MAX_TOL_SHIFT)


# ----------------------------------------------------------------------------------------------------------------------
# tests: the bf16 hand-over buffer and the module
# ----------------------------------------------------------------------------------------------------------------------
def test_bf16_handover_buffer(cuda):
    """SIR's in-place [points || pad || feats] buffer with npt = 5 (pad 3): the block reads the features past the pad and writes
    its point features over them; the point and pad columns keep their contents, the result equals the dense call bit for bit"""
    from sst_b200.sir_modules import group_csr
    npt, pad, N = 5, 3, 2000
    m = _layer(npt + 128, seed=8).to(cuda)
    m.precision = "bf16"
    x, fcl = _inputs(N, npt + 128, 3, seed=8)
    inv, G = _groups(_random_counts(8, N, 1, 20), seed=8)
    x, fcl, inv = x.to(cuda), fcl.to(cuda), inv.to(cuda)
    coors = torch.stack([torch.zeros_like(inv), inv], 1)
    new_coors = torch.stack([torch.zeros(G, dtype=torch.long, device=cuda), torch.arange(G, device=cuda)], 1)
    csr = group_csr(inv, G)
    kw = dict(unq_inv_once=inv, new_coors_once=new_coors, csr_once=csr)
    with torch.no_grad():
        dense_p, dense_g = m(x, coors, fcl, **kw)
        buf = torch.empty((N, npt + pad + 128), device=cuda)
        buf[:, :npt] = x[:, :npt]
        buf[:, npt:npt + pad] = -12345.0
        buf[:, npt + pad:] = x[:, npt:]
        keep = buf[:, :npt + pad].clone()
        p, g = m(buf, coors, fcl, point_feats_out=buf[:, npt + pad:], feat_gap=(npt, pad), **kw)
    torch.cuda.synchronize()
    assert torch.equal(buf[:, :npt + pad], keep)
    assert torch.equal(buf[:, npt + pad:], dense_p) and torch.equal(g, dense_g)


def test_bf16_point_out_view_offset(cuda):
    """point_feats_out = buf[:, 1:129] of a [N, 132] buffer: row pitch a multiple of 4 floats, base 4 bytes off 16-byte alignment;
    the result equals the dense call bit for bit and the columns outside the view keep their contents"""
    N = 1000
    m = _layer(84, seed=9).to(cuda)
    m.precision = "bf16"
    x, fcl = _inputs(N, 84, 3, seed=9)
    inv, G = _groups(_random_counts(9, N, 1, 20), seed=9)
    x, fcl, inv = x.to(cuda), fcl.to(cuda), inv.to(cuda)
    coors = torch.stack([torch.zeros_like(inv), inv], 1)
    new_coors = torch.stack([torch.zeros(G, dtype=torch.long, device=cuda), torch.arange(G, device=cuda)], 1)
    kw = dict(unq_inv_once=inv, new_coors_once=new_coors)
    with torch.no_grad():
        dense_p, dense_g = m(x, coors, fcl, **kw)
        buf = torch.full((N, 132), SENTINEL, device=cuda)
        view = buf[:, 1:129]
        assert view.data_ptr() % 16 == 4 and view.stride(0) % 4 == 0
        p, g = m(x, coors, fcl, point_feats_out=view, **kw)
    torch.cuda.synchronize()
    assert torch.equal(view, dense_p) and torch.equal(g, dense_g)
    assert bool((buf[:, 0] == SENTINEL).all()) and bool((buf[:, 129:] == SENTINEL).all())


def test_bf16_refuses_misaligned_group_out(cuda):
    """the tensor-core route reads the pooled layer-0 features back from out_group as float4: a base off 16 bytes is refused"""
    from sst_b200 import _lib as L
    from sst_b200._lib import SSTB200Error
    N = 300
    m = _layer(84, seed=10).to(cuda)
    x, fcl = _inputs(N, 84, 3, seed=10)
    inv, G = _groups(_random_counts(10, N, 1, 9), seed=10)
    x, fcl, inv = x.to(cuda), fcl.to(cuda), inv.to(cuda)
    point = torch.empty((N, 128), device=cuda)
    group = torch.empty((G * 256 + 1,), device=cuda)[1:]
    s = _struct(m, False)
    c = L.ctx(cuda)
    with pytest.raises(SSTB200Error):
        L.check(c, L.lib().sstb200_sir_layer_forward_ex(c, C.byref(s), x.data_ptr(), 0, 0, 0, fcl.data_ptr(), inv.data_ptr(), N, G, None,
                                                         None, 1, point.data_ptr(), 0, group.data_ptr()))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_module_groups_and_inverse(cuda, precision):
    """through SIRLayer.forward from coordinates: the group coordinates and the inverse equal torch.unique's exactly, and the
    features meet the per-row bound"""
    N = 3000
    g = torch.Generator().manual_seed(11)
    coors = torch.stack([torch.randint(0, 2, (N,), generator=g), torch.randint(0, 5, (N,), generator=g),
                         torch.randint(0, 40, (N,), generator=g)], 1)
    new_coors, inv = torch.unique(coors, return_inverse=True, dim=0)
    G = new_coors.shape[0]
    x, fcl = _inputs(N, 84, 3, seed=11)
    m = _layer(84, seed=11)
    m.return_point_feats = False
    m = m.to(cuda)
    m.precision = precision
    with torch.no_grad():
        vf, nc, ui = m(x.to(cuda), coors.to(cuda), fcl.to(cuda), return_inv=True)
    assert torch.equal(nc.cpu(), new_coors) and torch.equal(ui.cpu(), inv)
    _, gref = _reference(m.cpu(), x, fcl, inv, G, False)
    _, mg, _, dg, _ = _magnitudes(m, x, fcl, inv, G, False, precision == "bf16")
    _row_check(vf, gref, mg + dg / DEV_UNIT, ROW_TOL[precision], MAX_TOL[precision], f"{precision} module group")
