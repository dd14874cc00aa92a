"""The 16-bit mode of the SRA encoder layer (precision 'bf16', IEEE fp16 operands with fp32 accumulation; csrc/sra_bf16.cu,
csrc/wgmma_gemm.cuh, csrc/sra_attn.cuh, csrc/sra_chain2.cu) pinned to a rounding-exact emulation and to a float64 oracle on every
route, tile edge and window shape.

The emulation computes in float64 and rounds to fp16 (nearest even, as cvt.rn / __floats2half2_rn) exactly where the kernels do:

    QKV GEMM   (PRO_F32; EPI_F16 for tensor-core attention, EPI_H16 with fp16 format for the SIMT kernel)
               q|k = f16(f16(x + pos) . Wqk16^T + bqk), the sum x + pos formed in fp32;  v = f16(f16(x) . Wv16^T + bv)
    attention  a window of one token gives att = v exactly in every attention kernel (a single logit's softmax is 1, also with
               cosine logits, and P . v is exact)
    chain      t = att . Wo16^T + bo + x;  x1 = Norm1(t)            (two-pass LayerNorm, or eval BatchNorm folded to scale / shift)
               h = f16(gelu_ex2(f16(x1) . W1_16^T + b1))
               y = Norm2(h . W2_16^T + b2 + x1)                     (x1 the fp32 value, not its fp16 operand copy)
    tail       next q|k = f16(f16(y + pos') . Wqk16^T + bqk), next v = f16(f16(y) . Wv16^T + bv)   (stack, all layers but the last)

Three kinds of checks:
  - layouts with one token per window (voxels on a lattice whose stride is the window size): y of the single-layer API and of
    the stack with 1, 2 and 3 layers, each layer's y against the emulation of its chain: per row within EMU_ROW, and most rows
    within EMU_FLOOR (only rounding ties resolved the other way by the kernel's fp32 values lie between);
  - q|k|v read from the context's arena after a call, on windows (10, 10), (12, 12, 1) and (16, 16, 1): every element equal to
    the emulated GEMM / chain tail or one fp16 ulp from it, at most ULP_FRAC of them one ulp;
  - every route on real multi-token windows against the float64 oracle: the 1e-2 contract plus ROW_TOL per row; refused shapes
    raise SSTB200Error without writing output; operand scale.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import sst_oracle as O
from test_gpu_sra_chain_epilogue import gelu_ex2_mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-2            # the 16-bit contract: max-norm and element-wise, against the output's max-abs
# y of one layer against its emulation (the layer's own GPU input and attention rows fed to the emulation), per row.  A row
# whose fp16 roundings all agree differs only by fp32 accumulation order, rsqrtf and ex2.approx: below EMU_FLOOR.  A rounding
# tie that the kernel's fp32 value resolves the other way flips one h or f16(x1) element by one fp16 ulp, which moves its row
# by up to EMU_ROW; at most FLIP_SHARE of the rows (of 32 or more) may be above the floor.  Measured on an H100 80GB HBM3
# (700 W power limit) over every layer of every case here: rows without a flip at 3e-7 to 7e-7 (median) and 1.8e-6 (90th
# percentile) of their max-abs, so EMU_FLOOR = 1e-5; rows with one at most 3.3e-4, so EMU_ROW = 1.5e-3; at most 15.4 % of the
# rows above the floor (4.7 to 5.2 % at 34011 rows), so FLIP_SHARE = 0.35.  Each chain mutation of the mutation check (h
# rounded to bf16, LN2's residual from the fp16 copy of x1, a tanh GELU) puts every row above the floor.
EMU_FLOOR = 1e-5
EMU_ROW = 1.5e-3
FLIP_SHARE = 0.35
# per row against the float64 oracle on multi-token windows.  Measured as above: at most 1.05e-3 (fused stack, 3 BatchNorm
# cosine layers), so 4e-3
ROW_TOL = 4e-3
# q|k|v from the arena against the emulation: at most ULP_FRAC of the elements one fp16 ulp apart, the rest equal, except
# outputs that cancel to far below their terms, which may differ by ACC_REL of sum_k |a_k w_k| (fp32 accumulation order).
# Measured as above: one-ulp share 7.7e-4 to 9.4e-4; 13 to 22 of 576000 elements further apart (up to 6 ulp), all by at
# most 6.8e-8 of their terms.  So ULP_FRAC = 4e-3 and ACC_REL = 2^-22 (2.4e-7).
ULP_FRAC = 4e-3
ACC_REL = 2.0 ** -22
SSTB_ERR_UNSUPPORTED = -3   # csrc/common.cuh
ATT_MAXT = 144              # csrc/common.cuh: tokens per window of the tensor-core attention
ODD = "odd_tiles"           # (2 x SMs + 2) 128-row tiles, the last one partial
SENTINEL = 7.0


def _drop(top):
    return {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
            2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': top, 'drop_range': (100, 100000)}}


DROP144, DROP256 = _drop(144), _drop(256)
LN = ({}, "gelu")
BN_COS = (dict(use_bn=True, cosine=True, non_shared_tau=True, tau_min=0.01), "gelu")
NORMS = {"layernorm": LN, "batchnorm_cosine": BN_COS}


# ------------------------------------------------------------------------------------------------------------------------------
# routes, mirrored from the dispatch of csrc/sra_api.cu and csrc/sra_bf16.cu
# ------------------------------------------------------------------------------------------------------------------------------
def _pos_geom(win, d=128):
    """(pos_ndim, pos_maxw, pos_L) of SSTInputLayerV2's positional table for window `win`"""
    from sst_b200.sst_modules import _pos_table
    _, ndim, maxw, Lp = _pos_table(win, d, 10000, False)
    return ndim, maxw, Lp


def route(api, win, max_tokens, d=128, ff=256, nhead=8, post_norm=True, act="gelu", bn=False, tau_n=0):
    """Route of one layer through sstb200_sra_layer_forward (api "layer") or of a stack of such layers through
    sstb200_sra_stack_forward (api "stack"): "fused" (QKV GEMM once, then attention + chain with the next layer's q|k|v per layer),
    "layer_tc" / "layer_simt" (QKV GEMM, tensor-core or SIMT attention, chain), "fallback_layer_*" (the stack refused, per-layer
    calls), or "refused" (SSTB_ERR_UNSUPPORTED)."""
    ndim, maxw, Lp = _pos_geom(win, d)
    tau_ok = tau_n in (0, 1, 8)
    if api == "stack":
        if (d == 128 and ff == 256 and post_norm and act == "gelu" and nhead == 8 and tau_ok and 0 < max_tokens <= ATT_MAXT
                and Lp % 32 == 0 and 1 <= ndim <= 3 and ndim * maxw <= 32 and ndim * Lp <= 128):
            return "fused"
        r = route("layer", win, max_tokens, d, ff, nhead, post_norm, act, bn, tau_n)
        return r if r == "refused" else "fallback_" + r
    if d != 128 or ff != 256 or not post_norm or bn or act != "gelu" or Lp % 8:
        return "refused"
    return "layer_tc" if nhead == 8 and tau_ok and 0 < max_tokens <= ATT_MAXT else "layer_simt"


def test_route_matrix():
    """CPU: the dispatch rules `route` restates are the ones in the sources, and the cases of this file reach every route."""
    src = open(os.path.join(ROOT, "sst_b200", "csrc", "sra_bf16.cu")).read()
    api = open(os.path.join(ROOT, "sst_b200", "csrc", "sra_api.cu")).read()
    common = open(os.path.join(ROOT, "sst_b200", "csrc", "common.cuh")).read()
    flat = " ".join(src.split())
    assert "if (d != 128 || ff != 256 || !L->post_norm || L->norm1_mean || L->act != 2)" in flat
    assert "if (P->pos_table && P->pos_L % 8 != 0)" in flat
    assert ("const bool tc_attn = L->nhead == 8 && (!L->tau || L->tau_n == 1 || L->tau_n == 8) && P->max_window_tokens > 0 && "
            "P->max_window_tokens <= ATT_MAXT && P->num_windows_dev && P->win_batch;") in flat
    assert "qkv_gemm(c, L, P, x, qkv, n_cap, n_dev, tc_attn)" in flat
    assert ("return L->d_model == 128 && L->dim_ff == 256 && L->post_norm && L->act == 2 && L->nhead == 8 && (!L->tau || "
            "L->tau_n == 1 || L->tau_n == 8) && (!L->norm1_mean || (L->norm1_var && L->norm2_mean && L->norm2_var)) && "
            "L->in_proj_w_f16 && L->out_proj_w_f16 && L->lin1_w_f16 && L->lin2_w_f16 && P->max_window_tokens > 0 && "
            "P->max_window_tokens <= ATT_MAXT && P->num_windows_dev && P->win_batch && P->pos_table && P->pos_code && "
            "P->pos_L % 32 == 0 && P->pos_ndim >= 1 && P->pos_ndim <= 3 && P->pos_ndim * P->pos_maxw <= 32 && "
            "P->pos_ndim * P->pos_L <= 128;") in flat
    assert "if (!layer_supported_tc(&layers[l], &plans[l & 1])) return SSTB_ERR_UNSUPPORTED;" in flat
    assert "if (rc != SSTB_ERR_UNSUPPORTED) return rc;" in api and "sstb200_sra_layer_forward(c, &layers[l], &plans[l & 1]" in api
    assert f"#define ATT_MAXT {ATT_MAXT}" in common
    # the geometry of the windows used here
    assert _pos_geom((10, 10)) == (2, 10, 64) and _pos_geom((12, 12, 1)) == (2, 12, 64)
    assert _pos_geom((16, 16, 1)) == (2, 16, 64) and _pos_geom((20, 20, 1)) == (2, 20, 64)
    assert _pos_geom((12, 12, 4)) == (3, 12, 42)
    # every route of this file
    assert route("stack", (12, 12, 1), 144) == "fused" and route("stack", (10, 10), 144) == "fused"
    assert route("stack", (16, 16, 1), 144) == "fused"                          # pos_ndim x pos_maxw == 32: the edge
    assert route("stack", (12, 12, 1), 144, bn=True, tau_n=8) == "fused"
    assert route("layer", (12, 12, 1), 144) == "layer_tc"
    assert route("layer", (12, 12, 1), 144, tau_n=8) == "layer_tc"
    for h in (4, 16):
        assert route("layer", (12, 12, 1), 144, nhead=h) == "layer_simt"
        assert route("stack", (12, 12, 1), 144, nhead=h) == "fallback_layer_simt"
    assert route("layer", (16, 16, 1), 256) == "layer_simt" and route("stack", (16, 16, 1), 256) == "fallback_layer_simt"
    assert route("stack", (20, 20, 1), 144) == "fallback_layer_tc"               # pos_ndim x pos_maxw == 40
    for kw in (dict(d=64, nhead=4, ff=256), dict(ff=512), dict(post_norm=False), dict(act="relu")):
        assert route("layer", (12, 12, 1), 144, **kw) == "refused" and route("stack", (12, 12, 1), 144, **kw) == "refused"
    assert route("layer", (12, 12, 1), 144, bn=True) == "refused"               # BatchNorm: the fused stack only
    assert route("stack", (20, 20, 1), 144, bn=True) == "refused"
    assert route("layer", (12, 12, 4), 144) == "refused" and route("stack", (12, 12, 4), 144) == "refused"   # pos_L 42


# ------------------------------------------------------------------------------------------------------------------------------
# the rounding-exact emulation
# ------------------------------------------------------------------------------------------------------------------------------
def f16(x):
    """fp32 value -> fp16 (nearest even, inf past 65504 as __floats2half2_rn), returned as float64"""
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float32).astype(np.float16).astype(np.float64)


def _np(t):
    return t.detach().cpu().double().numpy()


def layer_params(layer):
    """A layer's parameters as the 16-bit path sees them: the fp16 weight copies (EncoderLayer.half_weights casts with
    Tensor.to(float16), nearest even), fp32 biases and norms; BatchNorm folded to one scale and shift per channel."""
    sa = layer.win_attn.self_attn
    h = lambda w: w.detach().cpu().to(torch.float16).double().numpy()
    p = dict(w_in=h(sa.in_proj_weight), b_in=_np(sa.in_proj_bias), w_o=h(sa.out_proj.weight), b_o=_np(sa.out_proj.bias),
             w1=h(layer.linear1.weight), b1=_np(layer.linear1.bias), w2=h(layer.linear2.weight), b2=_np(layer.linear2.bias),
             eps=float(layer.norm1.eps), bn=bool(layer.use_bn))
    for i, nm in ((1, layer.norm1), (2, layer.norm2)):
        w, b = _np(nm.weight), _np(nm.bias)
        if layer.use_bn:
            s = w / np.sqrt(_np(nm.running_var) + p["eps"])
            w, b = s, b - _np(nm.running_mean) * s
        p[f"g{i}"], p[f"be{i}"] = w, b
    return p


def _norm(t, p, i):
    if p["bn"]:
        return t * p[f"g{i}"] + p[f"be{i}"]
    c = t - t.mean(1, keepdims=True)
    return c / np.sqrt((c * c).mean(1, keepdims=True) + p["eps"]) * p[f"g{i}"] + p[f"be{i}"]


def emu_qkv(x, pos, p, pos_after_round=False):
    """The QKV GEMM (or the chain's tail) on fp32 rows x with positional rows pos: fp16 q|k|v [n, 3 d] as float64.
    pos_after_round: the positional term added to f16(x) instead of to x (a wrong order, for the mutation test)."""
    d = x.shape[1]
    x32, pos32 = np.asarray(x, np.float32), np.asarray(pos, np.float32)
    a_qk = f16(f16(x32).astype(np.float32) + pos32) if pos_after_round else f16(x32 + pos32)
    qk = f16(a_qk @ p["w_in"][:2 * d].T + p["b_in"][:2 * d])
    v = f16(f16(x32) @ p["w_in"][2 * d:].T + p["b_in"][2 * d:])
    return np.concatenate([qk, v], 1)


def qkv_terms(x, pos, p):
    """sum_k |a_k w_k| of every q|k|v output of emu_qkv: the scale of its fp32 accumulation error"""
    d = x.shape[1]
    x32, pos32 = np.asarray(x, np.float32), np.asarray(pos, np.float32)
    return np.concatenate([np.abs(f16(x32 + pos32)) @ np.abs(p["w_in"][:2 * d]).T, np.abs(f16(x32)) @ np.abs(p["w_in"][2 * d:]).T], 1)


def emu_chain(att, x, p, mutation=None):
    """The fused chain on fp16 attention rows att and fp32 residual rows x: y [n, d] float64.  `mutation` emulates a wrong
    kernel (mutation test): "bf16_h", "residual_f16", "tanh_gelu"."""
    x1 = _norm(att @ p["w_o"].T + p["b_o"] + x, p, 1)
    z = (f16(x1) @ p["w1"].T + p["b1"]).astype(np.float32)
    if mutation == "tanh_gelu":
        g = 0.5 * z * (1 + np.tanh(0.7978845608028654 * (z + 0.044715 * z.astype(np.float64) ** 3)))
    else:
        g = gelu_ex2_mirror(z)
    if mutation == "bf16_h":
        h = torch.from_numpy(np.asarray(g, np.float32)).to(torch.bfloat16).double().numpy()
    else:
        h = f16(g)
    res = f16(x1) if mutation == "residual_f16" else x1
    return _norm(h @ p["w2"].T + p["b2"] + res, p, 2)


def emu_one_token(x, params, mutation=None):
    """Layers `params` in sequence on a layout with one token per window (att = v): the final y, float64"""
    y = np.asarray(x, np.float64)
    for p in params:
        d = y.shape[1]
        att = emu_qkv(np.asarray(y, np.float32), np.zeros_like(y, np.float32), p)[:, 2 * d:]
        y = emu_chain(att, np.asarray(y, np.float32).astype(np.float64), p, mutation)
    return y


def pos_rows(coors, win, grid, shift, d=128):
    """Flat positional rows [n, d] float32 of voxels `coors` for shift `shift`: the table the kernels read (SSTInputLayerV2's),
    indexed by the float64 oracle's in-window coordinates (so the kernels' pos_code addressing is not used here)"""
    from sst_b200.sst_modules import _pos_table
    tab, ndim, _, Lp = _pos_table(win, d, 10000, False)
    _, ciw = O.get_window_coors(coors.long(), grid, win, shift == 1)
    pe = torch.zeros((coors.shape[0], d), dtype=torch.float32)
    for a in range(ndim):   # axis 0 = x = column 2 of (z, y, x)
        pe[:, a * Lp:(a + 1) * Lp] = tab[a][ciw[:, 2 - a]]
    return pe.numpy()


# ------------------------------------------------------------------------------------------------------------------------------
# models, layouts, float64 oracle, error accounting
# ------------------------------------------------------------------------------------------------------------------------------
def _model(norm="layernorm", blocks=1, nhead=8, d=128, ff=256, post_norm=True, act=None, seed=0, edit="random"):
    """SSTv2 of `blocks` blocks.  edit "random": non-trivial biases, norms, BN running statistics and per-head temperatures;
    "zero_bias": every bias zeroed, so that an input scale reaches every GEMM operand."""
    from sst_b200.sst_modules import SSTv2
    lc, a = NORMS[norm]
    lc = dict(lc, post_norm=post_norm)
    torch.manual_seed(seed)
    m = SSTv2(d_model=[d] * blocks, nhead=[nhead] * blocks, num_blocks=blocks, dim_feedforward=[ff] * blocks,
              output_shape=[468, 468], num_attached_conv=0, to_bev=False, layer_cfg=lc, activation=act or a).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("tau"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.5 + 0.05)
            elif p.dim() == 1 and edit == "random":
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            elif p.dim() == 1 and edit == "zero_bias" and n_.endswith("bias"):
                p.zero_()
        for n_, b in m.named_buffers():
            if "running_mean" in n_:
                b.copy_(torch.randn(b.shape, generator=g) * 0.3)
            if "running_var" in n_:
                b.copy_(torch.rand(b.shape, generator=g) + 0.5)
    return m, lc


def _layers(m):
    return [l for blk in m.block_list for l in blk.encoder_list]


def _lattice(n, win, seed, d=128):
    """n voxels of one sweep, one per window in both shifts: on a lattice of stride `win`, at in-window offset (5, 7).  Returns
    features, coordinates and a sparse shape large enough for n."""
    side = int(np.ceil(np.sqrt(max(n, 1)))) + 1
    grid = (side * win[0], side * win[1], 1)
    g = torch.Generator().manual_seed(seed)
    cell = torch.randperm(side * side, generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), (cell // side) * win[1] + 7,
                         (cell % side) * win[0] + 5], 1).int()
    return torch.randn(n, d, generator=g), coors, grid


def _random(n, grid, seed, d=128, scale=1.0):
    """n distinct random voxels of one sweep in `grid`"""
    g = torch.Generator().manual_seed(seed)
    cell = torch.randperm(grid[0] * grid[1], generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), cell // grid[0], cell % grid[0]], 1).int()
    return torch.randn(n, d, generator=g) * scale, coors


def _info(cuda, feats, coors, win, grid, drop):
    from sst_b200.sst_modules import SSTInputLayerV2
    il = SSTInputLayerV2((drop, drop), win, grid, shuffle_voxels=False, mute=True).eval()
    with torch.no_grad():
        info = il(feats.to(cuda), coors.to(cuda), 1)
    assert info["voxel_feats"].shape[0] == feats.shape[0], "voxels dropped"
    return info


def _oracle64(m, lc, feats, coors, win, grid, drop, num_layers):
    """float64 oracle of the first `num_layers` encoder layers of m (shift i % 2 for layer i)"""
    w = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    info = O.input_layer_v2(feats.double(), coors, drop, win, grid)
    assert info["voxel_feats"].shape[0] == feats.shape[0]
    l0 = _layers(m)[0]
    x = info["voxel_feats"]
    for i in range(num_layers):
        s = i % 2
        x = O.encoder_layer(x, info[f"pos_dict_shift{s}"], info[f"flat2win_inds_shift{s}"], info[f"key_mask_shift{s}"], w,
                            f"block_list.{i // 2}.encoder_list.{s}.", l0.nhead, l0.activation, lc)
    return x


def _rows(n):
    if n != ODD:
        return n
    return (2 * torch.cuda.get_device_properties(0).multi_processor_count + 2) * 128 - 37


def row_errors(got, ref):
    """per row: max |got - ref| over the row's max-abs (at least 1e-3 of the output's max-abs)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = np.maximum(np.abs(ref).max(1), 1e-3 * np.abs(ref).max())
    return np.abs(got - ref).max(1) / scale


def check_emu(got, emu, what):
    """per row within EMU_ROW of the emulation, and (32 rows or more) at most FLIP_SHARE of the rows above EMU_FLOOR"""
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else got
    assert got.shape == emu.shape and np.isfinite(got).all(), f"{what}: shape or non-finite output"
    row = row_errors(got, emu)
    share = float((row > EMU_FLOOR).mean())
    q = np.quantile(row, [0.5, 0.9, 0.99])
    print(f"MEASURE emu {what}: per-row max {row.max():.3e} (row {int(row.argmax())}), quantiles 50/90/99% {q[0]:.2e} {q[1]:.2e} "
          f"{q[2]:.2e}, share above floor {share:.3f}")
    bad = np.flatnonzero(row > EMU_ROW)
    assert bad.size == 0, f"{what}: {bad.size} of {row.size} rows above {EMU_ROW:g} of the emulation; worst {row.max():.3e}, rows {bad[:8]}"
    if row.size >= 32:
        assert share <= FLIP_SHARE, f"{what}: {share:.3f} of the rows above {EMU_FLOOR:g} of the emulation"
    return row.max()


def check_ref(got, ref, what, tol=ROW_TOL):
    """the 16-bit contract (max-norm and element-wise, REL of the output's max-abs) and the per-row `tol`"""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape and torch.isfinite(got).all(), f"{what}: shape or non-finite output"
    amax = ref.abs().max().item()
    err = (got - ref).abs().max().item() / amax
    row = row_errors(got.numpy(), ref.numpy())
    print(f"MEASURE ref {what}: per-row {row.max():.3e} (row {int(row.argmax())}), max-norm {err:.3e}")
    assert err < REL, f"{what}: max-norm error {err:.3e} above the contract {REL:g}"
    torch.testing.assert_close(got, ref, rtol=REL, atol=REL * amax)
    bad = np.flatnonzero(row > tol)
    assert bad.size == 0, f"{what}: {bad.size} of {row.size} rows above {tol:g}; worst {row.max():.3e}, rows {bad[:8]}"


def _ord16(h):
    """fp16 values -> integers in the order of the values, one per representable value (+0 and -0 both 0)"""
    b = np.asarray(h, np.float64).astype(np.float16).view(np.int16).astype(np.int32)
    return np.where(b < 0, -(b & 0x7FFF), b)


def check_ulps(got, emu, terms, what, frac=ULP_FRAC):
    """every element equal to the emulation or one fp16 ulp from it, at most `frac` of them one ulp; elements further apart
    only where the output cancels: |difference| <= ACC_REL sum_k |a_k w_k|"""
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else got
    assert np.isfinite(got).all() and np.isfinite(emu).all()
    dist = np.abs(_ord16(got) - _ord16(emu))
    one = float((dist == 1).mean())
    far = dist > 1
    acc = float((np.abs(got - emu)[far] / terms[far]).max()) if far.any() else 0.0
    print(f"MEASURE ulp {what}: one-ulp share {one:.2e}, {int(far.sum())} of {dist.size} further (max {dist.max()} ulp, "
          f"|difference| / sum|terms| at most {acc:.2e})")
    assert acc <= ACC_REL, f"{what}: {int(far.sum())} elements more than one fp16 ulp apart, up to {acc:.2e} of their terms"
    assert one <= frac, f"{what}: {one:.2e} of the elements one ulp apart, above {frac:g}"


# ------------------------------------------------------------------------------------------------------------------------------
# CPU: the emulation against the float64 oracle, and what the tight bound catches
# ------------------------------------------------------------------------------------------------------------------------------
def _cpu_one_token(norm, num_layers, n=517, seed=3):
    feats, coors, grid = _lattice(n, (12, 12, 1), seed)
    m, lc = _model(norm, blocks=(num_layers + 1) // 2, seed=seed)
    ref = _oracle64(m, lc, feats, coors, (12, 12, 1), grid, DROP144, num_layers)
    params = [layer_params(l) for l in _layers(m)[:num_layers]]
    return feats, coors, grid, params, ref


@pytest.mark.parametrize("num_layers", [1, 2, 3])
@pytest.mark.parametrize("norm", list(NORMS))
def test_emulation_vs_oracle(norm, num_layers):
    """CPU: on a one-token-per-window layout the emulation stays within the 16-bit contract of the float64 oracle; its per-row
    error (printed) is what fp16 operands cost the path by themselves; the kernels are held to the emulation far below it."""
    feats, coors, grid, params, ref = _cpu_one_token(norm, num_layers)
    # the layout really is one token per window in both shifts
    for s in (0, 1):
        win_inds, _ = O.get_window_coors(coors.long(), grid, (12, 12, 1), s == 1)
        assert win_inds.unique().numel() == feats.shape[0]
    emu = emu_one_token(feats.float().numpy(), params)
    err = np.abs(emu - ref.numpy()).max() / ref.abs().max().item()
    row = row_errors(emu, ref.numpy())
    print(f"MEASURE inherent {norm} {num_layers} layers: per-row {row.max():.3e}, max-norm {err:.3e}")
    assert err < REL and row.max() < ROW_TOL
    assert float((row > EMU_FLOOR).mean()) > 0.9


@pytest.mark.parametrize("mutation", ["bf16_h", "residual_f16", "tanh_gelu"])
@pytest.mark.parametrize("norm", list(NORMS))
def test_emulated_mutations_leave_emu_tight(norm, mutation):
    """CPU: each wrong rounding or GELU the chain could take moves nearly every row of one layer's y above EMU_FLOOR (at most
    FLIP_SHARE of them may be), while two such layers stay inside the 1e-2 contract that the older tests hold the path to."""
    feats, coors, grid, params, ref = _cpu_one_token(norm, 2)
    good = emu_one_token(feats.float().numpy(), params[:1])
    bad = emu_one_token(feats.float().numpy(), params[:1], mutation)
    row = row_errors(bad, good)
    share = float((row > EMU_FLOOR).mean())
    print(f"MEASURE mutation {norm} {mutation}: per-row max {row.max():.3e}, share above floor {share:.3f}")
    assert share > 0.9 > FLIP_SHARE
    bad2 = emu_one_token(feats.float().numpy(), params, mutation)
    assert np.abs(bad2 - ref.numpy()).max() / ref.abs().max().item() < REL


def test_emulated_pos_order_leaves_one_ulp():
    """CPU: the positional term added after x is rounded to fp16 moves many q|k elements by more than one fp16 ulp."""
    feats, coors = _random(600, (96, 96, 1), 5)
    m, _ = _model()
    p = layer_params(_layers(m)[0])
    x = feats.float().numpy()
    pos = pos_rows(coors, (12, 12, 1), (96, 96, 1), 0)
    good, bad = emu_qkv(x, pos, p), emu_qkv(x, pos, p, pos_after_round=True)
    dist = np.abs(_ord16(good) - _ord16(bad))
    print(f"MEASURE mutation pos order: {float((dist > 1).mean()):.2e} of q|k|v elements more than one ulp apart")
    assert (dist[:, 256:] == 0).all() and (dist > 1).mean() > 0.05


# ------------------------------------------------------------------------------------------------------------------------------
# GPU calls
# ------------------------------------------------------------------------------------------------------------------------------
def _lib():
    from sst_b200 import _lib as L
    return L


def _layer_call(c, layer, plan, x, y, n, n_dev=None):
    from sst_b200.sst_modules import PRECISIONS, make_sra_plan
    ls, ps = layer._struct(PRECISIONS["bf16"]), make_sra_plan(plan)
    return _lib().lib().sstb200_sra_layer_forward(c, C.byref(ls), C.byref(ps), x.data_ptr(), y.data_ptr(), n,
                                                  None if n_dev is None else n_dev.data_ptr(), PRECISIONS["bf16"])


def _stack_call(c, layers, info, x, y, tmp, n, n_dev=None):
    from sst_b200.sst_modules import PRECISIONS, _SraLayer, make_sra_plan
    arr = (_SraLayer * len(layers))(*[l._struct(PRECISIONS["bf16"]) for l in layers])
    p0, p1 = make_sra_plan(info["sra_plan_shift0"]), make_sra_plan(info["sra_plan_shift1"])
    return _lib().lib().sstb200_sra_stack_forward(c, arr, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(),
                                                  tmp.data_ptr(), n, None if n_dev is None else n_dev.data_ptr(),
                                                  PRECISIONS["bf16"])


def run_layers(cuda, api, layers, info, c=None):
    """`layers` through sstb200_sra_layer_forward one by one (api "layer") or one sstb200_sra_stack_forward (api "stack")"""
    L = _lib()
    c = c or L.ctx(cuda)
    x = info["voxel_feats"].float().contiguous()
    n = x.shape[0]
    if api == "stack":
        y, tmp = torch.full_like(x, SENTINEL), torch.full_like(x, -SENTINEL)
        L.check(c, _stack_call(c, layers, info, x, y, tmp, n))
    else:
        y = x
        for i, l in enumerate(layers):
            nxt = torch.full_like(x, SENTINEL)
            L.check(c, _layer_call(c, l, info[f"sra_plan_shift{i % 2}"], y, nxt, n))
            y = nxt
    torch.cuda.synchronize()
    return y


class _Cuda:
    """Zero-copy view of device memory this test does not own"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def arena_qkv(c, cuda, n):
    """q|k|v [n, 384] and the attention output [n, 128], fp16, as the last bf16 call on context c left them: the first two
    allocations after the arena reset of both sstb_sra_layer_bf16 and sstb_sra_stack_bf16, so q|k|v starts at the arena's base
    and att at the next 256-byte boundary (context fields `int device; cudaStream_t stream; int num_sms; char* arena;`,
    checked through num_sms)"""
    assert C.c_int.from_address(c + 16).value == torch.cuda.get_device_properties(cuda).multi_processor_count, "context layout changed"
    ptr = C.c_uint64.from_address(c + 24).value
    qkv = torch.as_tensor(_Cuda(ptr, (n, 384), "<f2"), device=cuda).clone()
    att = torch.as_tensor(_Cuda(ptr + (n * 384 * 2 + 255) // 256 * 256, (n, 128), "<f2"), device=cuda).clone()
    return qkv, att


# ------------------------------------------------------------------------------------------------------------------------------
# 1. one token per window: y against the emulation
# ------------------------------------------------------------------------------------------------------------------------------
ONE_TOKEN = [("layer", "layernorm", 1), ("layer", "layernorm", 2)] + \
            [("stack", nm, k) for nm in NORMS for k in (1, 2, 3)]


def one_token_layers(cuda, api, m, num_layers, info, params, mutation=None):
    """Layers 1 .. num_layers on a one-token-per-window layout, each checked against the emulation of its chain fed with the
    layer's own GPU input (the previous layer's call, or the stack of one layer fewer) and attention rows read from the arena:
    a rounding flip in one layer then does not carry into the next one's check.  Through the stack, layer k's q|k|v come from
    the chain's tail of layer k - 1."""
    L = _lib()
    c = L.ctx(cuda)
    layers = _layers(m)[:num_layers]
    x = info["voxel_feats"].float().contiguous()
    n = x.shape[0]
    for k in range(1, num_layers + 1):
        if api == "stack":
            y = run_layers(cuda, "stack", layers[:k], info, c)
        else:
            y = torch.full_like(x, SENTINEL)
            L.check(c, _layer_call(c, layers[k - 1], info[f"sra_plan_shift{(k - 1) % 2}"], x, y, n))
            torch.cuda.synchronize()
        qkv, att = arena_qkv(c, cuda, n)
        assert torch.equal(att, qkv[:, 256:]), "one token per window: attention must pass v through exactly"
        emu = emu_chain(att.cpu().double().numpy(), x.cpu().double().numpy(), params[k - 1], mutation)
        check_emu(y, emu, f"{api} {num_layers} layers, layer {k}, n {n}")
        x = y


@pytest.mark.gpu
@pytest.mark.parametrize("api,norm,num_layers", ONE_TOKEN, ids=[f"{a}-{nm}-{k}" for a, nm, k in ONE_TOKEN])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, ODD])
def test_one_token_windows_vs_emulation(cuda, n, api, norm, num_layers):
    """Single-layer API (LayerNorm; the per-layer path refuses BatchNorm) and the fused stack with 1, 2, 3 layers on windows
    of one token each, at row counts on the chain's half-tile and tile edges and (2 x SMs + 2) tiles, against the emulation.
    Attention then passes v through exactly, so the GEMM epilogues, GEMM1-3, GELU and both norms are what is checked."""
    n = _rows(n)
    win = (12, 12, 1)
    feats, coors, grid = _lattice(n, win, seed=n + num_layers)
    m, _ = _model(norm, blocks=(num_layers + 1) // 2, seed=num_layers)
    params = [layer_params(l) for l in _layers(m)[:num_layers]]
    m = m.to(cuda)
    one_token_layers(cuda, api, m, num_layers, _info(cuda, feats, coors, win, grid, DROP144), params)


# ------------------------------------------------------------------------------------------------------------------------------
# 2. q|k|v from the arena: the QKV GEMM and the chain's tail against the emulation, on any window layout
# ------------------------------------------------------------------------------------------------------------------------------
QKV_WINDOWS = [(10, 10), (12, 12, 1), (16, 16, 1)]
QKV_GRID = (96, 96, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", list(NORMS))
@pytest.mark.parametrize("win", QKV_WINDOWS, ids=["10x10", "12x12x1", "16x16x1"])
def test_qkv_gemm_and_tail_vs_emulation(cuda, win, norm):
    """After a single-layer call the arena holds the QKV GEMM's output on x; after a 2-layer stack it holds the chain tail's
    output for layer 1 on y0 (the 1-layer stack's output, checked bitwise against the single-layer API's and, through layer 1,
    against the 2-layer stack's own).  Both against the emulation with the positional rows built from the oracle's in-window
    coordinates: this pins pos_code, pos_grp / pos_shift and the biases of both kernels."""
    L = _lib()
    n = 1500
    feats, coors = _random(n, QKV_GRID, seed=17)
    m, _ = _model(norm, blocks=1, seed=4)
    p = [layer_params(l) for l in _layers(m)]
    pos0, pos1 = (pos_rows(coors, win, QKV_GRID, s) for s in (0, 1))
    m = m.to(cuda)
    layers = _layers(m)
    info = _info(cuda, feats, coors, win, QKV_GRID, DROP144)
    c = L.ctx(cuda)
    x = info["voxel_feats"].float().contiguous()
    if norm == "layernorm":   # the single-layer API (LayerNorm only)
        y0_layer = torch.empty_like(x)
        L.check(c, _layer_call(c, layers[0], info["sra_plan_shift0"], x, y0_layer, n))
        torch.cuda.synchronize()
        check_ulps(arena_qkv(c, cuda, n)[0], emu_qkv(x.cpu().numpy(), pos0, p[0]), qkv_terms(x.cpu().numpy(), pos0, p[0]),
                   f"QKV GEMM {win} {norm}")
    y0 = run_layers(cuda, "stack", layers[:1], info, c)
    check_ulps(arena_qkv(c, cuda, n)[0], emu_qkv(x.cpu().numpy(), pos0, p[0]), qkv_terms(x.cpu().numpy(), pos0, p[0]),
               f"stack QKV GEMM {win} {norm}")
    y1 = run_layers(cuda, "stack", layers, info, c)
    check_ulps(arena_qkv(c, cuda, n)[0], emu_qkv(y0.cpu().numpy(), pos1, p[1]), qkv_terms(y0.cpu().numpy(), pos1, p[1]),
               f"chain tail {win} {norm}")
    if norm == "layernorm":
        assert torch.equal(y0, y0_layer), "the 1-layer stack and the single-layer API differ"
        y1_layer = torch.empty_like(x)
        L.check(c, _layer_call(c, layers[1], info["sra_plan_shift1"], y0, y1_layer, n))
        torch.cuda.synchronize()
        assert torch.equal(y1, y1_layer), "the 2-layer stack's layer 1 differs from a single-layer call on the 1-layer stack's y0"


# ------------------------------------------------------------------------------------------------------------------------------
# 3. every route against float64 on multi-token windows
# ------------------------------------------------------------------------------------------------------------------------------
# name -> (api, norm, nhead, window, grid, n, drop, layers, expected route)
ROUTES = {
    "fused_stack_12x12": ("stack", "layernorm", 8, (12, 12, 1), (96, 96, 1), 2500, DROP144, 3, "fused"),
    "fused_stack_bn_cos": ("stack", "batchnorm_cosine", 8, (12, 12, 1), (96, 96, 1), 2500, DROP144, 3, "fused"),
    "fused_stack_10x10": ("stack", "layernorm", 8, (10, 10), (96, 96, 1), 2500, DROP144, 2, "fused"),
    "fused_stack_16x16": ("stack", "layernorm", 8, (16, 16, 1), (96, 96, 1), 2500, DROP144, 2, "fused"),
    "layer_tc": ("layer", "layernorm", 8, (12, 12, 1), (96, 96, 1), 2500, DROP144, 2, "layer_tc"),
    "layer_simt_nhead4": ("layer", "layernorm", 4, (12, 12, 1), (96, 96, 1), 2500, DROP144, 2, "layer_simt"),
    "layer_simt_nhead16": ("layer", "layernorm", 16, (12, 12, 1), (96, 96, 1), 2500, DROP144, 2, "layer_simt"),
    "stack_simt_nhead4": ("stack", "layernorm", 4, (12, 12, 1), (96, 96, 1), 2500, DROP144, 2, "fallback_layer_simt"),
    "layer_simt_256_tokens": ("layer", "layernorm", 8, (16, 16, 1), (64, 64, 1), 3300, DROP256, 2, "layer_simt"),
    "stack_simt_256_tokens": ("stack", "layernorm", 8, (16, 16, 1), (64, 64, 1), 3300, DROP256, 2, "fallback_layer_simt"),
    "stack_fallback_20x20": ("stack", "layernorm", 8, (20, 20, 1), (100, 100, 1), 2000, DROP144, 2, "fallback_layer_tc"),
}


def test_route_cases_reach_their_routes():
    """CPU: each case of test_route_vs_oracle takes the route it is named for, and the 256-token cases hold windows of more
    than 144 tokens"""
    for name, (api, norm, h, win, grid, n, drop, k, want) in ROUTES.items():
        top = max(v["max_tokens"] for v in drop.values())
        assert route(api, win, top, nhead=h, bn=norm != "layernorm", tau_n=8 if norm != "layernorm" else 0) == want, name
        if top > ATT_MAXT:
            _, coors = _random(n, grid, seed=len(name))
            win_inds, _ = O.get_window_coors(coors.long(), grid, win, False)
            assert torch.bincount(win_inds).max().item() > ATT_MAXT, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ROUTES))
def test_route_vs_oracle(cuda, name):
    """Each route on real multi-token windows: the 1e-2 contract and ROW_TOL per row against the float64 oracle"""
    api, norm, h, win, grid, n, drop, k, _ = ROUTES[name]
    feats, coors = _random(n, grid, seed=len(name))
    m, lc = _model(norm, blocks=(k + 1) // 2, nhead=h, seed=7)
    ref = _oracle64(m, lc, feats, coors, win, grid, drop, k)
    m = m.to(cuda)
    info = _info(cuda, feats, coors, win, grid, drop)
    check_ref(run_layers(cuda, api, _layers(m)[:k], info), ref, name)


# name -> (model kwargs, window, sparse shape, what the error message names)
REFUSED = {
    "d_model_64": (dict(d=64, nhead=4, ff=256), (12, 12, 1), (96, 96, 1), "d=64"),
    "dim_ff_512": (dict(ff=512), (12, 12, 1), (96, 96, 1), "ff=512"),
    "pre_norm": (dict(post_norm=False), (12, 12, 1), (96, 96, 1), "pre-norm"),
    "relu": (dict(act="relu"), (12, 12, 1), (96, 96, 1), "relu"),
    "window_3d": ({}, (12, 12, 4), (96, 96, 8), "positional length (42)"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["layer", "stack"])
@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_shapes(cuda, name, api):
    """Shapes the 16-bit path is not built for end in SSTB200Error naming the cause, with no output row written"""
    L = _lib()
    kw, win, grid, cause = REFUSED[name]
    d = kw.get("d", 128)
    g = torch.Generator().manual_seed(9)
    cell = torch.randperm(grid[0] * grid[1] * grid[2], generator=g)[:400]
    coors = torch.stack([torch.zeros_like(cell), cell // (grid[0] * grid[1]), (cell // grid[0]) % grid[1], cell % grid[0]], 1).int()
    feats = torch.randn(400, d, generator=g)
    m, _ = _model(blocks=1, seed=2, **kw)
    m = m.to(cuda)
    info = _info(cuda, feats, coors, win, grid, DROP144)
    x = info["voxel_feats"].float().contiguous()
    y, tmp = torch.full_like(x, SENTINEL), torch.full_like(x, -SENTINEL)
    c = L.ctx(cuda)
    layers = _layers(m)
    if api == "layer":
        rc = _layer_call(c, layers[0], info["sra_plan_shift0"], x, y, x.shape[0])
    else:
        rc = _stack_call(c, layers, info, x, y, tmp, x.shape[0])
    torch.cuda.synchronize()
    msg = L.lib().sstb200_last_error(c).decode()
    assert rc == SSTB_ERR_UNSUPPORTED, (rc, msg)
    assert cause in msg, msg
    assert (y == SENTINEL).all() and (tmp == -SENTINEL).all()
    with pytest.raises(L.SSTB200Error, match=re.escape(cause)):
        with torch.no_grad():
            if api == "layer":
                layers[0](x, info["sra_plan_shift0"], "bf16")
            else:
                m.precision = "bf16"
                m(info)


@pytest.mark.gpu
def test_batchnorm_refused_by_the_single_layer_api(cuda):
    """BatchNorm runs in the fused stack only: the single-layer API, and so a stack that falls back to it (window 20 x 20),
    refuse it by name"""
    L = _lib()
    feats, coors = _random(500, (100, 100, 1), seed=8)
    m, _ = _model("batchnorm_cosine", blocks=1, seed=2)
    m = m.to(cuda)
    c = L.ctx(cuda)
    for win in ((12, 12, 1), (20, 20, 1)):
        info = _info(cuda, feats, coors, win, (100, 100, 1), DROP144)
        x = info["voxel_feats"].float().contiguous()
        y, tmp = torch.full_like(x, SENTINEL), torch.full_like(x, -SENTINEL)
        rcs = [_layer_call(c, _layers(m)[0], info["sra_plan_shift0"], x, y, x.shape[0])]
        if win[0] == 20:
            rcs.append(_stack_call(c, _layers(m), info, x, y, tmp, x.shape[0]))
        torch.cuda.synchronize()
        assert rcs == [SSTB_ERR_UNSUPPORTED] * len(rcs)
        assert "BatchNorm" in L.lib().sstb200_last_error(c).decode()
        assert (y == SENTINEL).all()


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["layer", "stack"])
@pytest.mark.parametrize("k", [-8, 0, 8])
def test_operand_scale(cuda, k, api):
    """Input features x 2^k with every bias zeroed, so the scale reaches every GEMM operand (fp16 overflows at 65504: |x + pos|
    beyond it gives inf; see sra_bf16.cu).  On one token per window, two layers against the emulation; on multi-token windows,
    two layers against the float64 oracle (contract and ROW_TOL), for k > 0 with the q|k rows of the in-projection x 2^-k so
    that the attention logits keep their size: logits of 1e4 and more, which x 2^8 alone gives, carry fp16 q|k's relative 2^-11 into
    units of the logit, and the softmax of near-tied windows then differs by construction."""
    win = (12, 12, 1)
    feats, coors, grid = _lattice(1000, win, seed=70 + k)
    m, _ = _model(blocks=1, seed=6, edit="zero_bias")
    params = [layer_params(l) for l in _layers(m)]
    m = m.to(cuda)
    one_token_layers(cuda, api, m, 2, _info(cuda, feats * 2.0 ** k, coors, win, grid, DROP144), params)

    grid = (96, 96, 1)
    feats, coors = _random(2000, grid, seed=60 + k, scale=2.0 ** k)
    m, lc = _model(blocks=1, seed=6, edit="zero_bias")
    with torch.no_grad():
        for l in _layers(m):
            l.win_attn.self_attn.in_proj_weight[:256].mul_(2.0 ** -max(k, 0))
    ref = _oracle64(m, lc, feats, coors, win, grid, DROP144, 2)
    m = m.to(cuda)
    info = _info(cuda, feats, coors, win, grid, DROP144)
    check_ref(run_layers(cuda, api, _layers(m), info), ref, f"{api} input x 2^{k}")
