"""The fp32 mode of the SRA encoder layer (csrc/sra_fp32.cu) pinned to a float64 oracle on every GEMM route, row edge, device row
count and operand scale.

Each of the layer's five Linears (q|k, v or q|k|v, out_proj, linear1, linear2) runs on one of two GEMMs:

    x3     sstb_row_gemm_x3 (csrc/spconv.cu)   split-fp16 wgmma, K and N multiples of 64; NT 128 when N % 128 == 0, else NT 64;
                                                K / 64 stages; q|k gets its positional term from add_pos_kernel first
    ffma   gemm_rows_kernel (csrc/rows.cu)      fp32 FFMA, any K and N; the q|k|v GEMM takes it whenever d_model or dim_ff is not a
                                                multiple of 64, with the positional term fused into its A loads (pos_ncols = 2 d)

and the norms run on add_norm_kernel (csrc/rows.cu: post- or pre-norm, LayerNorm or eval BatchNorm, at most 8 values per lane:
d_model <= 256).
Every comparison is held to two bounds against the float64 oracle: the fp32 contract (max-norm, 1e-3 of the output's max-abs) and,
per row, TIGHT of that row's max-abs (or 1e-3 of the output's max-abs, whichever is larger), so that an error confined to a few
rows, columns or tile edges cannot hide in a max-norm over the frame.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import sst_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN = (12, 12, 1)
GRID = (468, 468, 1)
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
REL = 1e-3          # the fp32 contract: max-norm against the output's max-abs
# per row.  Measured on an H100 80GB HBM3 (700 W power limit): at most 5.15e-6 of a row's max-abs over every case of this file
# but the LayerNorm shift (192 x 12 heads x 384, post-norm BatchNorm ReLU), so TIGHT = 2e-5 leaves a margin of about 4x
TIGHT = 2e-5
# rows that enter a LayerNorm at +1024 are formed in fp32, whose ulp there (2^-13 = 1.2e-4) is the floor for a unit-variance
# row's normalised output; measured at most 1.22e-4 (FFMA family), so 5e-4.  A one-pass E[t^2] - mean^2 variance misses by percent
SHIFT_TIGHT = 5e-4
SSTB_ERR_UNSUPPORTED = -3   # csrc/common.cuh
ODD = "odd_tiles"   # (2 x SMs + 2) 128-row tiles, the last one partial
SENTINEL = 7.0

# (d_model, heads, dim_ff) -> route family
SHAPES = {
    (128, 8, 256): "x3",      # every GEMM on x3
    (64, 4, 128): "x3",       # K = 64: one stage; N = 64: NT 64
    (192, 12, 384): "x3",     # N = 192: NT 64, K = 192: three stages
    (128, 8, 320): "x3",      # K = 320: five stages (odd); N = 320: NT 64
    (256, 8, 512): "x3",      # add_norm_kernel's v[8] full
    (128, 8, 96): "mixed",    # q|k|v FFMA with fused pos, out_proj x3, linear1 / linear2 FFMA
    (128, 8, 100): "mixed",   # the same with N and K tails of 36 and 4
    (96, 6, 192): "ffma",
    (160, 10, 320): "ffma",
    (32, 2, 64): "ffma",
}
FAMILY_SHAPE = {"x3": (128, 8, 256), "mixed": (128, 8, 100), "ffma": (96, 6, 192)}

# name -> (layer_cfg, activation); every variant meets every route family (test_route_variant)
VARIANTS = {
    "post_ln_gelu": ({}, "gelu"),
    "post_ln_relu": ({}, "relu"),
    "post_bn_gelu": (dict(use_bn=True), "gelu"),
    "post_bn_relu": (dict(use_bn=True), "relu"),
    "pre_ln_gelu": (dict(post_norm=False), "gelu"),
    "pre_ln_relu": (dict(post_norm=False), "relu"),
    "pre_bn_gelu": (dict(post_norm=False, use_bn=True), "gelu"),
    "pre_bn_relu": (dict(post_norm=False, use_bn=True), "relu"),
    "cosine_tau_per_head": (dict(cosine=True, non_shared_tau=True, tau_min=0.01), "gelu"),
}


# ------------------------------------------------------------------------------------------------------------------------------
# routes, mirrored from the dispatch of csrc/sra_fp32.cu and csrc/spconv.cu
# ------------------------------------------------------------------------------------------------------------------------------
def _x3(N, K):
    """sstb_row_gemm_x3's route for an [N, K] weight, or None when it refuses the shape (the FFMA kernel runs)."""
    if N % 64 or K % 64:
        return None
    return ("x3", 128 if N % 128 == 0 else 64, K // 64)


def gemm_routes(d, ff):
    """Route of every GEMM of sstb_sra_layer_fp32: ("x3", NT, stages), "ffma" or "ffma_pos" (positional term fused)."""
    lin = lambda N, K: _x3(N, K) or "ffma"
    if d % 64 == 0 and ff % 64 == 0:
        qkv = {"qk": lin(2 * d, d), "v": lin(d, d)}
    else:
        qkv = {"qkv": "ffma_pos"}
    return dict(qkv, out_proj=lin(d, d), linear1=lin(ff, d), linear2=lin(d, ff))


def family(d, ff):
    kinds = {r if isinstance(r, str) else "x3" for r in gemm_routes(d, ff).values()}
    return "x3" if kinds == {"x3"} else "ffma" if "x3" not in kinds else "mixed"


def test_row_gemm_route_matrix():
    """CPU: the dispatch rules the route mirror restates are still the ones in the sources, and the shape matrix reaches every
    route the issue of each shape claims: both x3 tile widths, 1 / 2 / 3 / 4 / 5 / 8 stages, the fused-pos FFMA q|k|v beside x3
    GEMMs in one layer, FFMA with N and K tails, and d_model 256 (v[8] full)."""
    fp32 = open(os.path.join(ROOT, "sst_b200", "csrc", "sra_fp32.cu")).read()
    spc = open(os.path.join(ROOT, "sst_b200", "csrc", "spconv.cu")).read()
    assert "if (d % 64 == 0 && ff % 64 == 0) {" in fp32
    qkv = fp32[fp32.index("} else {  // q|k|v in one FFMA GEMM"):]
    qkv = qkv[:qkv.index("sstb_row_gemm(st, g);")]
    assert "g.A = xin, g.lda = d, g.W = L->in_proj_w," in qkv and "g.N = 3 * d, g.K = d;" in qkv, "q|k|v in one FFMA GEMM"
    assert "g.pos = pt, g.pos_ncols = 2 * d;" in qkv, "q|k|v FFMA: pos_ncols = 2 d"
    assert "static int linear_fp32(sstb200_ctx* c, const RowGemm& g) {\n  const int rc = sstb_row_gemm_x3(c, g);" in fp32
    assert "if (d > 256 || d % 32)" in fp32
    x3 = spc[spc.index("int sstb_row_gemm_x3("):]
    x3 = x3[:x3.index("\n}\n")]
    assert "if ((K & 63) || (N & 63) || (r.lda & 3) || (r.ldo & 3) || (r.ldr & 3) || (r.act == 1 && r.res))" in x3
    assert "if ((r.ldw && r.ldw != K) || r.res_index || r.pos.tab) return SSTB_ERR_UNSUPPORTED;" in x3
    assert "dispatch_spconv_wgmma(c, g, true)" in x3
    assert "if (g.Cout % 128 == 0) return launch_spconv_wgmma<128, 2, true>(c, g);" in spc
    for shape, fam in SHAPES.items():
        assert family(shape[0], shape[2]) == fam, shape
    r = {s: gemm_routes(s[0], s[2]) for s in SHAPES}
    assert r[(128, 8, 256)] == dict(qk=("x3", 128, 2), v=("x3", 128, 2), out_proj=("x3", 128, 2), linear1=("x3", 128, 2),
                                     linear2=("x3", 128, 4))
    assert r[(64, 4, 128)]["v"] == ("x3", 64, 1) and r[(64, 4, 128)]["linear1"] == ("x3", 128, 1)
    assert r[(192, 12, 384)]["out_proj"] == ("x3", 64, 3) and r[(192, 12, 384)]["qk"] == ("x3", 128, 3)
    assert r[(128, 8, 320)]["linear1"] == ("x3", 64, 2) and r[(128, 8, 320)]["linear2"] == ("x3", 128, 5)
    assert r[(256, 8, 512)]["linear2"] == ("x3", 128, 8)
    for ff in (96, 100):
        assert r[(128, 8, ff)] == dict(qkv="ffma_pos", out_proj=("x3", 128, 2), linear1="ffma", linear2="ffma")
    assert (100 % 64, 100 % 16) == (36, 4)
    for s in ((96, 6, 192), (160, 10, 320), (32, 2, 64)):
        assert set(r[s].values()) == {"ffma_pos", "ffma"}
    assert max(d for d, _, _ in SHAPES) == 256
    # every variant meets every family in test_route_variant
    for fam in FAMILY_SHAPE:
        assert {v for s, v in _variant_cases() if SHAPES[s] == fam} == set(VARIANTS)


def _variant_cases():
    """Each shape with the base variant; the other variants spread over the shapes of each family."""
    cases = [(s, "post_ln_gelu") for s in SHAPES]
    for fam in FAMILY_SHAPE:
        shapes = [s for s in SHAPES if SHAPES[s] == fam]
        cases += [(shapes[i % len(shapes)], v) for i, v in enumerate(list(VARIANTS)[1:])]
    return cases


# ------------------------------------------------------------------------------------------------------------------------------
# the x3 operand split, emulated: why the kernel scales its operands
# ------------------------------------------------------------------------------------------------------------------------------
def _f16(x):
    """fp32 -> fp16, round to nearest even, saturating to +-65504 (cvt.rn.satfinite.f16)"""
    return np.clip(x, -65504.0, 65504.0).astype(np.float16)


def _pow2_top(amax):
    """the power of two that puts amax in [2^13, 2^14), as sp_row_exp_kernel / split_f16_rows_kernel take it (frexp convention)"""
    _, e = np.frexp(amax.astype(np.float32))
    return np.clip(14 - e, -100, 100).astype(np.float64)


def x3_emulated(a, w, scaled):
    """out = a . w^T as sstb_row_gemm_x3 forms it: each operand element split into hi = fp16(x), lo = fp16(x - hi) (after the
    row's / output channel's power of two when `scaled`), the three products hi.hi + lo.hi + hi.lo summed exactly (float64)."""
    a, w = a.astype(np.float32), w.astype(np.float32)
    ea = _pow2_top(np.abs(a).max(1)) if scaled else np.zeros(a.shape[0])
    ew = _pow2_top(np.abs(w).max(1)) if scaled else np.zeros(w.shape[0])
    a_s, w_s = np.ldexp(a, ea[:, None].astype(int)).astype(np.float32), np.ldexp(w, ew[:, None].astype(int)).astype(np.float32)

    def split(x):
        hi = _f16(x)
        return hi.astype(np.float64), _f16(x - hi.astype(np.float32)).astype(np.float64)

    ah, al = split(a_s)
    wh, wl = split(w_s)
    out = ah @ wh.T + al @ wh.T + ah @ wl.T
    return np.ldexp(np.ldexp(out, -ea[:, None].astype(int)), -ew[None, :].astype(int))


def _row_err(got, ref):
    return float((np.abs(got - ref).max(1) / np.abs(ref).max(1)).max())


def test_x3_split_operand_scale_emulated():
    """CPU: the rounding of the x3 GEMM's operands on the scale cases of test_operand_scale.  With each row of A and each output
    channel of W lifted to the top of fp16's range (what sstb_row_gemm_x3 does), the split keeps every row of A . W^T within
    2^-20 of its max-abs at every scale - 22 bits per element, accumulated over K.  Converted as they are, the pair has no
    normal fp16 residue below about 2^-3, where the weights of an encoder layer lie (xavier: |w| <= 0.18 for these shapes):
    activations x 2^-8 and below and any weight matrix x 2^-6 leave that bound, and from 2^-12 on (or w x 2^-6) the layer's
    TIGHT too, which is why the kernel scales."""
    g = np.random.default_rng(0)
    K, N = 256, 128
    a0 = g.standard_normal((512, K)).astype(np.float32)
    bound = np.sqrt(6.0 / (K + N))    # xavier_uniform_, as SSTv2 initialises every weight matrix
    w0 = g.uniform(-bound, bound, (N, K)).astype(np.float32)
    cases = {f"a x 2^{k}": (np.ldexp(a0, k), w0) for k in (-16, -12, -8, 0, 8)}
    cases["w x 2^-6"] = (a0, np.ldexp(w0, -6))
    cases["w in [2^-3, 1)"] = (a0, np.sign(w0) * (0.125 + np.abs(w0) * 7))
    cases["a x 2^-12, w x 2^-6"] = (np.ldexp(a0, -12), np.ldexp(w0, -6))
    bound20 = 2.0 ** -20
    unscaled = {}
    for name, (a, w) in cases.items():
        ref = a.astype(np.float64) @ w.astype(np.float64).T
        e = _row_err(x3_emulated(a, w, True), ref)
        assert e <= bound20, (name, e)
        unscaled[name] = _row_err(x3_emulated(a, w, False), ref)
    print({k: f"{v:.2e}" for k, v in unscaled.items()})
    # unscaled, operands at or above 2^-3 keep the bound; below it the pair leaves it (measured: 7.4e-6 at a x 2^-8), from 2^-12
    # on it leaves the layer's tight bound as well (1.3e-4 at 2^-12, 3.0e-5 for w x 2^-6) and at 2^-16 the fp32 contract (2.3e-3)
    assert unscaled["w in [2^-3, 1)"] <= bound20
    assert unscaled["a x 2^-8"] > 4 * bound20
    for name in ("a x 2^-12", "a x 2^-16", "w x 2^-6", "a x 2^-12, w x 2^-6"):
        assert unscaled[name] > TIGHT, (name, unscaled[name])
    assert unscaled["a x 2^-16"] > REL
    # scaled results are homogeneous in the scale of either operand, to the last bit
    for k in (-16, -8, 8):
        assert np.array_equal(x3_emulated(np.ldexp(a0, k), w0, True), np.ldexp(x3_emulated(a0, w0, True), k))


# ------------------------------------------------------------------------------------------------------------------------------
# models, inputs, float64 oracle, error accounting
# ------------------------------------------------------------------------------------------------------------------------------
def _voxels(n, d, seed, scale=1.0):
    """n distinct voxels of one sweep: a 12 x 12 window holds at most 144, so no voxel is dropped and the layer sees n rows."""
    g = torch.Generator().manual_seed(seed)
    cell = torch.randperm(GRID[0] * GRID[1], generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), cell // GRID[0], cell % GRID[0]], 1).int()
    return torch.randn(n, d, generator=g) * scale, coors


def _model(shape, variant, blocks=1, seed=0, edit="random"):
    """SSTv2 of `blocks` blocks at `shape` with `variant`.  edit "random": non-trivial biases, norms, BN running statistics and
    temperatures; "zero_bias": every bias (Linear and norm) zeroed, so that an input scale reaches every GEMM operand; "init":
    the modules' own initialisation (xavier weights, default biases) left as it is."""
    from sst_b200.sst_modules import SSTv2
    d, h, ff = shape
    lc, act = VARIANTS[variant]
    torch.manual_seed(seed)
    m = SSTv2(d_model=[d] * blocks, nhead=[h] * blocks, num_blocks=blocks, dim_feedforward=[ff] * blocks, output_shape=[468, 468],
              num_attached_conv=0, to_bev=False, layer_cfg=lc, activation=act).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("tau"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.5 + 0.05)
            elif p.dim() == 1 and edit == "random":
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            elif p.dim() == 1 and edit == "zero_bias" and n_.endswith("bias"):
                p.zero_()
        if edit != "init":
            for n_, b in m.named_buffers():
                if "running_mean" in n_:
                    b.copy_(torch.randn(b.shape, generator=g) * 0.3 if edit == "random" else torch.zeros_like(b))
                if "running_var" in n_:   # down to 0.02, where BatchNorm's eps (1e-5) moves the result by 2.5e-4
                    b.copy_(torch.rand(b.shape, generator=g) + 0.02)
    return m


def _layers(m):
    return [l for blk in m.block_list for l in blk.encoder_list]


def _info(cuda, feats, coors):
    from sst_b200.sst_modules import SSTInputLayerV2
    il = SSTInputLayerV2((DROP_TEST, DROP_TEST), WIN, GRID, shuffle_voxels=False, mute=True).eval()
    with torch.no_grad():
        return il(feats.to(cuda), coors.to(cuda), 1)


def _oracle64(m, variant, feats, coors, num_layers=1):
    """float64 oracle of the first `num_layers` encoder layers of m (shift i % 2 for layer i)."""
    w = {k: v.detach().double() for k, v in m.state_dict().items()}
    info = O.input_layer_v2(feats.double(), coors, DROP_TEST, WIN, GRID)
    assert info["voxel_feats"].shape[0] == feats.shape[0]
    l0 = _layers(m)[0]
    lc = VARIANTS[variant][0]
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


def check(got, ref, what, tight=TIGHT):
    """fp32 contract (max-norm REL) and the per-row `tight` bound; returns the worst per-row error over its bound's scale."""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    amax = ref.abs().max().item()
    err_max = (got - ref).abs().max().item() / amax
    row_scale = torch.clamp(ref.abs().amax(1), min=1e-3 * amax)
    row = (got - ref).abs().amax(1) / row_scale
    worst = row.max().item()
    print(f"TIGHT-MEASURE {what}: per-row {worst:.3e} (row {int(row.argmax())}), max-norm {err_max:.3e}")
    assert err_max < REL, f"{what}: max-norm error {err_max:.3e} above the fp32 contract {REL:g}"
    bad = (row > tight).nonzero().flatten()
    assert bad.numel() == 0, (f"{what}: {bad.numel()} of {row.numel()} rows above {tight:g}; worst {worst:.3e} at row "
                              f"{int(row.argmax())}, first bad rows {bad[:8].tolist()}")
    return worst


def _lib():
    from sst_b200 import _lib as L
    return L


def _layer_call(c, layer, plan, x, y, n, n_dev=None):
    """sstb200_sra_layer_forward(precision fp32); returns its status without raising"""
    from sst_b200.sst_modules import PRECISIONS, make_sra_plan
    ls, ps = layer._struct(PRECISIONS["fp32"]), make_sra_plan(plan)
    return _lib().lib().sstb200_sra_layer_forward(c, C.byref(ls), C.byref(ps), x.data_ptr(), y.data_ptr(), n,
                                                  None if n_dev is None else n_dev.data_ptr(), PRECISIONS["fp32"])


def _run_layer(cuda, m, info, c=None):
    """first encoder layer of m on info's shift-0 plan, n == capacity"""
    L = _lib()
    c = c or L.ctx(cuda)
    x = info["voxel_feats"].float().contiguous()
    y = torch.empty_like(x)
    L.check(c, _layer_call(c, _layers(m)[0], info["sra_plan_shift0"], x, y, x.shape[0]))
    torch.cuda.synchronize()
    return y


def _padded(x, cap, fill):
    out = torch.full((cap, x.shape[1]), fill, dtype=torch.float32, device=x.device)
    out[:x.shape[0]] = x
    return out


def _case(cuda, shape, variant, n, seed, scale=1.0, **kw):
    feats, coors = _voxels(n, shape[0], seed, scale)
    m = _model(shape, variant, **kw)
    ref = _oracle64(m, variant, feats, coors)
    m = m.to(cuda)
    return m, _info(cuda, feats, coors), ref


# ------------------------------------------------------------------------------------------------------------------------------
# routes x variants, row counts
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape,variant", _variant_cases(), ids=[f"{s[0]}x{s[1]}x{s[2]}-{v}" for s, v in _variant_cases()])
def test_route_variant(cuda, shape, variant):
    """One fp32 layer per (shape, variant) at 517 rows (four full 128-row tiles and a partial one)."""
    m, info, ref = _case(cuda, shape, variant, 517, seed=_variant_cases().index((shape, variant)))
    check(_run_layer(cuda, m, info), ref, f"{shape} {variant}")


@pytest.mark.gpu
@pytest.mark.parametrize("fam", list(FAMILY_SHAPE))
@pytest.mark.parametrize("n", [1, 7, 8, 9, 63, 64, 65, 127, 128, 129, 255, 257, ODD])
def test_row_counts(cuda, n, fam):
    """Row counts on the edges of the 128-row tiles of both GEMMs, the 8-row blocks of the row-exponent and norm kernels and
    (2 x SMs + 2) tiles; post-norm LayerNorm GELU for n <= 129, pre-norm BatchNorm ReLU above."""
    n = _rows(n)
    variant = "post_ln_gelu" if n <= 129 else "pre_bn_relu"
    m, info, ref = _case(cuda, FAMILY_SHAPE[fam], variant, n, seed=n)
    check(_run_layer(cuda, m, info), ref, f"{fam} n {n} {variant}")


# ------------------------------------------------------------------------------------------------------------------------------
# device row count, in place, dirty arena, stack
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["pre_ln_gelu", "post_bn_relu"])
@pytest.mark.parametrize("fam", list(FAMILY_SHAPE))
def test_device_row_count(cuda, fam, variant):
    """Row count read from device memory, buffers 200 rows larger, y prefilled with a sentinel: rows past the count keep it and
    the result is bit-identical to the call with n == capacity; also in place (y == x).  In the pre-norm layer the last write to
    y is linear2's GEMM itself (residual t1), so only there would a GEMM that ignores the device count show."""
    L = _lib()
    n = 333
    m, info, ref = _case(cuda, FAMILY_SHAPE[fam], variant, n, seed=5)
    exact = _run_layer(cuda, m, info)
    check(exact, ref, f"{fam} {variant} n == capacity")
    c, cap = L.ctx(cuda), n + 200
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    x = _padded(info["voxel_feats"].float(), cap, 3.0)
    y = torch.full_like(x, SENTINEL)
    L.check(c, _layer_call(c, _layers(m)[0], info["sra_plan_shift0"], x, y, cap, n_dev))
    torch.cuda.synchronize()
    assert (y[n:] == SENTINEL).all(), f"rows past the device count written: {(y[n:] != SENTINEL).any(1).sum().item()}"
    assert torch.equal(y[:n], exact)
    assert (x[n:] == 3.0).all() and torch.equal(x[:n], info["voxel_feats"].float())
    L.check(c, _layer_call(c, _layers(m)[0], info["sra_plan_shift0"], x, x, cap, n_dev))
    torch.cuda.synchronize()
    assert torch.equal(x[:n], exact), "in place (y == x) differs"
    assert (x[n:] == 3.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("fam", list(FAMILY_SHAPE))
def test_dirty_arena(cuda, fam):
    """A 'poison twin' (300 more rows, features x 1e4) runs first on the same context and leaves its temporaries in the arena;
    the real call, twice, is bit-identical to itself and to the call on a fresh context."""
    L = _lib()
    shape = FAMILY_SHAPE[fam]
    n = 300
    m, info, ref = _case(cuda, shape, "pre_ln_gelu", n, seed=11)
    feats_p, coors_p = _voxels(n + 300, shape[0], 12, 1e4)
    info_p = _info(cuda, feats_p, coors_p)
    lib = L.lib()
    fresh = lib.sstb200_create(cuda.index or 0)
    assert fresh
    try:
        lib.sstb200_set_stream(fresh, torch.cuda.current_stream(cuda).cuda_stream)
        clean = _run_layer(cuda, m, info, c=fresh)
    finally:
        torch.cuda.synchronize()
        lib.sstb200_destroy(fresh)
    c = L.ctx(cuda)
    _run_layer(cuda, m, info_p, c=c)
    a = _run_layer(cuda, m, info, c=c)
    b = _run_layer(cuda, m, info, c=c)
    assert torch.equal(a, b) and torch.equal(a, clean)
    check(a, ref, f"{fam} after a poison twin")


@pytest.mark.gpu
@pytest.mark.parametrize("num_layers", [1, 2, 3])
def test_stack(cuda, num_layers):
    """sstb200_sra_stack_forward(precision fp32) with 1, 2, 3 layers (odd counts start in y, even ones in tmp) and a device row
    count below capacity: bit-identical to the layers called one by one, rows of y past the count untouched."""
    from sst_b200.sst_modules import PRECISIONS, _SraLayer, make_sra_plan
    L = _lib()
    shape, n = FAMILY_SHAPE["x3"], 271
    feats, coors = _voxels(n, shape[0], 21)
    m = _model(shape, "pre_ln_gelu", blocks=2)
    ref = _oracle64(m, "pre_ln_gelu", feats, coors, num_layers)
    m = m.to(cuda)
    info = _info(cuda, feats, coors)
    layers = _layers(m)[:num_layers]
    plans = [info["sra_plan_shift0"], info["sra_plan_shift1"]]
    c = L.ctx(cuda)
    out = info["voxel_feats"].float().contiguous()
    for i, l in enumerate(layers):
        nxt = torch.empty_like(out)
        L.check(c, _layer_call(c, l, plans[i % 2], out, nxt, n))
        out = nxt
    torch.cuda.synchronize()
    check(out, ref, f"{num_layers} layers one by one")
    cap = n + 200
    arr = (_SraLayer * num_layers)(*[l._struct(PRECISIONS["fp32"]) for l in layers])
    p0, p1 = make_sra_plan(plans[0]), make_sra_plan(plans[1])
    x = _padded(info["voxel_feats"].float(), cap, 3.0)
    y, tmp = torch.full_like(x, SENTINEL), torch.full_like(x, -SENTINEL)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    L.check(c, L.lib().sstb200_sra_stack_forward(c, arr, num_layers, C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(),
                                                 tmp.data_ptr(), cap, n_dev.data_ptr(), PRECISIONS["fp32"]))
    torch.cuda.synchronize()
    assert torch.equal(y[:n], out)
    assert (y[n:] == SENTINEL).all() and (tmp[n:] == -SENTINEL).all()
    assert (x[n:] == 3.0).all() and torch.equal(x[:n], info["voxel_feats"].float())


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm shift, refusals, the engine
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fam", list(FAMILY_SHAPE))
def test_layernorm_shift(cuda, fam):
    """out_proj.bias and linear2.bias + 1024: the rows entering both post-norm LayerNorms carry a common offset of 1024, where a
    one-pass E[t^2] - mean^2 variance loses its bits; the two-pass statistics hold SHIFT_TIGHT, fp32's own floor at 1024."""
    shape = FAMILY_SHAPE[fam]
    feats, coors = _voxels(401, shape[0], 31)
    m = _model(shape, "post_ln_gelu")
    with torch.no_grad():
        for l in _layers(m):
            l.win_attn.self_attn.out_proj.bias.add_(1024.0)
            l.linear2.bias.add_(1024.0)
    ref = _oracle64(m, "post_ln_gelu", feats, coors)
    m = m.to(cuda)
    check(_run_layer(cuda, m, _info(cuda, feats, coors)), ref, f"{fam} LayerNorm shift +1024", SHIFT_TIGHT)


@pytest.mark.gpu
@pytest.mark.parametrize("d,h,code", [(288, 8, SSTB_ERR_UNSUPPORTED), (80, 4, SSTB_ERR_UNSUPPORTED)])
def test_refused_widths(cuda, d, h, code):
    """d_model 288 (more than add_norm_kernel's 8 values per lane) and 80 (not a multiple of 32) are refused with
    SSTB_ERR_UNSUPPORTED, and no output row is written."""
    L = _lib()
    feats, coors = _voxels(100, d, 41)
    m = _model((d, h, 2 * d), "post_ln_gelu").to(cuda)
    info = _info(cuda, feats, coors)
    x = info["voxel_feats"].float().contiguous()
    y = torch.full_like(x, SENTINEL)
    c = L.ctx(cuda)
    rc = _layer_call(c, _layers(m)[0], info["sra_plan_shift0"], x, y, x.shape[0])
    torch.cuda.synchronize()
    assert rc == code, rc
    assert "d_model" in L.lib().sstb200_last_error(c).decode()
    assert (y == SENTINEL).all()
    with pytest.raises(L.SSTB200Error):
        with torch.no_grad():
            _layers(m)[0](x, info["sra_plan_shift0"], "fp32")


@pytest.mark.gpu
def test_engine_fp32(cuda):
    """SSTEngine(precision='fp32') on the flagship configuration (2 blocks, batch of 2 frames, capacity-sized buffers, device row
    count), as test_engine_matches_oracle runs it: every row within TIGHT of the float64 oracle of the whole path."""
    from sst_b200 import flagship as fl
    from sst_b200.engine import SSTEngine
    cfg = fl.sst_cfg(num_blocks=2)
    vfe, il, bb = fl.build_sst(cfg)
    pts_list = [O.synth_frame(70 + b, 12000) for b in range(2)]
    coors = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(p, fl.VOXEL_SIZE, fl.PC_RANGE), (1, 0), value=b)
                       for b, p in enumerate(pts_list)])
    wv = {k: v.double() for k, v in vfe.state_dict().items()}
    vf, vc = O.dynamic_vfe_forward(torch.cat(pts_list).double(), coors, wv, fl.VOXEL_SIZE, fl.PC_RANGE, 2)
    info = O.input_layer_v2(vf, vc, fl.DROP_TEST, fl.WINDOW_SHAPE, (468, 468, 1))
    wb = {k: v.double() for k, v in bb.state_dict().items()}
    ref = O.sstv2_forward(info, wb, cfg['backbone']['nhead'], cfg['backbone']['num_blocks'])
    eng = SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe.to(cuda), il, bb.to(cuda), max_points=30000, batch_size=2, precision="fp32",
                    device=cuda)
    eng.load_frames_device(torch.cat(pts_list).to(cuda), torch.tensor([0, 12000, 24000], dtype=torch.int32, device=cuda))
    feats, co, num = eng.run()
    torch.cuda.synchronize()
    M = int(num.item())
    assert M == vc.shape[0] and torch.equal(co[:M].cpu(), vc)
    check(feats[:M], ref, "engine fp32, flagship 2 blocks")


# ------------------------------------------------------------------------------------------------------------------------------
# operand scale
# ------------------------------------------------------------------------------------------------------------------------------
WEIGHTS = {"in_proj": lambda l: l.win_attn.self_attn.in_proj_weight, "out_proj": lambda l: l.win_attn.self_attn.out_proj.weight,
           "linear1": lambda l: l.linear1.weight, "linear2": lambda l: l.linear2.weight}
SCALES = [f"input_2^{k}" for k in (-16, -12, -8, 0, 8)] + [f"{w}_2^-6" for w in WEIGHTS] + ["default_init"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SCALES)
@pytest.mark.parametrize("fam", ["x3", "ffma"])
def test_operand_scale(cuda, fam, case):
    """Input features x 2^k with every bias zeroed (the scale reaches every GEMM operand: post-norm, x feeds q|k|v directly and
    its scale passes through attention into out_proj), each weight matrix x 2^-6 in turn, and the modules' own init (xavier
    weights, |w| <= 0.18, and default biases) left as it is.  The x3 GEMM scales each operand row / channel to the top of fp16's
    range, so every case holds the tight bound; converted as they are, these operands lose bits in fp16 (see
    test_x3_split_operand_scale_emulated)."""
    shape = FAMILY_SHAPE[fam]
    scale, edit = 1.0, "random"
    if case.startswith("input_"):
        scale, edit = 2.0 ** int(case.split("^")[1]), "zero_bias"
    elif case == "default_init":
        edit = "init"
    feats, coors = _voxels(389, shape[0], 51, scale)
    m = _model(shape, "post_ln_gelu", edit=edit)
    if case.endswith("_2^-6") and not case.startswith("input_"):
        with torch.no_grad():
            for l in _layers(m):
                WEIGHTS[case.split("_2^")[0]](l).mul_(2.0 ** -6)
    if case == "default_init":
        for l in _layers(m):   # xavier_uniform_, unedited: |w| <= sqrt(6 / (fan_in + fan_out)), 0.108 .. 0.177 here
            assert all(WEIGHTS[k](l).abs().max().item() <= (6.0 / sum(WEIGHTS[k](l).shape)) ** 0.5 for k in WEIGHTS)
    ref = _oracle64(m, "post_ln_gelu", feats, coors)
    m = m.to(cuda)
    check(_run_layer(cuda, m, _info(cuda, feats, coors)), ref, f"{fam} {case}")
