"""The deformable convolution (csrc/dcn.cu, ops.deform_conv2d, DeformConv2d / DeformConv2dPack) against the float64 oracle
(oracle/dcn_oracle.py) at every tile, split and axis edge, forward and backward.

Where the kernels can go wrong:
    axes          kh / kw, sh / sw, ph / pw and dh / dw enter separately (the ki / kj split of a tap, the Ho / Wo formulas, the offset pair
                  h at 2k, w at 2k + 1); every asymmetric axis is run on its own from one symmetric base
    forward tiles BN = 16 / 32 / 64 outputs from Og = Cout / groups, BM = 4096 / BN = 256 / 128 / 64 pixels per block; each BN at
                  NP = BM - 1, BM, BM + 1 and over several tiles that straddle images, every Og edge of BN and of the output tiles
    reduction     R = Cg K around the 16-deep staged slice
    grad_weight   split-K over 2048-pixel chunks, staged 64 pixels at a time: NP = 2047, 2048, 2049, 2 * 2048 + 65 at each BN
    lane loops    grad_offset and grad_x loop lanes over the Cd = Cin / dg channels of a deformable group: Cd = 1 .. 96, with conv
                  groups and deformable groups that do not nest
    sort width    grad_x radix-sorts keys below N dg H W + 1: N dg H W = 255, 256, 257 around the 8-bit end_bit
    offsets       normal, large, whole-pixel, zero; positions exactly at -1, nextafter(-1, 0), L - 1, nextafter(L - 1, L) and
                  nextafter(L, 0) (one fp32 addition, as the kernel forms them); NaN and +-inf (the sample adds 0 and gets a zero offset
                  gradient); every sample of every pixel on one input pixel (one long run of the sorted keys)
Bounds per element, relative to the float64 sum of the absolute values of the terms that element adds: 1e-5 for y, grad_x and
grad_offset, 1e-4 for grad_weight.  Through the C ABI with caller-owned, NaN-prefilled and guarded outputs: every element written, nothing
written past the end, untouched input pixels and invalid samples exactly 0, a workspace of 0xFF bytes gives the bits of a zeroed one,
every subset of the three gradients the bits of the full call.  The limits are checked through the workspace size query only.

The oracle itself is pinned to torchvision.ops.deform_conv2d in float64 on the asymmetric grid first (CPU).  The worst observed
error / bound ratio per quantity is printed when the module finishes (visible with `pytest -s`)."""
import ctypes
import json
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dcn_oracle as D

dev = torch.device("cuda:0")
OBSERVED = {}
GUARD = 16
POISON = 0x7FC0DEAD  # a quiet NaN whose payload no arithmetic produces: a guard that still holds it was not written
RTOL = dict(y=1e-5, grad_x=1e-5, grad_offset=1e-5, grad_weight=1e-4)


def _case(N, C, H, W, O, k=(3, 3), s=(1, 1), p=(1, 1), d=(1, 1), G=1, dg=1):
    return (N, C, H, W, O, tuple(k), tuple(s), tuple(p), tuple(d), G, dg)


def _out(c):
    N, C, H, W, O, k, s, p, d, G, dg = c
    return D.out_size(H, W, k, s, p, d)


# --- axes: each asymmetric kernel / stride / padding / dilation on its own from one symmetric base (G = 2 and dg = 3 do not nest)
BASE = _case(2, 6, 11, 9, 8, G=2, dg=3)
AXES = {
    "k13": _case(2, 6, 11, 9, 8, k=(1, 3), G=2, dg=3),
    "k31": _case(2, 6, 11, 9, 8, k=(3, 1), G=2, dg=3),
    "k23": _case(2, 6, 11, 9, 8, k=(2, 3), G=2, dg=3),
    "k53": _case(2, 6, 11, 9, 8, k=(5, 3), G=2, dg=3),
    "s12": _case(2, 6, 11, 9, 8, s=(1, 2), G=2, dg=3),
    "s21": _case(2, 6, 11, 9, 8, s=(2, 1), G=2, dg=3),
    "p02": _case(2, 6, 11, 9, 8, p=(0, 2), G=2, dg=3),
    "d13": _case(2, 6, 11, 9, 8, d=(1, 3), G=2, dg=3),
    "d21": _case(2, 6, 11, 9, 8, d=(2, 1), G=2, dg=3),
    "hw13x1": _case(2, 6, 13, 1, 8, G=2, dg=3),           # Ho Wo = 13, prime
    "hw1x17": _case(1, 6, 1, 17, 8, G=2, dg=3),           # Ho Wo = 17, prime
    "mixed": _case(1, 8, 10, 13, 12, k=(2, 3), s=(2, 1), p=(0, 2), d=(1, 2), G=4, dg=2),
}
assert all(_out(c)[0] * _out(c)[1] in (13, 17) for c in (AXES["hw13x1"], AXES["hw1x17"]))

# --- forward tiles: every Og edge of BN 16 / 32 / 64 and of the output tiles (otiles > 1 with a partial last tile)
OG = {og: _case(2, 4, 9, 7, og * G, G=G) for og, G in ((1, 2), (15, 1), (16, 1), (17, 2), (31, 1), (32, 1), (33, 1), (63, 1),
                                                        (64, 1), (65, 2), (129, 1))}
# each BN at NP = BM - 1, BM, BM + 1, and over several BM-pixel tiles that straddle images (Ho Wo not a multiple of BM, N >= 3)
TILES = {
    "bn16_np255": _case(1, 4, 15, 17, 16), "bn16_np256": _case(2, 4, 8, 16, 16), "bn16_np257": _case(1, 4, 257, 1, 16),
    "bn16_np1173": _case(3, 4, 17, 23, 16),
    "bn32_np127": _case(1, 4, 127, 1, 32), "bn32_np128": _case(1, 4, 8, 16, 32), "bn32_np129": _case(1, 4, 3, 43, 32),
    "bn32_np297": _case(3, 4, 11, 9, 32),
    "bn64_np63": _case(1, 4, 7, 9, 64), "bn64_np64": _case(1, 4, 4, 16, 64), "bn64_np65": _case(1, 4, 5, 13, 64),
    "bn64_np140": _case(4, 4, 5, 7, 64),
}
for _k, _c in TILES.items():
    assert _c[0] * _out(_c)[0] * _out(_c)[1] == int(_k.split("np")[1]), _k
# --- reduction depth R = Cg K around the 16-deep slice
DEPTH = {
    "r15": _case(2, 5, 7, 6, 8, k=(1, 3)), "r16": _case(2, 16, 7, 6, 8, k=(1, 1), p=(0, 0)),
    "r17": _case(2, 17, 7, 6, 8, k=(1, 1), p=(0, 0)), "r144": _case(2, 16, 7, 6, 8), "r145": _case(2, 29, 7, 6, 8, k=(1, 5), p=(0, 2)),
}
# --- grad_weight split-K: NP = 2047, 2048, 2049, 2 * 2048 + 65 at each BN; the chunk boundaries of 2049 and 4161 fall inside images
SPLITS = {}
for _og in (16, 32, 64):
    for _np, (_n, _h, _w) in ((2047, (1, 23, 89)), (2048, (2, 16, 64)), (2049, (1, 3, 683)), (4161, (3, 19, 73))):
        SPLITS[f"og{_og}_np{_np}"] = _case(_n, 4, _h, _w, _og)
        assert _n * _h * _w == _np
# --- lane loops over Cd = Cin / dg channels; (G, dg) = (2, 3), (3, 2), (4, 2), (5, 2) do not nest
LANES = {
    "cd1": _case(1, 6, 6, 5, 4, G=2, dg=6), "cd31": _case(1, 62, 6, 5, 4, G=2, dg=2), "cd32": _case(1, 96, 6, 5, 6, G=2, dg=3),
    "cd33": _case(1, 66, 6, 5, 6, G=3, dg=2), "cd48": _case(1, 96, 6, 5, 8, G=4, dg=2), "cd65": _case(1, 130, 6, 5, 10, G=5, dg=2),
    "cd96": _case(1, 192, 6, 5, 8, G=4, dg=2),
}
# --- N dg H W around the sort's 8-bit end_bit (keys 0 .. N dg H W, the last one 'no pixel')
SORT = {"px255": _case(1, 2, 15, 17, 2), "px256": _case(2, 4, 8, 8, 2, dg=2), "px257": _case(1, 2, 1, 257, 2)}
OFFSET_GEOMS = {"base": BASE, "mixed": AXES["mixed"]}
OFFSET_MODES = ("normal", "large", "integer", "zero", "exact", "nonfinite", "collapsed")


def _seed(*parts):
    return zlib.crc32("/".join(map(str, parts)).encode())


def _bases(c):
    """fp32 integer bases of the sample positions, h [K, Ho, 1] and w [K, 1, Wo]"""
    N, C, H, W, O, (kh, kw), (sh, sw), (ph, pw), (dh, dw), G, dg = c
    Ho, Wo = _out(c)
    K = kh * kw
    ki = torch.arange(kh).repeat_interleave(kw).view(K, 1, 1)
    kj = torch.arange(kw).repeat(kh).view(K, 1, 1)
    return (torch.arange(Ho).view(1, Ho, 1) * sh - ph + ki * dh).float(), (torch.arange(Wo).view(1, 1, Wo) * sw - pw + kj * dw).float()


def _positions(c, off):
    """(p_h, p_w), each [N, dg, K, Ho, Wo], as the kernel forms them: one addition in the offset's dtype"""
    N, C, H, W, O, (kh, kw), s, p, d, G, dg = c
    Ho, Wo = _out(c)
    o = off.view(N, dg, kh * kw, 2, Ho, Wo)
    bh, bw = _bases(c)
    return bh.to(off.dtype) + o[:, :, :, 0], bw.to(off.dtype) + o[:, :, :, 1]


def _edge_targets(L):
    f = np.float32
    return [f(-1), np.nextafter(f(-1), f(0)), f(L - 1), np.nextafter(f(L - 1), f(L)), np.nextafter(f(L), f(0))]


def _exact_axis(base, L, g):
    """offsets that put each sample exactly on one of the edge positions of an axis of length L (a random one of those its base can
    reach with one fp32 addition), else on a whole pixel in [-2, L + 1]"""
    t = torch.tensor(_edge_targets(L), dtype=torch.float32).view(-1, *([1] * base.dim()))
    cand = (t.double() - base.double()).float()
    ok = (base + cand) == t
    pick = (torch.rand(ok.shape, generator=g) * ok).argmax(0, keepdim=True)
    whole = torch.randint(-2, L + 2, base.shape, generator=g).float() - base
    return torch.where(ok.any(0), cand.gather(0, pick)[0], whole)


def synth(c, mode, seed):
    """x, offset, weight, grad_y (fp32, CPU) of one case"""
    N, C, H, W, O, (kh, kw), s, p, d, G, dg = c
    Ho, Wo = _out(c)
    K = kh * kw
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C, H, W, generator=g)
    shape = (N, dg, K, Ho, Wo)
    bh, bw = (b.expand(shape).contiguous() for b in _bases(c))
    if mode in ("normal", "nonfinite"):
        oh, ow = torch.randn(shape, generator=g) * 1.5, torch.randn(shape, generator=g) * 1.5
        if mode == "nonfinite":
            for o in (oh, ow):
                u = torch.rand(shape, generator=g)
                o[u < 0.1] = float("nan")
                o[(u >= 0.1) & (u < 0.15)] = float("inf")
                o[(u >= 0.15) & (u < 0.2)] = float("-inf")
    elif mode == "large":
        oh, ow = ((torch.rand(shape, generator=g) * 2 - 1) * 2 * max(H, W) for _ in range(2))
    elif mode == "integer":
        oh, ow = (torch.randint(-(max(H, W) + 2), max(H, W) + 3, shape, generator=g).float() for _ in range(2))
    elif mode == "zero":
        oh, ow = torch.zeros(shape), torch.zeros(shape)
    elif mode == "exact":
        oh, ow = _exact_axis(bh, H, g), _exact_axis(bw, W, g)
    elif mode == "collapsed":  # every sample on input pixel (H // 2, W // 3)
        oh, ow = (H // 2) - bh, (W // 3) - bw
    else:
        raise ValueError(mode)
    off = torch.stack([oh, ow], 3).reshape(N, 2 * dg * K, Ho, Wo).contiguous()
    w = torch.randn(O, C // G, kh, kw, generator=g) / (C // G * K) ** 0.5
    gy = torch.randn(N, O, Ho, Wo, generator=g)
    return x, off, w, gy


def _args(c):
    N, C, H, W, O, k, s, p, d, G, dg = c
    return s, p, d, G, dg


def _oracle(c, x, off, w, gy):
    """float64 (y, grad_x, grad_offset, grad_weight) and their per-element bounds"""
    a = _args(c)
    ref = (D.deform_conv2d(x, off, w, *a),) + D.deform_conv2d_grads(x, off, w, gy, *a)
    bound = (D.deform_conv2d(x.abs(), off, w.abs(), *a),) + D.deform_conv2d_grads(x, off, w, gy, *a, absolute=True)
    return ref, bound


def _record(key, value):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    if OBSERVED:
        print("\n[dcn edges observed err / bound] " + json.dumps({k: f"{v:.3e}" for k, v in sorted(OBSERVED.items())}, indent=1))


def _check(name, got, ref, bound, rtol=None):
    """|got - ref| <= rtol * bound per element (exactly equal where the bound is 0); got must be finite"""
    rtol = RTOL[name] if rtol is None else rtol
    got = got.detach().cpu().double()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} non-finite elements"
    assert torch.isfinite(ref).all() and torch.isfinite(bound).all()
    err = (got - ref).abs()
    bad = err > rtol * bound + 1e-30
    ratio = (err / bound.clamp_min(1e-30)).max().item() if err.numel() else 0.0
    _record(name, ratio)
    assert not bad.any(), f"{name}: {int(bad.sum())} of {bad.numel()} elements off, worst err / bound {ratio:.3e} (rtol {rtol:.0e})"


def _run_ops(c, x, off, w, gy):
    """ops.deform_conv2d forward and backward on the GPU against the oracle"""
    from sst_b200 import ops
    xg, og, wg = (t.to(dev).requires_grad_(True) for t in (x, off, w))
    y = ops.deform_conv2d(xg, og, wg, *_args(c))
    y.backward(gy.to(dev))
    ref, bound = _oracle(c, x, off, w, gy)
    for name, got, r, b in zip(("y", "grad_x", "grad_offset", "grad_weight"), (y, xg.grad, og.grad, wg.grad), ref, bound):
        _check(name, got, r, b)
    return ref, bound


# ----------------------------------------------------------------------------------------------------------------------------------
# a. the oracle against torchvision (CPU, float64)
# ----------------------------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


CPU_GRID = {**AXES, **{k: LANES[k] for k in ("cd1", "cd33", "cd48")}, "px257": SORT["px257"]}


@pytest.mark.parametrize("mode", ("normal", "large", "integer", "exact"))
@pytest.mark.parametrize("key", list(CPU_GRID))
def test_oracle_matches_torchvision_asymmetric(key, mode):
    tv = pytest.importorskip("torchvision")
    c = CPU_GRID[key]
    x, off, w, gy = (t.double() for t in synth(c, mode, _seed("cpu", key, mode)))
    s, p, d, G, dg = _args(c)
    xr, orr, wr = (t.clone().requires_grad_(True) for t in (x, off, w))
    yt = tv.ops.deform_conv2d(xr, orr, wr, None, s, p, d)
    yt.backward(gy)
    y = D.deform_conv2d(x, off, w, s, p, d, G, dg)
    gx, goff, gw = D.deform_conv2d_grads(x, off, w, gy, s, p, d, G, dg)
    # a sample exactly at p = -1 on either axis lies outside mmcv's open domain, so its offset gradient is 0; torchvision's is not
    ph, pw = _positions(c, off)
    m = (ph == -1) | (pw == -1)
    at_m1 = torch.stack([m, m], 3).view(off.shape)
    if mode == "exact":
        assert at_m1.any()
    assert (goff[at_m1] == 0).all()
    tv_goff = torch.where(at_m1, 0.0, orr.grad)
    for name, a, b in (("y", y, yt), ("grad_x", gx, xr.grad), ("grad_offset", goff, tv_goff), ("grad_weight", gw, wr.grad)):
        assert _rel(a, b.detach()) <= 1e-12, name


@pytest.mark.parametrize("key", ["base", "mixed"] + [k for k in AXES if not k.startswith("hw")])
def test_exact_offsets_reach_every_edge_position(key):
    """the 'exact' offsets put samples on each of the five edge positions of both axes, as one fp32 addition"""
    c = {**AXES, **OFFSET_GEOMS}[key]
    H, W = c[2], c[3]
    _, off, _, _ = synth(c, "exact", _seed("exact", key))
    ph, pw = _positions(c, off)
    for p, L in ((ph, H), (pw, W)):
        for t in _edge_targets(L):
            assert (p == torch.tensor(t)).any(), (key, L, float(t))


# ----------------------------------------------------------------------------------------------------------------------------------
# b. the GPU against the oracle
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key,mode", [(k, m) for k in AXES for m in ("normal", "integer", "exact")
                                      if not (m == "exact" and k.startswith("hw"))])  # on an axis of length 1 they are subnormal
def test_axes(key, mode):
    _run_ops(AXES[key], *synth(AXES[key], mode, _seed("axes", key, mode)))


@pytest.mark.gpu
@pytest.mark.parametrize("og", list(OG))
def test_forward_output_tiles(og):
    _run_ops(OG[og], *synth(OG[og], "normal", _seed("og", og)))


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(TILES))
def test_forward_pixel_tiles(key):
    _run_ops(TILES[key], *synth(TILES[key], "normal", _seed("tiles", key)))


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(DEPTH))
def test_reduction_depth(key):
    _run_ops(DEPTH[key], *synth(DEPTH[key], "normal", _seed("depth", key)))


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(SPLITS))
def test_grad_weight_splits(key):
    _run_ops(SPLITS[key], *synth(SPLITS[key], "normal", _seed("splits", key)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ("normal", "integer"))
@pytest.mark.parametrize("key", list(LANES))
def test_lane_loops(key, mode):
    _run_ops(LANES[key], *synth(LANES[key], mode, _seed("lanes", key, mode)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ("normal", "integer"))
@pytest.mark.parametrize("key", list(SORT))
def test_sort_key_width(key, mode):
    _run_ops(SORT[key], *synth(SORT[key], mode, _seed("sort", key, mode)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", OFFSET_MODES)
@pytest.mark.parametrize("key", list(OFFSET_GEOMS))
def test_offsets(key, mode):
    c = OFFSET_GEOMS[key]
    x, off, w, gy = synth(c, mode, _seed("offsets", key, mode))
    ref, bound = _run_ops(c, x, off, w, gy)
    if mode == "nonfinite":
        ph, pw = _positions(c, off)
        assert (~torch.isfinite(ph)).any() and (~torch.isfinite(pw)).any()
    if mode == "collapsed":  # one input pixel per (n, d) gathers every sample: all other input pixels get exactly 0
        N, C, H, W = x.shape
        hit = torch.zeros(H, W, dtype=torch.bool)
        hit[H // 2, W // 3] = True
        assert (bound[1][:, :, hit] > 0).all() and (bound[1][:, :, ~hit] == 0).all()


# ----------------------------------------------------------------------------------------------------------------------------------
# c. bit-level properties through the C ABI, caller-owned buffers
# ----------------------------------------------------------------------------------------------------------------------------------
BITS = {16: _case(2, 8, 9, 11, 16, k=(2, 3), p=(1, 2), G=2, dg=2), 32: _case(2, 8, 9, 11, 64, k=(3, 2), s=(2, 1), G=2, dg=4),
        64: _case(3, 8, 10, 7, 130, k=(3, 1), d=(2, 1), G=2, dg=2)}


def _lib():
    from sst_b200 import _lib as L
    from sst_b200 import ops  # noqa: F401  (declares the dcn signatures)
    return L


def _geom(c):
    N, C, H, W, O, (kh, kw), (sh, sw), (ph, pw), (dh, dw), G, dg = c
    return _lib().arr(ctypes.c_int32, [N, C, H, W, O, kh, kw, sh, sw, ph, pw, dh, dw, G, dg])


def _guarded(n):
    return torch.full((n + GUARD,), POISON, dtype=torch.int32, device=dev).view(torch.float32)


def _abi_forward(c, x, off, w):
    L = _lib()
    ctx = L.ctx(dev)
    N, O = c[0], c[4]
    Ho, Wo = _out(c)
    y = _guarded(N * O * Ho * Wo)
    L.check(ctx, L.lib().sstb200_dcn_forward(ctx, _geom(c), x.data_ptr(), off.data_ptr(), w.data_ptr(), y.data_ptr()))
    return y


def _workspace_bytes(c):
    L = _lib()
    ctx = L.ctx(dev)
    n = ctypes.c_int64()
    rc = L.lib().sstb200_dcn_backward_workspace_bytes(ctx, _geom(c), ctypes.byref(n))
    return rc, n.value


def _abi_backward(c, x, off, w, gy, want=(True, True, True), fill=0):
    """guarded (grad_x, grad_offset, grad_weight), None where not wanted; the workspace starts as bytes `fill`"""
    L = _lib()
    ctx = L.ctx(dev)
    rc, nbytes = _workspace_bytes(c)
    L.check(ctx, rc)
    ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=dev)
    outs = [_guarded(t.numel()) if on else None for t, on in zip((x, off, w), want)]
    L.check(ctx, L.lib().sstb200_dcn_backward(ctx, _geom(c), x.data_ptr(), off.data_ptr(), w.data_ptr(), gy.data_ptr(), ws.data_ptr(),
                                              nbytes, *(L.ptr(t) for t in outs)))
    return outs


def _bits(t):
    return t.view(torch.int32).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("bn", list(BITS))
def test_abi_sentinels_dirty_workspace_determinism(bn):
    c = BITS[bn]
    x, off, w, gy = synth(c, "large", _seed("bits", bn))
    xd, od, wd, gyd = (t.to(dev) for t in (x, off, w, gy))
    ref, bound = _oracle(c, x, off, w, gy)
    y1, y2 = _abi_forward(c, xd, od, wd), _abi_forward(c, xd, od, wd)
    clean = _abi_backward(c, xd, od, wd, gyd, fill=0)
    dirty = _abi_backward(c, xd, od, wd, gyd, fill=0xFF)
    ph, pw = _positions(c, off)
    H, W = c[2], c[3]
    valid = (ph > -1) & (pw > -1) & (ph < H) & (pw < W)
    invalid = torch.stack([~valid, ~valid], 3).reshape(off.shape)
    untouched = bound[1] == 0  # no sample with a non-zero corner weight reaches the input pixel
    assert invalid.any() and untouched.any()
    for name, a, b, r, bd in zip(("y", "grad_x", "grad_offset", "grad_weight"), (y1,) + tuple(clean), (y2,) + tuple(dirty), ref, bound):
        n = r.numel()
        assert torch.equal(_bits(a), _bits(b)), f"{name}: two calls (clean / 0xFF workspace) differ"
        assert (_bits(a[n:]) == POISON).all(), f"{name}: written past the end"
        got = a[:n].view(r.shape)
        _check(name, got, r, bd)
        if name == "grad_x":
            assert (_bits(got.cpu()[untouched]) == 0).all(), "grad_x: an untouched input pixel is not +0"
        if name == "grad_offset":
            assert (_bits(got.cpu()[invalid]) == 0).all(), "grad_offset: an invalid sample's gradient is not +0"


@pytest.mark.gpu
@pytest.mark.parametrize("bn", list(BITS))
def test_abi_gradient_subsets(bn):
    c = BITS[bn]
    xd, od, wd, gyd = (t.to(dev) for t in synth(c, "normal", _seed("subsets", bn)))
    full = _abi_backward(c, xd, od, wd, gyd)
    for m in range(1, 7):
        want = tuple(bool(m >> i & 1) for i in range(3))
        part = _abi_backward(c, xd, od, wd, gyd, want=want, fill=0xFF)
        for i, (a, b) in enumerate(zip(full, part)):
            if want[i]:
                assert torch.equal(_bits(a), _bits(b)), (want, i)
            else:
                assert b is None


@pytest.mark.gpu
def test_non_contiguous_inputs():
    """a channels_last x, an offset that is a channel slice of a larger tensor and the stride-0 grad_y of y.sum() give the bits of
    contiguous inputs and an explicit grad_y of ones"""
    from sst_b200 import ops
    c = BITS[32]
    x, off, w, _ = synth(c, "normal", _seed("noncontig"))
    a = _args(c)
    xa, oa, wa = (t.to(dev).requires_grad_(True) for t in (x, off, w))
    ya = ops.deform_conv2d(xa, oa, wa, *a)
    ya.backward(torch.ones_like(ya))
    xb = x.to(dev).to(memory_format=torch.channels_last).requires_grad_(True)
    assert not xb.is_contiguous()
    big = torch.randn(off.shape[0], off.shape[1] + 3, *off.shape[2:])
    big[:, 1:1 + off.shape[1]] = off
    big = big.to(dev).requires_grad_(True)
    ob = big[:, 1:1 + off.shape[1]]
    assert not ob.is_contiguous()
    wb = w.to(dev).requires_grad_(True)
    yb = ops.deform_conv2d(xb, ob, wb, *a)
    yb.sum().backward()
    assert torch.equal(_bits(ya.detach().contiguous()), _bits(yb.detach().contiguous()))
    assert torch.equal(_bits(xa.grad.contiguous()), _bits(xb.grad.contiguous()))
    assert torch.equal(_bits(oa.grad), _bits(big.grad[:, 1:1 + off.shape[1]].contiguous()))
    assert (big.grad[:, 0] == 0).all() and (big.grad[:, 1 + off.shape[1]:] == 0).all()
    assert torch.equal(_bits(wa.grad), _bits(wb.grad))


# ----------------------------------------------------------------------------------------------------------------------------------
# d. limits, through the workspace size query only (nothing is allocated or launched)
# ----------------------------------------------------------------------------------------------------------------------------------
# M = 4 N dg K Ho Wo: 2^29 - 1 = 233 * 1103 * 2089 samples give M = 2^31 - 4, the largest the backward's int sort count takes
LIMITS = {
    "m_2p31_minus_4": (_case(1, 1, 233 * 1103, 2089, 1, k=(1, 1), p=(0, 0)), 0),
    "m_2p31": (_case(1, 1, 1 << 15, 1 << 14, 1, k=(1, 1), p=(0, 0)), -3),
    "m_3x2p30": (_case(1, 1, 3 << 14, 1 << 14, 1, k=(1, 1), p=(0, 0)), -3),
    "pixels_2p32_minus_2": (_case(1, 1, 2, (1 << 31) - 1, 1, k=(1, 1), s=(1, (1 << 31) - 1), p=(0, 0)), 0),
    "pixels_2p32": (_case(1, 1, 1 << 16, 1 << 16, 1, k=(1, 1), s=(256, 256), p=(0, 0)), -3),
    "n_65535": (_case(65535, 1, 1, 1, 1, k=(1, 1), p=(0, 0)), 0),
    "n_65536": (_case(65536, 1, 1, 1, 1, k=(1, 1), p=(0, 0)), -3),
    "rchunks_65535": (_case(1, 16 * 65535, 1, 1, 1, k=(1, 1), p=(0, 0)), 0),
    "rchunks_65536": (_case(1, 16 * 65535 + 1, 1, 1, 1, k=(1, 1), p=(0, 0)), -3),
    "rchunks_g_65536": (_case(1, 2 * 16 * 32768, 1, 1, 2, k=(1, 1), p=(0, 0), G=2), -3),
    "otiles_65535": (_case(1, 1, 1, 1, 16 * 65535, k=(1, 1), p=(0, 0)), 0),
    "otiles_65536": (_case(1, 1, 1, 1, 16 * 65535 + 1, k=(1, 1), p=(0, 0)), -3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(LIMITS))
def test_backward_limits(key):
    c, want = LIMITS[key]
    rc, nbytes = _workspace_bytes(c)
    assert rc == want, (key, rc)
    if want == 0:
        N, C, H, W, O, (kh, kw), s, p, d, G, dg = c
        Ho, Wo = _out(c)
        M = 4 * N * dg * kh * kw * Ho * Wo
        assert M <= (1 << 31) - 4
        assert nbytes >= 16 * M + 4 * (N * H * W * C + N * O * Ho * Wo)


@pytest.mark.gpu
def test_backward_workspace_one_byte_short():
    c = BITS[16]
    L = _lib()
    ctx = L.ctx(dev)
    xd, od, wd, gyd = (t.to(dev) for t in synth(c, "normal", 1))
    rc, nbytes = _workspace_bytes(c)
    assert rc == 0
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    outs = [torch.empty_like(t) for t in (xd, od, wd)]
    rc = L.lib().sstb200_dcn_backward(ctx, _geom(c), xd.data_ptr(), od.data_ptr(), wd.data_ptr(), gyd.data_ptr(), ws.data_ptr(), nbytes - 1,
                                      *(t.data_ptr() for t in outs))
    assert rc == -4


# ----------------------------------------------------------------------------------------------------------------------------------
# e. modules
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_deform_conv2d_input_smaller_than_kernel():
    """mmcv pads an input smaller than the kernel on the bottom and right, and crops the output back: the oracle on the same padded
    input, cropped"""
    from sst_b200.dcn_modules import DeformConv2d
    m = DeformConv2d(4, 6, 3, padding=1, groups=2, deform_groups=2).to(dev)
    g = torch.Generator().manual_seed(_seed("small"))
    x = torch.randn(2, 4, 2, 1, generator=g)
    off = torch.randn(2, 2 * 2 * 9, 2, 1, generator=g) * 1.5
    gy = torch.randn(2, 6, 2, 1, generator=g)
    w = m.weight.detach().cpu()
    xg, og = x.to(dev).requires_grad_(True), off.to(dev).requires_grad_(True)
    y = m(xg, og)
    y.backward(gy.to(dev))
    pad = (0, 2, 0, 1)
    c = _case(2, 4, 3, 3, 6, G=2, dg=2)
    ref, bound = _oracle(c, F.pad(x, pad), F.pad(off, pad), w, F.pad(gy, pad))
    crop = lambda t: t[:, :, :2, :1]  # noqa: E731
    for name, got, r, b in zip(("y", "grad_x", "grad_offset"), (y, xg.grad, og.grad), ref, bound):
        _check(name, got, crop(r), crop(b))
    _check("grad_weight", m.weight.grad, ref[3], bound[3])


@pytest.mark.gpu
def test_deform_conv2d_pack_asymmetric():
    """DeformConv2dPack with kernel (3, 1), stride (2, 1) and non-zero conv_offset weights, forward and backward, against the oracle's
    float64 offset conv + deform_conv2d.  Offsets of 0.3 .. 0.7 pixels plus a small input-dependent part keep every sample clear of
    integer positions, where grad_offset jumps.  The gradients that pass through conv_offset are bounded by the same |terms| sums pushed
    through the offset conv's backward with |conv_offset.weight|."""
    from sst_b200.dcn_modules import DeformConv2dPack
    torch.manual_seed(0)
    m = DeformConv2dPack(8, 12, (3, 1), stride=(2, 1), padding=(1, 0), groups=2, deform_groups=2)
    g = torch.Generator().manual_seed(_seed("pack"))
    with torch.no_grad():
        m.conv_offset.weight.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * 0.005)
        m.conv_offset.bias.copy_(torch.rand(m.conv_offset.bias.shape, generator=g) * 0.4 + 0.3)
    m = m.to(dev)
    x = torch.randn(2, 8, 13, 7, generator=g)
    gy = torch.randn(2, 12, 7, 7, generator=g)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        xg = x.to(dev).requires_grad_(True)
        y = m(xg)
        y.backward(gy.to(dev))
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64 = x.double().requires_grad_(True)
    kw = dict(stride=(2, 1), padding=(1, 0), dilation=1, groups=2, deform_groups=2)
    y64 = D.dcn_pack_forward(x64, sd, "", **kw)
    y64.backward(gy.double())
    c = _case(2, 8, 13, 7, 12, k=(3, 1), s=(2, 1), p=(1, 0), G=2, dg=2)
    off64 = F.conv2d(x.double(), sd["conv_offset.weight"].detach(), sd["conv_offset.bias"].detach(), (2, 1), (1, 0))
    frac = off64 - off64.floor()
    assert ((frac > 0.1) & (frac < 0.9)).all()
    w64 = sd["weight"].detach()
    _, bound = _oracle(c, x.double(), off64, w64, gy.double())
    by, bx, boff, bw = bound
    _check("y", y, y64.detach(), by)
    _check("grad_weight", m.weight.grad, sd["weight"].grad, bw)
    wo_abs = sd["conv_offset.weight"].detach().abs()
    bx_total = bx + torch.nn.grad.conv2d_input(x.shape, wo_abs, boff, (2, 1), (1, 0))
    _check("grad_x", xg.grad, x64.grad, bx_total)
    _check("grad_weight", m.conv_offset.weight.grad, sd["conv_offset.weight"].grad,
           torch.nn.grad.conv2d_weight(x.double().abs(), wo_abs.shape, boff, (2, 1), (1, 0)))
    _check("grad_weight", m.conv_offset.bias.grad, sd["conv_offset.bias"].grad, boff.sum((0, 2, 3)))
