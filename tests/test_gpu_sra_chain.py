"""GPU parity of the fused post-attention chain (csrc/sra_chain2.cu) at voxel counts on the edges of its schedule.

The chain walks 128-row tiles, one per CTA round, and splits each tile into two 64-row halves handled by two warpgroups in
ping-pong.  The counts below hit a half with no valid rows (fewer than 64 rows, 64), one valid row in the second half (65), a
full or nearly full single tile (127, 128), one row into a second tile (129), and 2 x SMs + 2 tiles (the grid has one CTA per
SM), which gives the first two CTAs three tiles and the others two.  Each runs through the fused bf16 stack (2 launches per
layer) and through the single-layer bf16 path, also with a device-resident row count below the buffers' capacity and in place
(y == x), against the CPU oracle with the bf16 bounds of test_gpu_sst.py: 1e-2 relative, max-norm and element-wise.
"""
import ctypes as C

import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

WIN = (12, 12, 1)
GRID = (468, 468, 1)
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
ODD = "odd_tiles"   # resolved on the device: (2 x SMs + 2) tiles, the last one partial
COUNTS = [50, 64, 65, 127, 128, 129, ODD]
LN = {}
BN_COS = dict(use_bn=True, cosine=True, tau_min=0.01)


def _voxels(n, seed):
    """n distinct voxels of one sweep: a 12 x 12 window holds at most 144, so no voxel is dropped and the stack sees n rows."""
    g = torch.Generator().manual_seed(seed)
    cell = torch.randperm(GRID[0] * GRID[1], generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), cell // GRID[0], cell % GRID[0]], 1).int()
    return torch.randn(n, 128, generator=g), coors


def _model(layer_cfg, blocks=1):
    from sst_b200.sst_modules import SSTv2
    torch.manual_seed(0)
    m = SSTv2(d_model=[128] * blocks, nhead=[8] * blocks, num_blocks=blocks, dim_feedforward=[256] * blocks, output_shape=[468, 468],
              num_attached_conv=0, to_bev=False, layer_cfg=layer_cfg).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():   # non-trivial norms / biases so that every epilogue term is exercised
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            if n_.endswith("tau"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.5 + 0.05)
        for n_, b in m.named_buffers():
            if "running_mean" in n_:
                b.copy_(torch.randn(b.shape, generator=g) * 0.3)
            if "running_var" in n_:
                b.copy_(torch.rand(b.shape, generator=g) + 0.5)
    return m


def _rows(n):
    if n != ODD:
        return n
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (2 * sms + 2) * 128 - 37


def _case(cuda, n, layer_cfg):
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels(n, 100 + n)
    m = _model(layer_cfg)
    il = SSTInputLayerV2((DROP_TEST, DROP_TEST), WIN, GRID, shuffle_voxels=False, mute=True).eval()
    info_o = O.input_layer_v2(feats, coors, DROP_TEST, WIN, GRID)
    assert info_o["voxel_feats"].shape[0] == n
    ref = O.sstv2_forward(info_o, {k: v.clone() for k, v in m.state_dict().items()}, [8], 1, "gelu", layer_cfg)
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        info_g = il(feats.to(cuda), coors.to(cuda), 1)
    return m, info_g, ref


def _check(got, ref):
    got = got.cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, err
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2 * ref.abs().max().item())


def _padded(x, cap, fill):
    out = torch.full((cap, x.shape[1]), fill, dtype=torch.float32, device=x.device)
    out[:x.shape[0]] = x
    return out


@pytest.mark.parametrize("layer_cfg", [LN, BN_COS], ids=["layernorm", "batchnorm_cosine"])
@pytest.mark.parametrize("n", COUNTS)
def test_fused_stack_edges(cuda, n, layer_cfg):
    """The fused stack (chain with the next layer's q|k|v, then the chain without it) at n == capacity; from the second layer on
    the chain runs in place."""
    n = _rows(n)
    m, info_g, ref = _case(cuda, n, layer_cfg)
    with torch.no_grad():
        got = m(info_g)[0]["voxel_feats"]
    _check(got, ref)


@pytest.mark.parametrize("layer_cfg", [LN, BN_COS], ids=["layernorm", "batchnorm_cosine"])
@pytest.mark.parametrize("n", [50, 65, 129, ODD])
def test_fused_stack_device_count_below_capacity(cuda, n, layer_cfg):
    """Row count read from device memory, buffers 200 rows larger: rows past the count are never written, and the result is
    bit-identical to the call with n == capacity."""
    from sst_b200 import _lib as L
    from sst_b200.sst_modules import PRECISIONS, _SraLayer, make_sra_plan
    n = _rows(n)
    m, info_g, ref = _case(cuda, n, layer_cfg)
    with torch.no_grad():
        exact = m(info_g)[0]["voxel_feats"]
    layers = [l for blk in m.block_list for l in blk.encoder_list]
    arr = (_SraLayer * len(layers))(*[l._struct(PRECISIONS["bf16"]) for l in layers])
    p0, p1 = make_sra_plan(info_g["sra_plan_shift0"]), make_sra_plan(info_g["sra_plan_shift1"])
    cap = n + 200
    x = _padded(info_g["voxel_feats"].float(), cap, 3.0)
    y, tmp = torch.full_like(x, 7.0), torch.empty_like(x)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    c = L.ctx(cuda)
    L.check(c, L.lib().sstb200_sra_stack_forward(c, arr, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(),
                                                 tmp.data_ptr(), cap, n_dev.data_ptr(), PRECISIONS["bf16"]))
    torch.cuda.synchronize()
    assert torch.equal(y[:n], exact)
    assert (y[n:] == 7.0).all()
    _check(y[:n], ref)


@pytest.mark.parametrize("n", COUNTS)
def test_single_layer_edges_in_place(cuda, n):
    """Single-layer bf16 path (QKV GEMM, attention, chain without the q|k|v tail), layer by layer through one block: out of
    place at n == capacity, and in place (y == x) with the row count on the device and 200 spare rows, bit-identical."""
    from sst_b200 import _lib as L
    from sst_b200.sst_modules import PRECISIONS, make_sra_plan
    n = _rows(n)
    m, info_g, ref = _case(cuda, n, LN)
    layers = [l for blk in m.block_list for l in blk.encoder_list]
    plans = [info_g["sra_plan_shift0"], info_g["sra_plan_shift1"]]
    x0 = info_g["voxel_feats"].float().contiguous()
    with torch.no_grad():
        out = x0
        for i, l in enumerate(layers):
            out = l(out, plans[i % 2], "bf16")
    _check(out, ref)
    cap = n + 200
    buf = _padded(x0, cap, 3.0)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    c = L.ctx(cuda)
    for i, l in enumerate(layers):
        ls, ps = l._struct(PRECISIONS["bf16"]), make_sra_plan(plans[i % 2])
        L.check(c, L.lib().sstb200_sra_layer_forward(c, C.byref(ls), C.byref(ps), buf.data_ptr(), buf.data_ptr(), cap, n_dev.data_ptr(),
                                                     PRECISIONS["bf16"]))
    torch.cuda.synchronize()
    assert torch.equal(buf[:n], out)
    assert (buf[n:] == 3.0).all()
