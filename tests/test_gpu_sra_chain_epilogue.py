"""Epilogues of the fused post-attention chain (csrc/sra_chain2.cu): the GELU of its hidden layer and its two LayerNorms.

- gelu_ex2 (csrc/common.cuh), the GELU of the chain's GEMM2 epilogue, restated as its exact fp32 operation sequence in numpy
  (fused multiply-adds rounded once, ex2 rounded to fp32) and held to the exact erf-GELU over [-12, 12]: at most 1e-6 absolute
  and at most one fp16 ulp of the result, which the kernel rounds to fp16.  The coefficients are read from the header.
- LayerNorm shift-safety: the pre-norm rows of both LayerNorms carry a common offset of +1024 (out_proj.bias feeds LN1,
  linear2.bias feeds LN2), where a one-pass E[t^2] - mean^2 variance cancels to a few percent.  The offset enters after the
  16-bit attention operands, so only the chain sees it.
- GELU range: linear1 scaled so that the hidden pre-activations span about +-10 (both GELU tails).
Both run through the fused bf16 stack at voxel counts on the chain's tile edges, against the float64 oracle with the bf16
bounds of test_gpu_sra_chain.py: 1e-2 relative, max-norm and element-wise.
"""
import os
import re

import numpy as np
import pytest
import torch

from oracle import sst_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN = (12, 12, 1)
GRID = (468, 468, 1)
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
ODD = "odd_tiles"   # (2 x SMs + 2) tiles, the last one partial: the first two CTAs take three tiles, the others two
SHIFT = 1024.0


def _gelu_ex2_coefficients():
    src = open(os.path.join(ROOT, "sst_b200", "csrc", "common.cuh")).read()
    body = src[src.index("float gelu_ex2(float x)"):]
    body = body[:body.index("\n}\n")]
    clamp = float(re.search(r"fminf\(fabsf\(x\), ([0-9.]+)f\)", body).group(1))
    coef = [float(v) for v in re.findall(r"([-+]?\d\.\d+e[-+]\d+)f", body)]   # Horner order: highest degree first
    return np.float32(clamp), [np.float32(c) for c in coef]


def _fma32(a, b, c):
    """fp32 fused multiply-add: the float64 product of two fp32 values is exact, the sum rounds once to fp32 (the rare double
    rounding through float64 differs from the hardware's single rounding by at most one fp32 ulp)"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def gelu_ex2_mirror(x):
    clamp, coef = _gelu_ex2_coefficients()
    x = x.astype(np.float32)
    a = np.minimum(np.abs(x), clamp)
    p = _fma32(np.full_like(a, coef[0]), a, np.full_like(a, coef[1]))
    for c in coef[2:]:
        p = _fma32(p, a, np.full_like(a, c))
    q = np.exp2(p.astype(np.float64)).astype(np.float32)   # ex2.approx: within 2 fp32 ulp of this
    return _fma32(-np.abs(x), q, np.maximum(x, np.float32(0)))


def _fp16_ulp(v):
    v = np.abs(v)
    e = np.floor(np.log2(np.maximum(v, 2.0 ** -24)))
    return np.where(v < 2.0 ** -14, 2.0 ** -24, 2.0 ** (e - 10))


def test_gelu_ex2_mirror_bounds():
    from scipy.special import ndtr
    clamp, coef = _gelu_ex2_coefficients()
    assert len(coef) == 7 and clamp == 6.0
    x = np.concatenate([np.linspace(-12.0, 12.0, 2_400_001, dtype=np.float32),
                        np.float32([0.0, 1e-30, -1e-30, 1e-8, -1e-8, 1e-4, -1e-4, 6.0, -6.0, 5.9999995, -5.9999995])])
    got = gelu_ex2_mirror(x).astype(np.float64)
    xd = x.astype(np.float64)
    ref = xd * ndtr(xd)
    err = np.abs(got - ref)
    assert err.max() <= 1e-6, (err.max(), x[err.argmax()])
    ulp = err / _fp16_ulp(ref)
    assert ulp.max() <= 1.0, (ulp.max(), x[ulp.argmax()])
    assert got[x == 0].max() == 0.0 and np.all(np.isfinite(got))


def _voxels(n, seed):
    g = torch.Generator().manual_seed(seed)
    cell = torch.randperm(GRID[0] * GRID[1], generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), cell // GRID[0], cell % GRID[0]], 1).int()
    return torch.randn(n, 128, generator=g), coors


def _model(shift, lin1_scale):
    from sst_b200.sst_modules import SSTv2
    torch.manual_seed(0)
    m = SSTv2(d_model=[128], nhead=[8], num_blocks=1, dim_feedforward=[256], output_shape=[468, 468], num_attached_conv=0,
              to_bev=False, layer_cfg={}).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            if n_.endswith("out_proj.bias") or n_.endswith("linear2.bias"):
                p.add_(shift)
            if n_.endswith("linear1.weight"):
                p.mul_(lin1_scale)
    return m


def _rows(n):
    if n != ODD:
        return n
    return (2 * torch.cuda.get_device_properties(0).multi_processor_count + 2) * 128 - 37


def _run(cuda, n, shift, lin1_scale):
    from sst_b200.sst_modules import SSTInputLayerV2
    n = _rows(n)
    feats, coors = _voxels(n, 300 + n)
    m = _model(shift, lin1_scale)
    il = SSTInputLayerV2((DROP_TEST, DROP_TEST), WIN, GRID, shuffle_voxels=False, mute=True).eval()
    info_o = O.input_layer_v2(feats.double(), coors, DROP_TEST, WIN, GRID)
    assert info_o["voxel_feats"].shape[0] == n
    ref = O.sstv2_forward(info_o, {k: v.double().clone() for k, v in m.state_dict().items()}, [8], 1, "gelu", {})
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        got = m(il(feats.to(cuda), coors.to(cuda), 1))[0]["voxel_feats"]
    got = got.cpu().double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, err
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2 * ref.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("n", [50, 65, 128, 129, ODD])
def test_fused_stack_layernorm_shift(cuda, n):
    """pre-norm rows of LN1 and LN2 offset by +1024: the two-pass statistics keep the variance"""
    _run(cuda, n, SHIFT, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [65, 129, ODD])
def test_fused_stack_gelu_range(cuda, n):
    """linear1 x 3: hidden pre-activations span about +-10, both GELU tails"""
    _run(cuda, n, 0.0, 3.0)
