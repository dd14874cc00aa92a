"""GPU: the SST training stack (csrc/sra_train.cu) against float64 autograd through the oracle at the row counts where its
schedule changes shape, forward and backward.

Everything but attention is row-tiled, and every tiling depends on the SM count the library launches with:
  * the LayerNorm backward (ln_bwd_kernel) walks 8 rows per block and pass over 2 x SMs blocks;
  * the weight-gradient GEMM (dw_gemm_kernel + dw_reduce_kernel) splits the rows into 64-row-aligned splits, ceil(2 x SMs / blocks)
    of them, so past 64 x SMs rows (2 output blocks) or 128 x SMs rows (1 block) some splits are empty;
  * the persistent wgmma GEMMs (launch_wgmma_gemm) run SMs x per_sm CTAs over ceil(n / 128) x ny items and wrap once there are more.
`stack_edges` restates those formulas and yields the row counts on either side of each boundary.  A dropped or doubled row
changes a dense-gradient sum by about 1 / n, far below the bf16 bounds, so every case also runs with an upstream gradient that is
zero except on a few probe rows placed on those boundaries: then the weight, bias and LayerNorm gradients are sums over the
probe rows only, and a lost row is a large share of them.

Bounds are the existing bf16 ones (test_gpu_train.py, test_gpu_train_cosine.py), element-wise: 1e-2 of max |ref| for y, 2e-2 for
dx and the parameter gradients, 3e-2 for d tau.  y and dx are also held to the same bounds row by row, each row's max error
against that row's own max |ref|.  The kernels' worst errors measured on an H100 are listed beside the bounds.

The contract tests call the C ABI directly: two backward calls give the same bits, the call adds to what `grads` holds (G0 + g
bit for bit), and n == 0 touches nothing.  A last group puts a common offset of up to 1024 into the pre-LayerNorm sums through
the biases added before each LayerNorm, which only a two-pass variance survives.
"""
import ctypes as C

import pytest
import torch

from oracle import sst_oracle as O

WIN = (12, 12, 1)
GRID = (468, 468, 1)
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
TOL_Y, TOL_G, TOL_TAU = 1e-2, 2e-2, 3e-2
# per row, against the row's own max |ref|.  Worst measured on an H100 80GB HBM3 (700 W) over every case here: y 8.0e-3 per row
# (3.8e-3 of the global max), dx 1.7e-2 per row (7.2e-3 global), parameter gradients and d tau with the dense upstream 1.2e-2.
TOL_Y_ROW, TOL_DX_ROW = TOL_Y, TOL_G

# ---------------------------------------------------------------------------------------------------------------------------------
# the schedule of csrc/sra_train.cu and csrc/wgmma_gemm.cuh, restated
# ---------------------------------------------------------------------------------------------------------------------------------
LN_WARPS = 8      # ln_bwd_kernel: 256 threads = 8 warps, one row per warp and pass; grid 2 x SMs (launch_ln_bwd)
DW_ROWS = 64      # dw_gemm_kernel: rows per slab; a split's rows are rounded up to whole slabs


def ln_rows_per_pass(sms):
    """Rows the LayerNorm backward covers per grid-stride pass (ln_bwd_kernel's loop, grid = 2 x SMs)."""
    return LN_WARPS * 2 * sms


def dw_schedule(n, sms, blocks):
    """launch_dw: splits = ceil(2 SMs / blocks) capped at ceil(n / 64); dw_gemm_kernel: rows_per = ceil(n / splits) rounded up to
    64.  Returns (splits, rows_per, non-empty splits)."""
    splits = (2 * sms + blocks - 1) // blocks
    splits = min(splits, max(1, (n + DW_ROWS - 1) // DW_ROWS))
    rows_per = ((n + splits - 1) // splits + DW_ROWS - 1) // DW_ROWS * DW_ROWS
    return splits, rows_per, (n + rows_per - 1) // rows_per


# dW GEMMs of the backward and their output blocks (nb * kb, 128 x 128 each): launch_dw's callers in sstb200_sra_stack_backward
DW_GEMMS = {"dW2": 2, "dW1": 2, "dWo": 1, "dWqk": 2, "dWv": 1}


def wgmma_per_sm(K, NT, f32_stage):
    """launch_wgmma_gemm: dynamic shared memory = max(operands, staging + accumulator tile) + 1 KB; CTAs per SM = 220 KB / (smem + 6 KB)."""
    ops = 128 * K * 2 + NT * K * 2
    stage = 128 * NT * (4 if f32_stage else 2) + 128 * NT * 4
    return max(1, (220 * 1024) // (max(ops, stage) + 1024 + 6144))


# wgmma GEMMs of the forward and backward: (K, NT, fp32 staging tile (EPI_RES_LN / EPI_ADD_F32), ny = n tiles per row tile)
WGMMA_GEMMS = {"qkv": (128, 128, False, 3), "out_proj_ln1": (128, 128, True, 1), "lin1_gelu": (128, 128, False, 2),
              "lin2_ln2": (256, 128, True, 1), "dz_gelugrad": (128, 128, False, 2), "dx1": (256, 128, True, 1),
              "datt": (128, 128, False, 1), "dx": (384, 128, True, 1)}


def wgmma_schedule(n, sms, gemm):
    """(items, grid) of launch_wgmma_gemm for `gemm` at n rows: items = ceil(n / 128) ny, grid = min(SMs per_sm, items)."""
    K, NT, f32, ny = WGMMA_GEMMS[gemm]
    items = (n + 127) // 128 * ny
    return items, min(sms * wgmma_per_sm(K, NT, f32), items)


def stack_edges(sms):
    """{tag: row count} for an SM count: small counts around the 64-row slab and the 128-row tile, and both sides of every
    SM-dependent boundary of the schedule above."""
    e = {str(k): k for k in (1, 2, 63, 64, 65, 127, 128, 129)}
    p = ln_rows_per_pass(sms)                                  # 16 SMs
    e["ln_pass-1"], e["ln_pass+1"] = p - 1, p + 1
    e["dw2_splits-1"], e["dw2_splits+1"] = 64 * sms - 1, 64 * sms + 1       # 2-block dW: SMs splits of 64 rows, then 128-row splits
    e["dw1_splits-1"], e["dw1_splits+1"] = 128 * sms - 1, 128 * sms + 1     # 1-block dW: 2 SMs splits; the 1-per-SM GEMMs wrap
    for name, (K, NT, f32, ny) in WGMMA_GEMMS.items():          # first row count at which some CTA takes a second item
        wrap = 128 * (sms * wgmma_per_sm(K, NT, f32) // ny) + 1
        if wrap not in e.values():
            e[f"{name}_wrap"] = wrap
    return e


EDGE_TAGS = list(stack_edges(132))   # the tags do not depend on the SM count (checked below); the row counts are resolved on the device


def test_stack_edges_hit_every_boundary():
    """For H100 SXM (132 SMs) and PCIe (114): the tags are the same, and for every boundary of the schedule there is a row count
    just below or at it and one just past it."""
    for sms in (132, 114):
        e = stack_edges(sms)
        assert list(e) == EDGE_TAGS
        ns = sorted(set(e.values()))
        # 64-row slabs and 128-row tiles: a full one, one short by a row, one row into the next
        for k in (64, 128):
            assert {k - 1, k, k + 1} <= set(ns)
        # LayerNorm passes: a last pass one row short of full, and a pass holding a single row
        p = ln_rows_per_pass(sms)
        assert p - 1 in ns and p + 1 in ns and p == 16 * sms
        # dW: every split non-empty, then some split empty, for both block counts
        for name, blocks in DW_GEMMS.items():
            sched = [dw_schedule(n, sms, blocks) for n in ns]
            assert any(s == ne and s == (2 * sms + blocks - 1) // blocks for s, _, ne in sched), name
            full = [n for n, (s, rp, ne) in zip(ns, sched) if ne == s == (2 * sms + blocks - 1) // blocks]
            empty = {n for n, (s, rp, ne) in zip(ns, sched) if ne < s}
            assert any(n + 2 in empty for n in full), name             # the two sides of the same boundary
        # wgmma GEMMs: the first row count at which a CTA takes a second item is tested, and one tile fewer wraps no CTA
        for name, (K, NT, f32, ny) in WGMMA_GEMMS.items():
            cap = sms * wgmma_per_sm(K, NT, f32)
            first = 128 * (cap // ny) + 1
            assert first in ns, name
            assert wgmma_schedule(first, sms, name)[0] > cap >= wgmma_schedule(first - 1, sms, name)[0], name
        # the q|k|v GEMM runs 2 CTAs per SM, the LayerNorm epilogues 1, the datt GEMM 2 (wraps at 256 SMs)
        assert wgmma_per_sm(128, 128, False) == 2 and wgmma_per_sm(128, 128, True) == 1 and wgmma_per_sm(384, 128, True) == 1
        assert e["qkv_wrap"] == 128 * (2 * sms // 3) + 1 and e["datt_wrap"] == 256 * sms + 1


# ---------------------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------------------
def _sms(cuda):
    from sst_b200 import _lib as L
    return L.lib().sstb200_num_sms(L.ctx(cuda))


def _voxels(n, seed):
    """n distinct voxels of one sweep: a 12 x 12 window holds at most 144, so no voxel is dropped and the stack sees n rows.  The
    cells come from a square of about 4 n cells, so that windows hold a few dozen voxels and attention mixes rows."""
    g = torch.Generator().manual_seed(seed)
    side = min(GRID[0], max(2, int((4 * n) ** 0.5) + 1))
    cell = torch.randperm(side * side, generator=g)[:n]
    coors = torch.stack([torch.zeros_like(cell), torch.zeros_like(cell), cell // side, cell % side], 1).int()
    return torch.randn(n, 128, generator=g), coors


def _model(layer_cfg, blocks=1, ln_shift=None):
    """bf16 SSTv2 with non-trivial norms and biases; taus ~ U[0.1, 0.6].  ln_shift = c puts c (+ noise) into out_proj.bias and
    linear2.bias, i.e. into the pre-LayerNorm sums, without touching any GEMM operand."""
    from sst_b200.sst_modules import SSTv2
    torch.manual_seed(0)
    m = SSTv2(d_model=[128] * blocks, nhead=[8] * blocks, num_blocks=blocks, dim_feedforward=[256] * blocks, output_shape=[468, 468],
              num_attached_conv=0, to_bev=False, precision="bf16", layer_cfg=layer_cfg)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("tau"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.5 + 0.1)
            elif p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            if ln_shift is not None and (n_.endswith("out_proj.bias") or n_.endswith("linear2.bias")):
                p.copy_(ln_shift + torch.randn(p.shape, generator=g) * 0.05)
    return m


def _oracle_weights(m):
    """float64 leaf copies of the module's state; a shared tau enters as 8 equal per-head copies (their gradients sum to its)."""
    return {k: (v.detach().reshape(-1)[:1].expand(1, 8, 1, 1) if k.endswith("tau") and v.numel() == 1 else v.detach())
            .double().clone().requires_grad_(True) for k, v in m.state_dict().items()}


def _tau_err(got, ref_heads):
    """As test_gpu_train_cosine.py: per-head tau against the layer's largest |d tau|; a shared tau against the sum of the eight
    heads' |shares| (the shares can cancel).  With one voxel per window every softmax is 1 and d tau is exactly 0: so must the
    kernel's be."""
    ref_heads = ref_heads.reshape(-1)
    if ref_heads.abs().max().item() == 0:
        return 0.0 if (got == 0).all() else float("inf")
    if got.numel() == ref_heads.numel():
        return (got.reshape(-1) - ref_heads).abs().max().item() / ref_heads.abs().max().item()
    return abs(got.reshape(-1)[0].item() - ref_heads.sum().item()) / ref_heads.abs().sum().item()


def probe_rows(n, sms):
    """Rows on the boundaries of the schedule at n rows: the first and last row, the first row of the last 128-row tile, the
    first row of the last non-empty dW split (both block counts), and the rows on either side of the last LayerNorm pass
    boundary."""
    rows = {0, n - 1, (n - 1) // 128 * 128}
    for blocks in (1, 2):
        _, rows_per, ne = dw_schedule(n, sms, blocks)
        rows.add((ne - 1) * rows_per)
    p = ln_rows_per_pass(sms)
    b = (n - 1) // p * p
    if b > 0:
        rows |= {b - 1, b}
    return sorted(r for r in rows if 0 <= r < n)


def _upstream(n, sms, mode, seed):
    g = torch.Generator().manual_seed(seed)
    dy = torch.randn(n, 128, generator=g)
    if mode == "probe":
        keep = torch.zeros(n, dtype=torch.bool)
        keep[probe_rows(n, sms)] = True
        dy[~keep] = 0.0
    return dy


def _run(cuda, n, layer_cfg, blocks=1, modes=("dense", "probe"), ln_shift=None):
    """Forward + backward of the training path and of float64 autograd through the oracle, for each upstream-gradient mode.
    Returns (y, y_ref, {mode: (dx, dx_ref, {name: (grad, grad_ref)})})."""
    from sst_b200.sst_modules import SSTInputLayerV2
    sms = _sms(cuda)
    feats, coors = _voxels(n, 100 + n)
    m = _model(layer_cfg, blocks, ln_shift)
    w = _oracle_weights(m)
    xo = feats.double().requires_grad_(True)
    info_o = O.input_layer_v2(xo, coors, DROP_TEST, WIN, GRID)
    assert info_o["voxel_feats"].shape[0] == n
    yo = O.sstv2_forward(info_o, w, [8] * blocks, blocks, "gelu", layer_cfg)
    il = SSTInputLayerV2(DROP_TEST, WIN, GRID, shuffle_voxels=False, mute=True).train()
    m = m.to(cuda).train()
    xg = feats.to(cuda).requires_grad_(True)
    info = il(xg, coors.to(cuda), 1)
    assert info["voxel_feats"].shape[0] == n
    yg = m(info)[0]["voxel_feats"]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    out = {}
    for i, mode in enumerate(modes):
        dy = _upstream(n, sms, mode, 5 + i)
        last = i + 1 == len(modes)
        gref = torch.autograd.grad(yo, [xo] + [w[k] for k in names], dy.double(), retain_graph=not last)
        got = torch.autograd.grad(yg, [xg] + params, dy.to(cuda), retain_graph=not last)
        out[mode] = (got[0].cpu(), gref[0], {k: (g.cpu(), r) for k, g, r in zip(names, got[1:], gref[1:])})
    return yg.detach().cpu(), yo.detach(), out


def _close(got, ref, tol, what):
    got = got.double()
    assert torch.isfinite(got).all(), what
    scale = ref.abs().max().item()
    torch.testing.assert_close(got, ref, rtol=tol, atol=tol * scale, msg=lambda s: f"{what}: {s}")


def _rows_close(got, ref, tol, what):
    """Row by row against the row's own max |ref|; a row whose reference is exactly 0 must be exactly 0."""
    got = got.double()
    err = (got - ref).abs().amax(1)
    scale = ref.abs().amax(1)
    zero = scale == 0
    assert (err[zero] == 0).all(), f"{what}: rows {zero.nonzero().flatten()[:8].tolist()} should be exactly 0"
    rel = err[~zero] / scale[~zero]
    if rel.numel():
        worst = rel.argmax().item()
        assert rel.max().item() < tol, f"{what}: row {(~zero).nonzero().flatten()[worst].item()} rel err {rel.max().item():.3e}"


def _worst(got, ref):
    """(max error / max |ref|, worst row's max error / that row's max |ref|) - printed with -s, to compare with the bounds."""
    err, scale = (got.double() - ref).abs(), ref.abs()
    rows = err.amax(-1) / scale.amax(-1).clamp_min(1e-300)
    return err.max().item() / max(scale.max().item(), 1e-300), rows.max().item()


def _check(y, yo, out, label):
    report = {"y": _worst(y, yo)}
    for mode, (dx, dxo, grads) in out.items():
        report[f"{mode} dx"] = _worst(dx, dxo)
        report[f"{mode} grads"] = max((_tau_err(g, r) if k.endswith("tau") else _worst(g, r)[0], k.split(".", 3)[-1])
                                      for k, (g, r) in grads.items())
    print(f"\n[{label}] " + ", ".join(f"{k} {v[0]:.2e}/{v[1]:.2e}" if not isinstance(v[1], str) else f"{k} {v[0]:.2e} ({v[1]})"
                                     for k, v in report.items()))
    _close(y, yo, TOL_Y, f"{label} y")
    _rows_close(y, yo, TOL_Y_ROW, f"{label} y")
    for mode, (dx, dxo, grads) in out.items():
        _close(dx, dxo, TOL_G, f"{label} {mode} dx")
        _rows_close(dx, dxo, TOL_DX_ROW, f"{label} {mode} dx")
        for name, (g, r) in grads.items():
            if name.endswith("tau"):
                if mode == "probe":   # attention is not row-tiled; d tau is held to its bound with every window contributing
                    continue
                err = _tau_err(g, r)
                assert err < TOL_TAU, f"{label} {mode} {name}: d tau err {err:.3e}"
            else:
                assert g.shape == r.shape, name
                _close(g, r, TOL_G, f"{label} {mode} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("edge", EDGE_TAGS)
def test_plain_stack_edges(cuda, edge):
    """One block (both window shifts), plain attention, at every edge of the schedule; dense and probe upstream gradients."""
    n = stack_edges(_sms(cuda))[edge]
    y, yo, out = _run(cuda, n, {})
    _check(y, yo, out, f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("non_shared", [False, True], ids=["shared_tau", "per_head_tau"])
@pytest.mark.parametrize("edge", ["1", "65", "129", "dw1_splits+1"])
def test_cosine_stack_edges(cuda, edge, non_shared):
    n = stack_edges(_sms(cuda))[edge]
    y, yo, out = _run(cuda, n, dict(cosine=True, tau_min=0.01, non_shared_tau=non_shared))
    _check(y, yo, out, f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["65", "dw2_splits+1"])
def test_two_block_stack_edges(cuda, edge):
    """Two blocks (4 layers): the inner layers' dx goes through the ping-pong pair of buffers of the backward."""
    n = stack_edges(_sms(cuda))[edge]
    y, yo, out = _run(cuda, n, {}, blocks=2)
    _check(y, yo, out, f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0.0, 64.0, 256.0, 1024.0])
def test_layernorm_shift(cuda, shift):
    """A common offset c in every pre-LayerNorm row (through out_proj.bias and linear2.bias): LayerNorm is shift-invariant, so y,
    dx and every gradient must still match float64.  The training LayerNorms (EPI_RES_LN, ln_bwd_kernel) take the variance from
    the centred values; E[t^2] - mean^2 in fp32 would reach the bounds at c = 256 and cancel to 0 at c = 1024."""
    y, yo, out = _run(cuda, 300, {}, modes=("dense",), ln_shift=shift)
    _check(y, yo, out, f"c={shift}")


# ---------------------------------------------------------------------------------------------------------------------------------
# contract of sstb200_sra_stack_backward, through the C ABI
# ---------------------------------------------------------------------------------------------------------------------------------
class _Stack:
    """One forward_train through the C ABI, kept so that the backward can be called on it several times."""

    def __init__(self, cuda, n, layer_cfg, blocks=1):
        from sst_b200 import _lib as L
        from sst_b200.sst_modules import SSTInputLayerV2, _SraLayer, make_sra_plan
        from sst_b200.train import _LayerWt, layer_params
        feats, coors = _voxels(max(n, 1), 100 + n)
        self.m = _model(layer_cfg, blocks).to(cuda).train()
        il = SSTInputLayerV2(DROP_TEST, WIN, GRID, shuffle_voxels=False, mute=True).train()
        with torch.no_grad():
            info = il(feats.to(cuda), coors.to(cuda), 1)
        self.info = info   # owns the plans' device tensors, which the plan structs below point into
        self.layers = [l for blk in self.m.block_list for l in blk.encoder_list]
        self.L, self.lib, self.c = L, L.lib(), L.ctx(cuda)
        self.n, self.dev = n, cuda
        structs, self.keep, wts = [], [], []
        for layer in self.layers:
            s = layer._struct(0)
            ps = layer_params(layer)
            w16 = [ps[j].detach().to(torch.bfloat16).contiguous() for j in (0, 2, 4, 6)]
            s.in_proj_w_f16, s.out_proj_w_f16, s.lin1_w_f16, s.lin2_w_f16 = [t.data_ptr() for t in w16]
            wt = [t.t().contiguous() for t in w16]
            self.keep += w16 + wt
            structs.append(s)
            wts.append(_LayerWt(*[t.data_ptr() for t in wt]))
        self.arr = (_SraLayer * len(structs))(*structs)
        self.wta = (_LayerWt * len(wts))(*wts)
        self.p0, self.p1 = make_sra_plan(info["sra_plan_shift0"]), make_sra_plan(info["sra_plan_shift1"])
        self.x = info["voxel_feats"].float().contiguous()[:n].clone()
        self.ws = torch.empty((self.lib.sstb200_sra_train_workspace_bytes(n, len(self.layers)),), dtype=torch.uint8, device=cuda)
        self.y = torch.full((max(n, 1), 128), 7.0, device=cuda)
        self.x_ptr = self.x.data_ptr() if n else self.y.data_ptr()
        L.check(self.c, self.lib.sstb200_sra_stack_forward_train(self.c, self.arr, len(self.layers), C.byref(self.p0), C.byref(self.p1),
                                                                 self.x_ptr, self.y.data_ptr(), self.ws.data_ptr(), n))

    def grads_like(self, fill=None, seed=0):
        """Per layer, fp32 buffers in the order of sstb200_sra_layer_grads: zeros, or random values."""
        from sst_b200.train import layer_params
        g = torch.Generator().manual_seed(seed)
        out = []
        for layer in self.layers:
            ps = layer_params(layer)
            out.append([(torch.randn(p.shape, generator=g) if fill == "random" else torch.zeros(p.shape)).to(self.dev) for p in ps])
        return out

    def backward(self, dy, grads, dx):
        from sst_b200.train import _LayerGrads
        gs = [_LayerGrads(*[t.data_ptr() for t in gl]) for gl in grads]
        ga = (_LayerGrads * len(gs))(*gs)
        self.L.check(self.c, self.lib.sstb200_sra_stack_backward(self.c, self.arr, self.wta, ga, len(self.layers), C.byref(self.p0),
                                                                 C.byref(self.p1), self.x_ptr, self.ws.data_ptr(), dy.data_ptr(),
                                                                 dx.data_ptr(), self.n))
        torch.cuda.synchronize()


CONTRACT_CASES = [({}, "dw1_splits+1"), (dict(cosine=True, tau_min=0.01, non_shared_tau=True), "ln_pass+1")]


@pytest.mark.gpu
@pytest.mark.parametrize("layer_cfg,edge", CONTRACT_CASES, ids=["plain", "cosine_per_head_tau"])
def test_backward_is_bit_reproducible(cuda, layer_cfg, edge):
    """Two backward calls on the same forward state: identical dx and identical bits in every parameter gradient."""
    s = _Stack(cuda, stack_edges(_sms(cuda))[edge], layer_cfg)
    dy = torch.randn(s.n, 128, generator=torch.Generator().manual_seed(3)).to(cuda)
    runs = []
    for _ in range(2):
        g, dx = s.grads_like(), torch.empty_like(s.x)
        s.backward(dy, g, dx)
        runs.append((dx, g))
    assert torch.equal(runs[0][0], runs[1][0]), "dx differs between two calls"
    from sst_b200.train import layer_params
    for li, layer in enumerate(s.layers):
        names = ["in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "lin1_w", "lin1_b", "lin2_w", "lin2_b", "norm1_w", "norm1_b",
                 "norm2_w", "norm2_b", "tau"][:len(layer_params(layer))]
        for name, a, b in zip(names, runs[0][1][li], runs[1][1][li]):
            assert torch.equal(a, b), f"layer {li} d {name} differs between two calls"


@pytest.mark.gpu
@pytest.mark.parametrize("layer_cfg,edge", CONTRACT_CASES, ids=["plain", "cosine_per_head_tau"])
def test_backward_adds_to_grads(cuda, layer_cfg, edge):
    """The call adds to `grads`: prefilled with G0 it leaves exactly G0 + g, g being what it writes into zeroed buffers."""
    s = _Stack(cuda, stack_edges(_sms(cuda))[edge], layer_cfg)
    dy = torch.randn(s.n, 128, generator=torch.Generator().manual_seed(4)).to(cuda)
    g, dx = s.grads_like(), torch.empty_like(s.x)
    s.backward(dy, g, dx)
    g0 = s.grads_like("random", seed=9)
    acc, dx2 = [[t.clone() for t in gl] for gl in g0], torch.empty_like(s.x)
    s.backward(dy, acc, dx2)
    assert torch.equal(dx, dx2)
    for li in range(len(g)):
        for k, (a, z, r) in enumerate(zip(acc[li], g0[li], g[li])):
            assert torch.equal(a, z + r), f"layer {li} gradient {k}: not G0 + g"


@pytest.mark.gpu
def test_zero_rows_touch_nothing(cuda):
    """n == 0: both entry points return SSTB_OK; dx and every gradient buffer keep their contents."""
    s = _Stack(cuda, 0, dict(cosine=True, tau_min=0.01))
    assert (s.y == 7.0).all()
    g0 = s.grads_like("random", seed=2)
    acc = [[t.clone() for t in gl] for gl in g0]
    dy, dx = torch.ones(1, 128, device=cuda), torch.full((1, 128), 3.0, device=cuda)
    s.backward(dy, acc, dx)
    assert (dx == 3.0).all()
    for a, b in zip(sum(acc, []), sum(g0, [])):
        assert torch.equal(a, b)
