"""Training path of the hot modules (BASELINE config 4): autograd bridges onto the C ABI's training entry points.

    SraStackFunction      SSTv2's encoder stack: sstb200_sra_stack_forward_train / sstb200_sra_stack_backward (csrc/sra_train.cu)
    FlatAdamW             one fused AdamW kernel over a flat fp32 parameter buffer (sstb200_adamw_step)

The reference trains through torch autograd over models/sst/sst_basic_block_v2.py:100-126 / backbones/sst_v2.py:129-133 under
mmcv fp16 autocast (configs/sst_refactor/sst_waymoD5_1x_3class_8heads_v2.py:82); here forward and backward are the library's
own kernels with bf16 GEMM operands and fp32 everything else.
"""
import ctypes as C

import torch

from . import _lib as L

class _LayerWt(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("in_proj_wt", "out_proj_wt", "lin1_wt", "lin2_wt")]


class _LayerGrads(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "lin1_w", "lin1_b", "lin2_w", "lin2_b",
                                          "norm1_w", "norm1_b", "norm2_w", "norm2_b", "tau")]


def _register():
    from .sst_modules import _SraLayer, _SraPlan
    P = C.POINTER
    L.SIGNATURES["sstb200_sra_train_workspace_bytes"] = (C.c_size_t, [C.c_int, C.c_int])
    L.SIGNATURES["sstb200_sra_stack_forward_train"] = (C.c_int, [L.vp, P(_SraLayer), C.c_int, P(_SraPlan), P(_SraPlan), L.vp, L.vp, L.vp, C.c_int])
    L.SIGNATURES["sstb200_sra_stack_backward"] = (C.c_int, [L.vp, P(_SraLayer), P(_LayerWt), P(_LayerGrads), C.c_int, P(_SraPlan), P(_SraPlan),
                                                            L.vp, L.vp, L.vp, L.vp, C.c_int])
    L.SIGNATURES["sstb200_adamw_step"] = (C.c_int, [L.vp, L.vp, L.vp, L.vp, L.vp, C.c_longlong, C.c_float, C.c_float, C.c_float, C.c_float,
                                                    C.c_float, C.c_int, C.c_float])


_register()


def layer_params(layer):
    """The parameters of an EncoderLayer in the order of sstb200_sra_layer_grads: 12, plus win_attn.self_attn.tau last for a
    cosine-attention layer."""
    sa = layer.win_attn.self_attn
    ps = [sa.in_proj_weight, sa.in_proj_bias, sa.out_proj.weight, sa.out_proj.bias, layer.linear1.weight, layer.linear1.bias,
          layer.linear2.weight, layer.linear2.bias, layer.norm1.weight, layer.norm1.bias, layer.norm2.weight, layer.norm2.bias]
    if layer.win_attn.cosine:
        ps.append(sa.tau)
    return ps


def _param_offsets(layers):
    """Start of every layer's parameters in the flat argument list of SraStackFunction."""
    offs, o = [], 0
    for layer in layers:
        offs.append(o)
        o += len(layer_params(layer))
    return offs, o


class SraStackFunction(torch.autograd.Function):
    """y = encoder_stack(x); parameters are explicit inputs so that autograd routes their gradients."""

    @staticmethod
    def forward(ctx, x, layers, plans, make_plan, *params):
        from .sst_modules import _SraLayer
        _register()
        offs, total = _param_offsets(layers)
        assert len(params) == total
        dev = x.device
        x = x.detach().float().contiguous()
        n = x.shape[0]
        lib, c = L.lib(), L.ctx(dev)
        structs, keep = [], []
        for i, layer in enumerate(layers):
            s = layer._struct(0)                        # fp32 pointers, shapes, eps
            w16 = [params[offs[i] + j].detach().to(torch.bfloat16).contiguous() for j in (0, 2, 4, 6)]
            s.in_proj_w_f16, s.out_proj_w_f16, s.lin1_w_f16, s.lin2_w_f16 = [w.data_ptr() for w in w16]
            structs.append(s)
            keep.append(w16)
        arr = (_SraLayer * len(layers))(*structs)
        p0, p1 = make_plan(plans[0]), make_plan(plans[1])
        ws_bytes = lib.sstb200_sra_train_workspace_bytes(n, len(layers))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        y = torch.empty_like(x)
        L.check(c, lib.sstb200_sra_stack_forward_train(c, arr, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(), ws.data_ptr(), n))
        ctx.layers, ctx.plans, ctx.make_plan = layers, plans, make_plan
        ctx.save_for_backward(x, ws, *params)
        ctx.keep = keep
        return y

    @staticmethod
    def backward(ctx, dy):
        from .sst_modules import _SraLayer
        x, ws, *params = ctx.saved_tensors
        layers = ctx.layers
        dev = x.device
        n = x.shape[0]
        lib, c = L.lib(), L.ctx(dev)
        dy = dy.detach().float().contiguous()
        offs, _ = _param_offsets(layers)
        structs, wts, grads, gstructs, keep = [], [], [], [], []
        for i, layer in enumerate(layers):
            s = layer._struct(0)
            w16 = ctx.keep[i]
            s.in_proj_w_f16, s.out_proj_w_f16, s.lin1_w_f16, s.lin2_w_f16 = [w.data_ptr() for w in w16]
            structs.append(s)
            wt = [w.t().contiguous() for w in w16]          # bf16 [in, out]
            keep.append(wt)
            wts.append(_LayerWt(*[w.data_ptr() for w in wt]))
            g = [torch.zeros_like(params[offs[i] + j], dtype=torch.float32) for j in range(len(layer_params(layer)))]
            grads.extend(g)
            gstructs.append(_LayerGrads(*[t.data_ptr() for t in g]))
        arr = (_SraLayer * len(layers))(*structs)
        wta = (_LayerWt * len(layers))(*wts)
        ga = (_LayerGrads * len(layers))(*gstructs)
        p0, p1 = ctx.make_plan(ctx.plans[0]), ctx.make_plan(ctx.plans[1])
        dx = torch.empty_like(x)
        L.check(c, lib.sstb200_sra_stack_backward(c, arr, wta, ga, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), ws.data_ptr(),
                                                  dy.data_ptr(), dx.data_ptr(), n))
        del keep
        return (dx, None, None, None, *grads)


class FlatAdamW:
    """AdamW over ONE flat fp32 buffer that the parameters are views of (so a single NCCL all-reduce covers every gradient and a
    single kernel does the update).  `params`: iterable of leaf tensors on one CUDA device; after construction each p.data and
    p.grad is a view into .flat / .flat_grad.  Every view starts on a 16-byte boundary (the kernels read parameters such as LayerNorm
    weights as float4), so a parameter whose size is not a multiple of 4 (e.g. a cosine-attention layer's one-element tau) is followed
    by zero padding; padding has zero gradient and stays zero under the update."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        _register()
        self.params = [p for p in params if p.requires_grad]
        dev = self.params[0].device
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.flat = torch.zeros((n,), dtype=torch.float32, device=dev)
        self.flat_grad = torch.zeros((n,), dtype=torch.float32, device=dev)
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
        with torch.no_grad():
            for p, o in zip(self.params, offs):
                k = p.numel()
                self.flat[o:o + k].copy_(p.detach().reshape(-1))
                p.data = self.flat[o:o + k].view_as(p)
                p.grad = self.flat_grad[o:o + k].view_as(p)
                # p keeps its own version counter, which no write through the buffer moves: caches derived from p (the 16-bit
                # weight copies and folded BatchNorms of spconv_modules) also key on the buffer's
                p._flat_base = self.flat
        self.lr, self.betas, self.eps, self.wd, self.t = lr, betas, eps, weight_decay, 0

    def zero_grad(self):
        self.flat_grad.zero_()

    def step(self, grad_scale=1.0):
        self.t += 1
        c = L.ctx(self.flat.device)
        L.check(c, L.lib().sstb200_adamw_step(c, self.flat.data_ptr(), self.flat_grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                              self.flat.numel(), self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.t,
                                              float(grad_scale)))
        # the kernel wrote through a raw pointer: tell torch, as an in-place torch op on the buffer would have
        torch.autograd.graph.increment_version(self.flat)


class TrainStep:
    """One data-parallel training step of the SST hot path (BASELINE config 4), per rank:

        points of B frames -> dynamic_voxelize -> DynamicVFE (train) -> SSTInputLayerV2 (train drop_info, shuffle) -> SSTv2 (bf16)
        -> loss = mean(out^2) (the stand-in head of SURVEY 8d) -> backward -> ONE flat NCCL all-reduce of every gradient
        -> fused AdamW (gradient averaged over the ranks inside the kernel).

    mirrors the reference's DynamicVoxelNet.forward_train under MMDistributedDataParallel + Fp16OptimizerHook + AdamW
    (detectors/dynamic_voxelnet.py:38-71, tools/dist_train.sh:7-9, configs/_base_/schedules/cosine_2x.py) for the part of the
    model that is on the hot path.  naiveSyncBN exchanges its statistics inside the forward (sst_b200/norm.py)."""

    def __init__(self, vfe, il, bb, voxel_size, pc_range, lr=1e-4, weight_decay=0.05):
        import torch.distributed as dist
        self.vfe, self.il, self.bb = vfe.train(), il.train(), bb.train()
        self.vs, self.rng = voxel_size, pc_range
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.opt = FlatAdamW(list(vfe.parameters()) + list(bb.parameters()), lr=lr, weight_decay=weight_decay)
        self.ar_events = []

    def voxelize(self, frames):
        """DynamicVoxelNet.voxelize (dynamic_voxelnet.py:49-71): per-frame dynamic_voxelize, batch index prepended."""
        from . import ops
        pts, coors = [], []
        for b, p in enumerate(frames):
            c = torch.zeros((p.shape[0], 3), dtype=torch.int32, device=p.device)
            ops.dynamic_voxelize(p.contiguous(), c, self.vs, self.rng)
            coors.append(torch.nn.functional.pad(c, (1, 0), value=b))
            pts.append(p)
        return torch.cat(pts), torch.cat(coors)

    def step(self, frames, time_allreduce=False):
        import torch.distributed as dist
        self.opt.zero_grad()
        pts, coors = self.voxelize(frames)
        vf, vc = self.vfe(pts, coors)
        info = self.il(vf, vc, len(frames))
        out = self.bb(info)[0]["voxel_feats"]
        loss = out.float().square().mean()
        loss.backward()
        if self.world > 1:
            if time_allreduce:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
            dist.all_reduce(self.opt.flat_grad)           # ONE collective over the flat gradient buffer (NCCL over NVLink)
            if time_allreduce:
                b.record()
                self.ar_events.append((a, b))
        self.opt.step(grad_scale=1.0 / self.world)
        return loss.detach()

    @property
    def grad_bytes(self):
        return self.opt.flat_grad.numel() * 4
