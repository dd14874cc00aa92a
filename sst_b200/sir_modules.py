"""FSD's SIR modules under the reference's registered names (S1-S3).

    SIRLayer   mmdet3d/models/voxel_encoders/voxel_encoder.py:617-764
    SIR        mmdet3d/models/backbones/sir.py:15-87

Same constructor kwargs / forward signatures / state-dict keys (`rel_mlp.{k}.{0,1}.*`,
`vfe_layers.{j}.{linear,norm}.*`).  Eval forward = one sstb200_sir_layer_forward call per block; with gradients, one
SirLayerFunction (sstb200_sir_layer_forward_train / _backward, fp32) per block.
"""
import ctypes as C

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib as L
from . import ops
from .registry import BACKBONES, VOXEL_ENCODERS
from .voxel_modules import DynamicVFELayerV2


class _SirLayer(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("rel_in", C.c_int32), ("num_rel", C.c_int32), ("rel_dims", C.c_int32 * 4),
                ("num_vfe", C.c_int32), ("feat_channels", C.c_int32 * 2), ("act", C.c_int32), ("mode_max", C.c_int32),
                ("with_shortcut", C.c_int32), ("norm_eps", C.c_float), ("xyz_normalizer", C.c_float * 3),
                ("rel_dist_scaler", C.c_float), ("rel_w", C.c_void_p * 4), ("rel_ln_w", C.c_void_p * 4),
                ("rel_ln_b", C.c_void_p * 4), ("vfe_w", C.c_void_p * 2), ("vfe_ln_w", C.c_void_p * 2),
                ("vfe_ln_b", C.c_void_p * 2)]


L.SIGNATURES["sstb200_sir_layer_forward"] = (C.c_int, [L.vp, C.POINTER(_SirLayer), L.vp, L.vp, L.vp, C.c_int, C.c_int,
                                                       L.vp, L.vp])
L.SIGNATURES["sstb200_sir_layer_forward_ex"] = (C.c_int, [L.vp, C.POINTER(_SirLayer), L.vp, C.c_int, C.c_int, C.c_int, L.vp, L.vp,
                                                          C.c_int, C.c_int, L.vp, L.vp, C.c_int, L.vp, C.c_int, L.vp])
L.SIGNATURES["sstb200_group_csr"] = (C.c_int, [L.vp, L.vp, C.c_int, C.c_int, L.vp, L.vp])
_PREC = {"fp32": 0, "bf16": 1}


class _SirGrads(C.Structure):
    _fields_ = [("rel_w", C.c_void_p * 4), ("rel_ln_w", C.c_void_p * 4), ("rel_ln_b", C.c_void_p * 4), ("vfe_w", C.c_void_p * 2),
                ("vfe_ln_w", C.c_void_p * 2), ("vfe_ln_b", C.c_void_p * 2)]


L.SIGNATURES["sstb200_sir_layer_train_state_bytes"] = (C.c_size_t, [C.POINTER(_SirLayer), C.c_int, C.c_int])
L.SIGNATURES["sstb200_sir_layer_forward_train"] = (C.c_int, [L.vp, C.POINTER(_SirLayer), L.vp, L.vp, L.vp, C.c_int, C.c_int, L.vp, L.vp,
                                                             L.vp, L.vp, L.vp, C.c_size_t])
L.SIGNATURES["sstb200_sir_layer_backward"] = (C.c_int, [L.vp, C.POINTER(_SirLayer), L.vp, L.vp, L.vp, C.c_int, C.c_int, L.vp, L.vp, L.vp,
                                                        C.c_size_t, L.vp, L.vp, L.vp, L.vp, C.POINTER(_SirGrads)])


class SirLayerFunction(torch.autograd.Function):
    """(point_feats [N, C_last], group_feats [G, C0+C1]) = one SIRLayer in fp32 through sstb200_sir_layer_forward_train /
    _backward.  The parameters are explicit inputs (SIRLayer._train_params order) so that autograd routes their gradients;
    the layer's state (pre-LN values and arg-max rows) lives on ctx until the backward."""

    @staticmethod
    def forward(ctx, layer, with_shortcut, in_feats, f_cluster, unq_inv, num_groups, csr, *params):
        ops._need_cuda(in_feats, f_cluster, unq_inv)
        in_feats = in_feats.float().contiguous()
        f_cluster = f_cluster.float().contiguous()
        unq_inv = unq_inv.long().contiguous()
        params = [p.contiguous() for p in params]
        N, G, dev = in_feats.shape[0], num_groups, in_feats.device
        assert in_feats.shape[1] == layer.in_channels and f_cluster.shape == (N, layer.rel_in), (in_feats.shape, f_cluster.shape)
        point = torch.empty((N, layer.feat_channels[-1]), dtype=torch.float32, device=dev)
        group = torch.empty((G, sum(layer.feat_channels)), dtype=torch.float32, device=dev)
        s = layer._struct(params)
        s.with_shortcut = int(with_shortcut)
        if csr is None and N and G:
            csr = group_csr(unq_inv, G)
        off, order = csr if csr is not None else (None, None)
        nbytes = L.lib().sstb200_sir_layer_train_state_bytes(C.byref(s), N, G)
        state = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        c = L.ctx(dev)
        L.check(c, L.lib().sstb200_sir_layer_forward_train(
            c, C.byref(s), in_feats.data_ptr(), f_cluster.data_ptr(), unq_inv.data_ptr(), N, G, L.ptr(off), L.ptr(order),
            point.data_ptr(), group.data_ptr(), state.data_ptr(), nbytes))
        ctx.save_for_backward(in_feats, f_cluster, unq_inv, *params)
        ctx.layer, ctx.with_shortcut, ctx.G, ctx.csr, ctx.state = layer, with_shortcut, G, (off, order), state
        ctx.set_materialize_grads(False)  # an unused output arrives as None and is passed as NULL
        return point, group

    @staticmethod
    @once_differentiable
    def backward(ctx, d_point, d_group):
        in_feats, f_cluster, unq_inv, *params = ctx.saved_tensors
        N, G = in_feats.shape[0], ctx.G
        d_point = None if d_point is None else d_point.float().contiguous()
        d_group = None if d_group is None else d_group.float().contiguous()
        want_in, want_fc = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        pg = [torch.zeros_like(p) for p in params]
        if not (N and G and (d_point is not None or d_group is not None)):
            return (None, None, torch.zeros_like(in_feats) if want_in else None, torch.zeros_like(f_cluster) if want_fc else None,
                    None, None, None, *pg)
        g_in = torch.empty_like(in_feats) if want_in else None
        g_fc = torch.empty_like(f_cluster) if want_fc else None
        s = ctx.layer._struct(params)
        s.with_shortcut = int(ctx.with_shortcut)
        gs = _SirGrads()
        for i in range(s.num_rel):
            gs.rel_w[i], gs.rel_ln_w[i], gs.rel_ln_b[i] = (t.data_ptr() for t in pg[3 * i:3 * i + 3])
        for i in range(s.num_vfe):
            gs.vfe_w[i], gs.vfe_ln_w[i], gs.vfe_ln_b[i] = (t.data_ptr() for t in pg[3 * (s.num_rel + i):3 * (s.num_rel + i) + 3])
        off, order = ctx.csr
        c = L.ctx(in_feats.device)
        L.check(c, L.lib().sstb200_sir_layer_backward(
            c, C.byref(s), in_feats.data_ptr(), f_cluster.data_ptr(), unq_inv.data_ptr(), N, G, L.ptr(off), L.ptr(order),
            ctx.state.data_ptr(), ctx.state.numel(), L.ptr(d_point), L.ptr(d_group), L.ptr(g_in), L.ptr(g_fc), C.byref(gs)))
        return (None, None, g_in, g_fc, None, None, None, *pg)


def group_csr(unq_inv, num_groups):
    """(offsets [G+1] int32, order [N] int32): points grouped by their group id - shared by the blocks of a SIR backbone."""
    ops._need_cuda(unq_inv)
    unq_inv = unq_inv.long().contiguous()
    N, dev = unq_inv.shape[0], unq_inv.device
    offsets = torch.empty((num_groups + 1,), dtype=torch.int32, device=dev)
    order = torch.empty((N,), dtype=torch.int32, device=dev)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_group_csr(c, unq_inv.data_ptr(), N, num_groups, offsets.data_ptr(), order.data_ptr()))
    return offsets, order


@VOXEL_ENCODERS.register_module()
class SIRLayer(nn.Module):
    """voxel_encoder.py:617-764."""

    def __init__(self, in_channels=4, feat_channels=[], with_distance=False, with_cluster_center=False, with_rel_mlp=True,
                 rel_mlp_hidden_dims=[16, ], rel_mlp_in_channel=3, with_voxel_center=False, voxel_size=(0.2, 0.2, 4),
                 point_cloud_range=(0, -40, -3, 70.4, 40, 1), norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01),
                 mode="max", fusion_layer=None, return_point_feats=False, return_inv=True, rel_dist_scaler=1.0,
                 with_shortcut=True, xyz_normalizer=[1.0, 1.0, 1.0], act="relu", dropout=0.0):
        super().__init__()
        assert len(feat_channels) > 0
        if with_distance or with_cluster_center or with_voxel_center:
            raise NotImplementedError("SIRLayer extra decorations are unused by the FSD configs and not built")
        self.in_channels = in_channels
        self.return_point_feats = return_point_feats
        self.rel_dist_scaler = rel_dist_scaler
        self.mode = mode
        self.with_shortcut = with_shortcut
        self._with_rel_mlp = with_rel_mlp
        self.xyz_normalizer = xyz_normalizer
        self.act = act
        self.norm_eps = norm_cfg.get("eps", 1e-5)
        self.norm_type = norm_cfg["type"]
        self.dropout_p = dropout
        self.fp16_enabled = False
        if with_rel_mlp:
            # the reference appends in place (voxel_encoder.py:665); a fresh list keeps shared config lists intact
            dims = list(rel_mlp_hidden_dims) + [in_channels]
            self.rel_dims = dims
            self.rel_in = rel_mlp_in_channel
            self.rel_mlp = ops.build_mlp(rel_mlp_in_channel, dims, norm_cfg, act=act)
        chans = [in_channels] + list(feat_channels)
        layers = []
        for i in range(len(chans) - 1):
            cin = chans[i] * (2 if i > 0 else 1)
            if act != "relu" or dropout > 0:
                layers.append(DynamicVFELayerV2(cin, chans[i + 1], norm_cfg, act=act, dropout=dropout))
            else:
                from .voxel_modules import DynamicVFELayer
                layers.append(DynamicVFELayer(cin, chans[i + 1], norm_cfg))
        self.vfe_layers = nn.ModuleList(layers)
        self.num_vfe = len(layers)
        self.feat_channels = list(feat_channels)

    def _train_params(self):
        """The parameters the fused layer reads, in _struct's order: per rel-MLP layer (weight, LN weight, LN bias), then per VFE
        layer (linear weight, LN weight, LN bias)."""
        ps = []
        for i in range(len(self.rel_dims)):
            ps += [self.rel_mlp[i][0].weight, self.rel_mlp[i][1].weight, self.rel_mlp[i][1].bias]
        for l in self.vfe_layers:
            ps += [l.linear.weight, l.norm.weight, l.norm.bias]
        return ps

    def _native_train(self):
        """The variants the fused training path covers (SirLayerFunction); the others train through _forward_composed."""
        return (self.norm_type == "LN" and self._with_rel_mlp and 1 <= self.num_vfe <= 2 and len(self.rel_dims) <= 4
                and self.mode == "max" and self.dropout_p == 0 and self.act in ("relu", "gelu"))

    def _struct(self, params=None):
        if self.norm_type != "LN":
            raise NotImplementedError("fused SIRLayer expects norm_cfg type 'LN' (as in configs/fsd)")
        if not self._with_rel_mlp or self.num_vfe > 2 or len(self.rel_dims) > 4:
            raise NotImplementedError("SIRLayer variant not built")
        ptrs = [p.data_ptr() for p in (self._train_params() if params is None else params)]
        s = _SirLayer()
        s.in_channels, s.rel_in, s.num_rel = self.in_channels, self.rel_in, len(self.rel_dims)
        for i, d in enumerate(self.rel_dims):
            s.rel_dims[i] = d
            s.rel_w[i], s.rel_ln_w[i], s.rel_ln_b[i] = ptrs[3 * i:3 * i + 3]
        s.num_vfe = self.num_vfe
        k = 3 * len(self.rel_dims)
        for i in range(self.num_vfe):
            s.feat_channels[i] = self.feat_channels[i]
            s.vfe_w[i], s.vfe_ln_w[i], s.vfe_ln_b[i] = ptrs[k + 3 * i:k + 3 * i + 3]
        s.act = {"relu": 1, "gelu": 2}[self.act]
        s.mode_max = int(self.mode == "max")
        s.with_shortcut = int(bool(self.with_shortcut))
        s.norm_eps = float(self.norm_eps)
        for i in range(3):
            s.xyz_normalizer[i] = float(self.xyz_normalizer[i])
        s.rel_dist_scaler = float(self.rel_dist_scaler)
        return s

    precision = "fp32"  # 'bf16': rel-MLP layer 3 and both VFE layers on the tensor cores (bf16 operands, fp32 accumulate / LN / pooling)

    def _forward_composed(self, features, coors, f_cluster, return_inv, return_both, unq_inv_once, new_coors_once):
        """voxel_encoder.py:696-764 as a composition when a gradient is needed: torch Linear / LayerNorm / activation modules (autograd)
        around `ops.segment_reduce` (segmented max / mean with their backward kernels) on ONE group index.  The fused kernels above
        are the eval()/no_grad() path."""
        features = features.float()
        if unq_inv_once is None:
            new_coors, unq_inv = ops.unique_rows(coors.long())
        else:
            new_coors, unq_inv = new_coors_once, unq_inv_once
        G = new_coors.shape[0]
        nz = features.new_tensor(self.xyz_normalizer)
        x0 = torch.cat([features[:, :3] / nz[None, :], features[:, 3:]], dim=1)
        shortcut = features[:, 3:]
        if f_cluster is None:
            mean, _ = ops.segment_reduce(features[:, :3].contiguous(), unq_inv, "mean", G, want_argmax=False)
            f_cluster = (features[:, :3] - mean[unq_inv]) / self.rel_dist_scaler
        else:
            f_cluster = f_cluster.float() / self.rel_dist_scaler
        if self._with_rel_mlp:
            x0 = x0 * self.rel_mlp(f_cluster)
        act = ops.get_activation(self.act)
        mode = "mean" if self.mode == "avg" else self.mode
        x, groups, point_feats = x0, [], None
        for i, vfe in enumerate(self.vfe_layers):
            if getattr(vfe, "dropout", None) is not None:
                x = vfe.dropout(x)
            point_feats = act(vfe.norm(vfe.linear(x)))
            g, _ = ops.segment_reduce(point_feats.contiguous(), unq_inv, mode, G)
            groups.append(g)
            if i != len(self.vfe_layers) - 1:
                x = torch.cat([point_feats, g[unq_inv]], dim=1)
        voxel_feats = torch.cat(groups, dim=1)
        if (return_both or self.return_point_feats) and self.with_shortcut and point_feats.shape == shortcut.shape:
            point_feats = point_feats + shortcut
        if return_both:
            return point_feats, voxel_feats, new_coors
        if self.return_point_feats:
            return point_feats, voxel_feats
        if return_inv:
            return voxel_feats, new_coors, unq_inv
        return voxel_feats, new_coors

    def _forward_train(self, features, coors, f_cluster, return_inv, return_both, unq_inv_once, new_coors_once, csr_once):
        """The training forward in fp32 (the reference runs SIRLayer under @force_fp32, whatever `precision` says): one
        SirLayerFunction call; f_cluster=None is built from the group mean here, so autograd carries its gradient to `features`."""
        ops._need_cuda(features, coors)
        features = features.float()
        if unq_inv_once is None:
            new_coors, unq_inv = ops.unique_rows(coors.long())
        else:
            new_coors, unq_inv = new_coors_once, unq_inv_once
        G = new_coors.shape[0]
        if f_cluster is None:  # voxel_encoder.py:717-723 (the division by rel_dist_scaler happens inside the kernels)
            mean, _ = ops.segment_reduce(features[:, :3].contiguous(), unq_inv, "mean", G, want_argmax=False)
            f_cluster = features[:, :3] - mean[unq_inv]
        wants_shortcut = return_both or self.return_point_feats
        point_feats, voxel_feats = SirLayerFunction.apply(self, bool(self.with_shortcut) and wants_shortcut, features, f_cluster.float(),
                                                          unq_inv, G, csr_once, *self._train_params())
        if return_both:
            return point_feats, voxel_feats, new_coors
        if self.return_point_feats:
            return point_feats, voxel_feats
        if return_inv:
            return voxel_feats, new_coors, unq_inv
        return voxel_feats, new_coors

    def forward(self, features, coors, f_cluster=None, points=None, img_feats=None, img_metas=None, return_inv=False,
                return_both=False, unq_inv_once=None, new_coors_once=None, csr_once=None, point_feats_out=None, feat_gap=None):
        """`csr_once` = group_csr(unq_inv, G) shared between blocks; `point_feats_out` = a [N, >=C] fp32 view (last dim
        contiguous) that receives the point features in place of a fresh tensor (bf16 path; SIR.forward uses it to write
        block i's output straight into block i+1's [points || feats] input).  `feat_gap` = (at, width): `features` is that
        hand-over buffer, whose columns >= at sit `width` floats further right (bf16 path)."""
        if torch.is_grad_enabled() and (self.training or features.requires_grad or (f_cluster is not None and f_cluster.requires_grad)):
            if features.is_cuda and self._native_train():
                return self._forward_train(features, coors, f_cluster, return_inv, return_both, unq_inv_once, new_coors_once, csr_once)
            return self._forward_composed(features, coors, f_cluster, return_inv, return_both, unq_inv_once, new_coors_once)
        ops._need_cuda(features, coors)
        features = features.float().contiguous()
        if unq_inv_once is None:
            new_coors, unq_inv = ops.unique_rows(coors.long())
        else:
            new_coors, unq_inv = new_coors_once, unq_inv_once
        G, N = new_coors.shape[0], features.shape[0]
        if f_cluster is None:  # voxel_encoder.py:717-723 (the division by rel_dist_scaler happens inside the kernel)
            mean, _ = ops.segment_reduce(features[:, :3].contiguous(), unq_inv, "mean", G)
            f_cluster = features[:, :3] - mean[unq_inv]
        f_cluster = f_cluster.float().contiguous()
        C_last = self.feat_channels[-1]
        if point_feats_out is not None:
            point_feats = point_feats_out
            assert point_feats.dtype == torch.float32 and point_feats.shape == (N, C_last) and point_feats.stride(1) == 1
            ld = point_feats.stride(0)
        else:
            point_feats = torch.empty((N, C_last), dtype=torch.float32, device=features.device)
            ld = C_last
        voxel_feats = torch.empty((G, sum(self.feat_channels)), dtype=torch.float32, device=features.device)
        s = self._struct()
        wants_shortcut = return_both or self.return_point_feats
        s.with_shortcut = int(bool(self.with_shortcut) and wants_shortcut)
        off, order = csr_once if csr_once is not None else (None, None)
        c = L.ctx(features.device)
        gap_at, gap = feat_gap if feat_gap is not None else (self.in_channels, 0)
        assert features.shape[1] == self.in_channels + gap, (features.shape, self.in_channels, gap)
        L.check(c, L.lib().sstb200_sir_layer_forward_ex(
            c, C.byref(s), features.data_ptr(), features.shape[1], gap_at, gap, f_cluster.data_ptr(),
            unq_inv.contiguous().data_ptr(), N, G, L.ptr(off), L.ptr(order), _PREC[self.precision], point_feats.data_ptr(), ld,
            voxel_feats.data_ptr()))
        if return_both:
            return point_feats, voxel_feats, new_coors
        if self.return_point_feats:
            return point_feats, voxel_feats
        if return_inv:
            return voxel_feats, new_coors, unq_inv
        return voxel_feats, new_coors


@BACKBONES.register_module()
class SIR(nn.Module):
    """models/backbones/sir.py:15-87."""

    def __init__(self, num_blocks=5, in_channels=[], feat_channels=[], rel_mlp_hidden_dims=[], with_rel_mlp=True,
                 with_distance=False, with_cluster_center=False, norm_cfg=dict(type="LN", eps=1e-3), mode="max",
                 xyz_normalizer=[1.0, 1.0, 1.0], act="relu", dropout=0, unique_once=False):
        super().__init__()
        self.num_blocks = num_blocks
        self.unique_once = unique_once
        self.block_list = nn.ModuleList([
            SIRLayer(in_channels=in_channels[i], feat_channels=feat_channels[i], with_distance=with_distance,
                     with_cluster_center=with_cluster_center, with_rel_mlp=with_rel_mlp,
                     rel_mlp_hidden_dims=rel_mlp_hidden_dims[i], with_voxel_center=False, voxel_size=[0.1, 0.1, 0.1],
                     point_cloud_range=[-74.88, -74.88, -2, 74.88, 74.88, 4], norm_cfg=norm_cfg, mode=mode,
                     fusion_layer=None, return_point_feats=(i != num_blocks - 1), return_inv=False, rel_dist_scaler=10.0,
                     xyz_normalizer=xyz_normalizer, act=act, dropout=dropout) for i in range(num_blocks)])

    precision = "fp32"  # forwarded to every block ('bf16' = tensor-core path, see SIRLayer.precision)

    def forward(self, points, features, coors, f_cluster=None):
        # unique + group CSR once regardless of the flag: the result is identical and both are reused by every block
        new_coors, unq_inv = ops.unique_rows(coors.long())
        csr = group_csr(unq_inv, new_coors.shape[0]) if points.shape[0] and new_coors.shape[0] and points.is_cuda else None
        out_feats = features
        cluster_feat_list = []
        out_coors = new_coors
        in_feats = torch.cat([points, out_feats], 1)
        grad = torch.is_grad_enabled() and (self.training or features.requires_grad or points.requires_grad)
        npt = points.shape[1]
        pad = (-npt) % 8  # the feature block of the hand-over buffer starts on a 32-byte boundary
        gap = None
        for i, block in enumerate(self.block_list):
            block.precision = self.precision
            last = i == self.num_blocks - 1
            kw = dict(unq_inv_once=unq_inv, new_coors_once=new_coors, csr_once=csr, feat_gap=gap)
            nxt = None
            Cb = block.feat_channels[-1]
            if (not last and not grad and self.precision == "bf16" and Cb + npt == self.block_list[i + 1].in_channels and Cb % 4 == 0
                    and not (block.with_shortcut and block.in_channels - 3 == Cb)):
                # this block's point features land next to the raw points: no torch.cat between blocks.  Block i >= 1 reads
                # and writes the same buffer (its kernel A has consumed the input before kernel B writes the output).
                if gap is not None and in_feats.shape[1] == npt + pad + Cb:
                    nxt = in_feats
                else:
                    nxt = torch.empty((points.shape[0], npt + pad + Cb), dtype=torch.float32, device=points.device)
                    nxt[:, :npt] = points
                kw["point_feats_out"] = nxt[:, npt + pad:]
            if not last:
                out_feats, out_cluster_feats = block(in_feats, coors, f_cluster, **kw)
                if nxt is not None:
                    in_feats, gap = nxt, (npt, pad)
                else:
                    in_feats, gap = torch.cat([points, out_feats], 1), None
            else:
                out_feats, out_cluster_feats, out_coors = block(in_feats, coors, f_cluster, return_both=True, **kw)
            cluster_feat_list.append(out_cluster_feats)
        return out_feats, torch.cat(cluster_feat_list, dim=1), out_coors
