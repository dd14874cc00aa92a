"""SST modules registered under the reference's type names, backed by libsstb200.

    SSTInputLayerV2, PseudoMiddleEncoderForSpconvFSD   models/middle_encoders/sst_input_layer_v2.py:15-126
    WindowAttention, EncoderLayer, BasicShiftBlockV2   models/sst/sst_basic_block_v2.py:14-169
    SSTv2                                              models/backbones/sst_v2.py:16-196

Constructor kwargs, forward signatures, returned dict keys and state-dict keys follow the reference so that
`configs/sst_refactor/*.py` build unchanged and reference checkpoints load.  The arithmetic is not
torch's: window bucketing is one fused plan per shift (csrc/window.cu) and every encoder layer is the ragged
SRA kernel set (csrc/sra_*.cu); torch only holds parameters and device buffers.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib as L
from . import ops
from .registry import BACKBONES, MIDDLE_ENCODERS


# ------------------------------------------------------------------------------------------------
# lazily-materialised reference-layout views (API parity, never touched by the fused path)
# ------------------------------------------------------------------------------------------------
class _LazyDict(dict):
    def __init__(self, fill):
        super().__init__()
        self._fill_fn = fill

    def _fill(self):
        if self._fill_fn is not None:
            f, self._fill_fn = self._fill_fn, None
            super().update(f())

    def __getitem__(self, k):
        self._fill()
        return super().__getitem__(k)

    def __iter__(self):
        self._fill()
        return super().__iter__()

    def __len__(self):
        self._fill()
        return super().__len__()

    def __contains__(self, k):
        self._fill()
        return super().__contains__(k)

    def keys(self):
        self._fill()
        return super().keys()

    def items(self):
        self._fill()
        return super().items()

    def values(self):
        self._fill()
        return super().values()

    def get(self, k, d=None):
        self._fill()
        return super().get(k, d)


@MIDDLE_ENCODERS.register_module()
class PseudoMiddleEncoderForSpconvFSD(nn.Module):
    def forward(self, voxel_feats, voxel_coors, batch_size=None):
        return {"voxel_feats": voxel_feats, "voxel_coors": voxel_coors}


def _pos_table(window_shape, feat_dim, pos_temperature, normalize_pos):
    """Host-side table of SSTInputLayerV2.get_pos_embed (sst_input_layer_v2.py:238-305): the embedding of a
    token only depends on its in-window coordinate per axis, so [ndim][maxw][L] values cover every token."""
    if len(window_shape) == 2:
        ndim, wins = 2, (window_shape[0], window_shape[1], 0)
    elif window_shape[-1] == 1:
        ndim, wins = 2, (window_shape[0], window_shape[1], 0)
    else:
        ndim, wins = 3, tuple(window_shape)
    Lp = feat_dim // ndim
    maxw = max(int(w) for w in wins[:ndim])
    inv_freq = torch.arange(Lp, dtype=torch.float32)
    inv_freq = pos_temperature ** (2 * (inv_freq // 2) / Lp)
    tab = torch.zeros((ndim, maxw, Lp), dtype=torch.float32)
    for a in range(ndim):
        w = wins[a]
        v = torch.arange(w, dtype=torch.int64) - w / 2
        if normalize_pos:
            v = v / w * 2 * 3.1415
        e = v[:, None] / inv_freq[None, :]
        tab[a, :w] = torch.stack([e[:, ::2].sin(), e[:, 1::2].cos()], dim=-1).flatten(1)
    return tab, ndim, maxw, Lp


@MIDDLE_ENCODERS.register_module()
class SSTInputLayerV2(nn.Module):
    """models/middle_encoders/sst_input_layer_v2.py:41-331."""

    def __init__(self, drop_info, window_shape, sparse_shape, shuffle_voxels=True, debug=True, normalize_pos=False,
                 pos_temperature=10000, mute=False):
        super().__init__()
        self.fp16_enabled = False
        self.meta_drop_info = drop_info
        self.sparse_shape = sparse_shape
        self.shuffle_voxels = shuffle_voxels
        self.debug = debug
        self.window_shape = window_shape
        self.normalize_pos = normalize_pos
        self.pos_temperature = pos_temperature
        self.mute = mute
        self._pos_cache = {}

    def set_drop_info(self):
        if hasattr(self, "drop_info"):
            return
        meta = self.meta_drop_info
        if isinstance(meta, tuple):
            self.drop_info = meta[0] if self.training else meta[1]
        else:
            self.drop_info = meta
        if not self.mute:
            print(f"drop_info is set to {self.drop_info}, in input_layer")

    def _may_drop(self):
        """True if some window could hold more tokens than its level keeps (host check, no device work)."""
        w3 = ops._window_shape3(self.window_shape, self.sparse_shape)
        cap = min(w3[0], self.sparse_shape[0]) * min(w3[1], self.sparse_shape[1]) * min(w3[2], self.sparse_shape[2])
        for dl in self.drop_info:
            lo, hi = self.drop_info[dl]["drop_range"]
            if min(hi - 1, cap) > self.drop_info[dl]["max_tokens"] and min(hi - 1, cap) >= lo:
                return True
        return False

    def _pos(self, feat_dim, device):
        key = (feat_dim, str(device))
        if key not in self._pos_cache:
            tab, ndim, maxw, Lp = _pos_table(self.window_shape, feat_dim, self.pos_temperature, self.normalize_pos)
            self._pos_cache[key] = (tab.to(device).contiguous(), ndim, maxw, Lp)
        return self._pos_cache[key]

    @torch.no_grad()
    def _plans(self, voxel_coors, batch_size):
        """Both shifts' plans + keep indices (drop phase follows sst_input_layer_v2.py:152-226)."""
        n = voxel_coors.shape[0]
        dev = voxel_coors.device
        args = (self.sparse_shape, self.window_shape, self.drop_info)
        if not self._may_drop():
            p0 = ops.window_plan(voxel_coors, *args, False, batch_size)
            p1 = ops.window_plan(voxel_coors, *args, True, batch_size)
            return p0, p1, None
        mt = torch.zeros(max(self.drop_info.keys()) + 1, dtype=torch.int64, device=dev)
        for dl in self.drop_info:
            mt[dl] = self.drop_info[dl]["max_tokens"]
        keep_inds = torch.arange(n, device=dev)
        d0 = ops.window_plan(voxel_coors, *args, False, batch_size)
        k0 = d0.tok_inner.long() < mt[d0.drop_level]
        lvl0, keep_inds = d0.drop_level[k0], keep_inds[k0]
        c1 = voxel_coors[k0].contiguous()
        d1 = ops.window_plan(c1, *args, True, batch_size)
        k1 = d1.tok_inner.long() < mt[d1.drop_level]
        lvl0, keep_inds, lvl1 = lvl0[k1].contiguous(), keep_inds[k1], d1.drop_level[k1].contiguous()
        c2 = c1[k1].contiguous()
        p0 = ops.window_plan(c2, *args, False, batch_size, token_level=lvl0)
        p1 = ops.window_plan(c2, *args, True, batch_size, token_level=lvl1)
        return p0, p1, keep_inds

    def forward(self, voxel_feats, voxel_coors, batch_size=None):
        self.set_drop_info()
        voxel_coors = voxel_coors.long()
        if self.shuffle_voxels:
            shuffle_inds = torch.randperm(len(voxel_feats), device=voxel_feats.device)
            voxel_feats = voxel_feats[shuffle_inds]
            voxel_coors = voxel_coors[shuffle_inds]
        voxel_coors = voxel_coors.contiguous()
        if batch_size is None:
            batch_size = int(voxel_coors[:, 0].max()) + 1 if len(voxel_coors) else 1
        p0, p1, keep = self._plans(voxel_coors, batch_size)
        if keep is not None:
            voxel_feats = voxel_feats[keep]
            voxel_coors = voxel_coors[keep]
        info = {"voxel_feats": voxel_feats, "voxel_coors": voxel_coors,
                "voxel_keep_inds": keep if keep is not None else torch.arange(len(voxel_coors), device=voxel_coors.device)}
        tab, ndim, maxw, Lp = self._pos(voxel_feats.size(1), voxel_feats.device)
        for i, p in enumerate((p0, p1)):
            info[f"batch_win_inds_shift{i}"] = p.batch_win_inds
            info[f"coors_in_win_shift{i}"] = p.coors_in_win
            info[f"voxel_drop_level_shift{i}"] = p.drop_level
            info[f"sra_plan_shift{i}"] = dict(plan=p, pos_table=tab, pos_ndim=ndim, pos_maxw=maxw, pos_L=Lp,
                                              max_tokens=max(v["max_tokens"] for v in self.drop_info.values()))
            f2w = _LazyDict(lambda p=p: self._flat2win_dict(p))
            info[f"flat2win_inds_shift{i}"] = f2w
            info[f"pos_dict_shift{i}"] = _LazyDict(
                lambda p=p, f2w=f2w: self.get_pos_embed(f2w, p.coors_in_win, voxel_feats.size(1), voxel_feats.dtype))
            info[f"key_mask_shift{i}"] = _LazyDict(lambda f2w=f2w: self.get_key_padding_mask(f2w))
        if self.shuffle_voxels:
            info["shuffle_inds"] = shuffle_inds
        return info

    def _flat2win_dict(self, p):
        d = {}
        for dl in self.drop_info:
            m = p.drop_level == dl
            if not m.any():
                continue
            d[dl] = (p.flat2win_inds[m], torch.where(m))
        d["voxel_drop_level"] = p.drop_level
        d["batching_info"] = self.drop_info
        return d

    @torch.no_grad()
    def get_pos_embed(self, inds_dict, coors_in_win, feat_dim, dtype):
        """sst_input_layer_v2.py:238-305, reference (padded) layout, from the same table the kernels use."""
        tab, ndim, maxw, Lp = self._pos(feat_dim, coors_in_win.device)
        parts = [tab[a][coors_in_win[:, 2 - a]] for a in range(ndim)]  # axis 0 = x = column 2 of (z,y,x)
        pe = torch.cat(parts, dim=-1).to(dtype)
        gap = feat_dim - pe.size(1)
        if gap > 0:
            pe = torch.cat([pe, pe.new_zeros((pe.size(0), gap))], dim=1)
        return ops.flat2window_v2(pe, inds_dict)

    @torch.no_grad()
    def get_key_padding_mask(self, ind_dict):
        n = len(ind_dict["voxel_drop_level"])
        key_padding = torch.ones((n, 1), dtype=torch.bool, device=ind_dict["voxel_drop_level"].device)
        d = ops.flat2window_v2(key_padding, ind_dict)
        return {k: v.logical_not().squeeze(2) for k, v in d.items()}


# ------------------------------------------------------------------------------------------------
# SRA encoder
# ------------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_recover_bev"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, L.vp])
L.SIGNATURES["sstb200_recover_bev_backward"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, L.vp])


class _SraLayer(C.Structure):
    _fields_ = ([("d_model", C.c_int32), ("nhead", C.c_int32), ("dim_ff", C.c_int32), ("act", C.c_int32),
                 ("post_norm", C.c_int32), ("norm_eps", C.c_float)] +
                [(k, C.c_void_p) for k in ("in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "lin1_w", "lin1_b",
                                           "lin2_w", "lin2_b", "norm1_w", "norm1_b", "norm2_w", "norm2_b",
                                           "norm1_mean", "norm1_var", "norm2_mean", "norm2_var", "tau")] +
                [("tau_n", C.c_int32), ("tau_min", C.c_float)] +
                [(k, C.c_void_p) for k in ("in_proj_w_f16", "out_proj_w_f16", "lin1_w_f16", "lin2_w_f16")])


class _SraPlan(C.Structure):
    _fields_ = ([(k, C.c_void_p) for k in ("win_offsets", "tok_perm", "tok_win", "pos_code", "num_windows_dev",
                                           "pos_table")] +
                [("pos_L", C.c_int32), ("pos_maxw", C.c_int32), ("pos_ndim", C.c_int32),
                 ("max_window_tokens", C.c_int32), ("tok_slot", C.c_void_p), ("win_batch", C.c_void_p)])


L.SIGNATURES["sstb200_sra_layer_forward"] = (C.c_int, [L.vp, C.POINTER(_SraLayer), C.POINTER(_SraPlan), L.vp, L.vp,
                                                       C.c_int, L.vp, C.c_int])

L.SIGNATURES["sstb200_sra_stack_forward"] = (C.c_int, [L.vp, C.POINTER(_SraLayer), C.c_int, C.POINTER(_SraPlan),
                                                       C.POINTER(_SraPlan), L.vp, L.vp, L.vp, C.c_int, L.vp, C.c_int])

PRECISIONS = {"fp32": 0, "bf16": 1}


def make_sra_plan(sp):
    p = sp["plan"]
    return _SraPlan(p.win_offsets.data_ptr(), p.tok_perm.data_ptr(), p.tok_win.data_ptr(), p.pos_code.data_ptr(),
                    p.counters.data_ptr(), sp["pos_table"].data_ptr(), sp["pos_L"], sp["pos_maxw"], sp["pos_ndim"],
                    int(sp.get("max_tokens", 0) or 0), p.tok_slot.data_ptr(), p.win_batch.data_ptr())


class WindowAttention(nn.Module):
    """models/sst/sst_basic_block_v2.py:14-75.  `self_attn` is a parameter container with nn.MultiheadAttention's
    names/init (in_proj_weight, in_proj_bias, out_proj.{weight,bias}[, tau]); its torch forward is never called."""

    def __init__(self, d_model, nhead, dropout, batch_first=False, layer_id=None, layer_cfg=dict()):
        super().__init__()
        self.nhead = nhead
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.cosine = bool(layer_cfg.get("cosine", False))
        self.tau_min = layer_cfg.get("tau_min", 0.01)
        if self.cosine:  # models/sst/cosine_msa.py:459-465
            shape = (1, nhead, 1, 1) if layer_cfg.get("non_shared_tau", False) else (1, 1, 1)
            self.self_attn.tau = nn.Parameter(torch.ones(*shape))
        if layer_cfg.get("linear", False):
            raise NotImplementedError
        self.layer_id = layer_id


class EncoderLayer(nn.Module):
    """models/sst/sst_basic_block_v2.py:77-126."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", batch_first=False,
                 layer_id=None, mlp_dropout=0, layer_cfg=dict()):
        super().__init__()
        assert not batch_first
        # the reference applies nn.Dropout(mlp_dropout) three times and attention dropout inside nn.MultiheadAttention
        # (sst_basic_block_v2.py:85-98): identity in eval; a non-zero rate in training is refused, not silently ignored
        self.dropout_p, self.mlp_dropout_p = float(dropout), float(mlp_dropout)
        self.win_attn = WindowAttention(d_model, nhead, dropout, layer_id=layer_id, layer_cfg=layer_cfg)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.use_bn = layer_cfg.get("use_bn", False)
        if self.use_bn:
            self.norm1 = ops.build_norm_layer(dict(type="naiveSyncBN1d", momentum=layer_cfg.get("mom", 0.1)), d_model)[1]
            self.norm2 = ops.build_norm_layer(dict(type="naiveSyncBN1d", momentum=layer_cfg.get("mom", 0.1)), d_model)[1]
        else:
            self.norm1 = nn.LayerNorm(d_model)
            self.norm2 = nn.LayerNorm(d_model)
        if activation not in ("relu", "gelu"):
            raise RuntimeError(f"activation should be relu/gelu, not {activation}.")
        self.activation = activation
        self.post_norm = layer_cfg.get("post_norm", True)
        self.fp16_enabled = False
        self.d_model, self.nhead, self.dim_feedforward = d_model, nhead, dim_feedforward
        self._bf16 = None

    def _struct(self, precision):
        sa = self.win_attn.self_attn
        f = lambda t: t.data_ptr()
        bn = self.use_bn
        s = _SraLayer()
        s.d_model, s.nhead, s.dim_ff = self.d_model, self.nhead, self.dim_feedforward
        s.act = 1 if self.activation == "relu" else 2
        s.post_norm = int(bool(self.post_norm))
        s.norm_eps = float(self.norm1.eps)
        s.in_proj_w, s.in_proj_b = f(sa.in_proj_weight), f(sa.in_proj_bias)
        s.out_proj_w, s.out_proj_b = f(sa.out_proj.weight), f(sa.out_proj.bias)
        s.lin1_w, s.lin1_b, s.lin2_w, s.lin2_b = f(self.linear1.weight), f(self.linear1.bias), f(self.linear2.weight), f(self.linear2.bias)
        s.norm1_w, s.norm1_b, s.norm2_w, s.norm2_b = f(self.norm1.weight), f(self.norm1.bias), f(self.norm2.weight), f(self.norm2.bias)
        if bn:
            s.norm1_mean, s.norm1_var = f(self.norm1.running_mean), f(self.norm1.running_var)
            s.norm2_mean, s.norm2_var = f(self.norm2.running_mean), f(self.norm2.running_var)
        if self.win_attn.cosine:
            s.tau, s.tau_n, s.tau_min = f(sa.tau), sa.tau.numel(), float(self.win_attn.tau_min)
        if precision == 1:
            ws = self.half_weights()
            s.in_proj_w_f16, s.out_proj_w_f16, s.lin1_w_f16, s.lin2_w_f16 = [w.data_ptr() for w in ws]
        return s

    def half_weights(self, refresh=False):
        """fp16 copies of the four weight matrices for the tensor-core path, re-cast whenever any of the four parameters
        changed (version counter, storage or device).  Callers that bake the pointers into a CUDA graph (SSTEngine) keep the
        returned tensors alive themselves and call `SSTEngine.refresh_weights()` after an update."""
        sa = self.win_attn.self_attn
        srcs = (sa.in_proj_weight, sa.out_proj.weight, self.linear1.weight, self.linear2.weight)
        key = tuple((w._version, w.data_ptr(), str(w.device)) for w in srcs)
        if refresh or self._bf16 is None or self._bf16[0] != key:
            self._bf16 = (key, [w.detach().to(torch.float16).contiguous() for w in srcs])
        return self._bf16[1]

    def _check_input(self, src):
        if src.dim() != 2 or src.shape[1] != self.d_model:
            raise RuntimeError(f"EncoderLayer expects [n, {self.d_model}] features, got {tuple(src.shape)} "
                               "(the kernels only receive the row count: a width mismatch would read out of bounds)")
        if self.training and (self.dropout_p > 0 or self.mlp_dropout_p > 0):
            raise NotImplementedError("dropout > 0 in training mode is not built (the reference's configs use dropout = 0)")

    def forward(self, src, sra_plan, precision="fp32"):
        """src [n,d] fp32 flat voxel order; sra_plan: voxel_info['sra_plan_shift{i}']."""
        if torch.is_grad_enabled() and (src.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("gradients flow through the stack-level path (SSTv2.forward); a single EncoderLayer call is "
                                      "inference-only - run it under torch.no_grad()")
        ops._need_cuda(src)
        self._check_input(src)
        src = src.float().contiguous()
        out = torch.empty_like(src)
        prec = PRECISIONS[precision]
        c = L.ctx(src.device)
        ls, ps = self._struct(prec), make_sra_plan(sra_plan)
        L.check(c, L.lib().sstb200_sra_layer_forward(c, C.byref(ls), C.byref(ps), src.data_ptr(), out.data_ptr(),
                                                     src.shape[0], None, prec))
        return out


class BasicShiftBlockV2(nn.Module):
    """models/sst/sst_basic_block_v2.py:129-169."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", batch_first=False,
                 block_id=-100, layer_cfg=dict()):
        super().__init__()
        self.encoder_list = nn.ModuleList([
            EncoderLayer(d_model, nhead, dim_feedforward, dropout, activation, batch_first, layer_id=block_id * 2 + i,
                         layer_cfg=layer_cfg) for i in range(2)])

    def forward(self, src, plan_list, precision="fp32"):
        num_shifts = len(plan_list)
        assert num_shifts in (1, 2)
        out = src
        for i in range(2):
            out = self.encoder_list[i](out, plan_list[i % num_shifts], precision)
        return out


@BACKBONES.register_module()
class SSTv2(nn.Module):
    """models/backbones/sst_v2.py:16-196."""

    def __init__(self, d_model=[], nhead=[], num_blocks=6, dim_feedforward=[], dropout=0.0, activation="gelu",
                 output_shape=None, num_attached_conv=2, conv_in_channel=64, conv_out_channel=64,
                 norm_cfg=dict(type="naiveSyncBN2d", eps=1e-3, momentum=0.01), conv_cfg=dict(type="Conv2d", bias=False),
                 debug=True, in_channel=None, to_bev=True, conv_kwargs=dict(kernel_size=3, dilation=2, padding=2, stride=1),
                 checkpoint_blocks=[], layer_cfg=dict(), conv_shortcut=False, precision=None):
        super().__init__()
        self.d_model, self.nhead = d_model, nhead
        self.checkpoint_blocks = checkpoint_blocks
        self.conv_shortcut = conv_shortcut
        self.to_bev = to_bev
        self.precision = precision  # None -> 'bf16' if fp16_enabled else 'fp32'
        self.fp16_enabled = False
        if in_channel is not None:
            self.linear0 = nn.Linear(in_channel, d_model[0])
        self.block_list = nn.ModuleList([
            BasicShiftBlockV2(d_model[i], nhead[i], dim_feedforward[i], dropout, activation, batch_first=False,
                              block_id=i, layer_cfg=layer_cfg) for i in range(num_blocks)])
        self._reset_parameters()
        self.output_shape = output_shape
        self.debug = debug
        self.num_attached_conv = num_attached_conv
        if num_attached_conv > 0:
            # attached dense convs sit on the module boundary but are not part of the hot path (SURVEY.md 8f
            # next-2): parameter-compatible torch/cuDNN layers.
            conv_list = []
            for i in range(num_attached_conv):
                kw = conv_kwargs if isinstance(conv_kwargs, dict) else conv_kwargs[i]
                if i > 0:
                    conv_in_channel = conv_out_channel
                cc = dict(conv_cfg or dict(type="Conv2d"))
                cc.pop("type", None)
                conv = nn.Conv2d(conv_in_channel, conv_out_channel, **kw, **cc)
                if norm_cfg is None:
                    conv_list.append(nn.Sequential(conv, nn.ReLU(inplace=True)))
                else:
                    conv_list.append(nn.Sequential(conv, ops.build_norm_layer(norm_cfg, conv_out_channel)[1],
                                                   nn.ReLU(inplace=True)))
            self.conv_layer = nn.ModuleList(conv_list)

    def _reset_parameters(self):
        for name, p in self.named_parameters():
            if p.dim() > 1 and "scaler" not in name and "tau" not in name:
                nn.init.xavier_uniform_(p)

    def forward(self, voxel_info):
        assert voxel_info["voxel_coors"].dtype == torch.int64, "data type of coors should be torch.int64!"
        if "sra_plan_shift0" not in voxel_info:
            raise L.SSTB200Error("voxel_info lacks 'sra_plan_shift{0,1}': build it with sst_b200's SSTInputLayerV2")
        plans = [voxel_info[f"sra_plan_shift{i}"] for i in range(2)]
        precision = self.precision or ("bf16" if self.fp16_enabled else "fp32")
        out = voxel_info["voxel_feats"]
        if hasattr(self, "linear0"):
            out = ops.linear(out, self.linear0.weight, self.linear0.bias)
        out = self._run_stack(out, plans, precision)
        if self.to_bev:
            batch_size = int(voxel_info["voxel_coors"][:, 0].max()) + 1
            out = self.recover_bev(out, voxel_info["voxel_coors"], batch_size)
        if self.num_attached_conv > 0:
            assert self.to_bev
            for conv in self.conv_layer:
                temp = conv(out)
                out = temp + out if (temp.shape == out.shape and self.conv_shortcut) else temp
        if not self.to_bev:
            out = {"voxel_feats": out, "voxel_coors": voxel_info["voxel_coors"]}
        return [out]

    def _run_stack(self, x, plans, precision):
        """All encoder layers through ONE C call (sstb200_sra_stack_forward): with precision 'bf16' and the SST-6 shape this
        is 2 launches per layer (window attention + fused wgmma / TMA chain incl. the next layer's QKV)."""
        layers = [l for blk in self.block_list for l in blk.encoder_list]
        if not layers:
            return x
        ops._need_cuda(x)
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for l in layers for p in l.parameters()))
        if needs_grad and not self.training and x.requires_grad:
            raise NotImplementedError("gradients w.r.t. the input in eval() mode are not built: call .train() (the eval-mode forward runs "
                                      "the inference kernels, which keep no activations)")
        if needs_grad and self.training:
            # training step: forward that keeps the activations + hand-written backward (csrc/sra_train.cu), bf16 operands
            from .train import SraStackFunction, layer_params
            for l in layers:
                l._check_input(x)
            if precision != "bf16":
                raise NotImplementedError("the training path runs with precision='bf16' (bf16 GEMM operands, fp32 accumulation / "
                                          "LayerNorm / gradients) - set SSTv2(precision='bf16') or fp16_enabled")
            flat = [p for l in layers for p in layer_params(l)]
            return SraStackFunction.apply(x, layers, plans, make_sra_plan, *flat)
        if len({l.d_model for l in layers}) != 1:
            raise NotImplementedError("per-block d_model lists with different widths are not built (the reference's configs use one width)")
        for l in layers:
            l._check_input(x)
        x = x.float().contiguous()
        prec = PRECISIONS[precision]
        arr = (_SraLayer * len(layers))(*[l._struct(prec) for l in layers])
        y, tmp = torch.empty_like(x), torch.empty_like(x)
        p0, p1 = make_sra_plan(plans[0]), make_sra_plan(plans[1])
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_sra_stack_forward(c, arr, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(),
                                                     tmp.data_ptr(), x.shape[0], None, prec))
        return y

    def recover_bev(self, voxel_feat, coors, batch_size):
        """models/backbones/sst_v2.py:161-196: sparse rows -> dense [B, C, ny, nx] canvas in one HBM-write-bound pass
        (csrc/bev.cu; the canvas is written exactly once, zeros included).  With a gradient to propagate, the canvas gradient
        is gathered back to the rows by sstb200_recover_bev_backward."""
        ny, nx = self.output_shape
        ops._need_cuda(voxel_feat, coors)
        coors = coors.long().contiguous()
        if torch.is_grad_enabled() and voxel_feat.requires_grad:
            return _RecoverBevFunction.apply(voxel_feat.float(), coors, batch_size, ny, nx)
        return _recover_bev(voxel_feat.float().contiguous(), coors, batch_size, ny, nx)


def _recover_bev(voxel_feat, coors, batch_size, ny, nx):
    M, C_ = voxel_feat.shape
    canvas = torch.empty((batch_size, C_, ny, nx), dtype=torch.float32, device=voxel_feat.device)
    c = L.ctx(voxel_feat.device)
    L.check(c, L.lib().sstb200_recover_bev(c, voxel_feat.data_ptr(), coors.data_ptr(), M, C_, batch_size, ny, nx,
                                           canvas.data_ptr()))
    return canvas


class _RecoverBevFunction(torch.autograd.Function):
    """recover_bev with its backward: d voxel_feat[m] = d canvas[b_m, :, y_m, x_m] for every row (rows sharing a cell each
    receive that cell's gradient, like the reference's index_put).  Saves only the coordinates and the canvas shape."""

    @staticmethod
    def forward(ctx, voxel_feat, coors, batch_size, ny, nx):
        ctx.save_for_backward(coors)
        ctx.shape = (voxel_feat.shape[0], voxel_feat.shape[1], batch_size, ny, nx)
        return _recover_bev(voxel_feat.contiguous(), coors, batch_size, ny, nx)

    @staticmethod
    def backward(ctx, grad_canvas):
        (coors,) = ctx.saved_tensors
        M, C_, B, ny, nx = ctx.shape
        g = grad_canvas.float().contiguous()
        grad = torch.empty((M, C_), dtype=torch.float32, device=g.device)
        c = L.ctx(g.device)
        L.check(c, L.lib().sstb200_recover_bev_backward(c, g.data_ptr(), coors.data_ptr(), M, C_, B, ny, nx, grad.data_ptr()))
        return grad, None, None, None, None


# ------------------------------------------------------------------------------------------------
# v1 names (configs/sst/*.py): SSTInputLayer + SSTv1.  Same maths as v2 (models/middle_encoders/sst_input_layer.py:14-364,
# models/backbones/sst_v1.py:17-270, models/sst/sst_basic_block.py:13-140): 2-D windows given as (num_x, num_y), the shift
# written as an explicit (shift_x, shift_y) list, the positional embedding computed inside the backbone, and a TUPLE
# (voxel_feat, flat2win_inds_list, voxel_info) handed from the input layer to the backbone.  Both classes drive the same
# window-plan / SRA kernels as their v2 counterparts.
# ------------------------------------------------------------------------------------------------
@MIDDLE_ENCODERS.register_module()
class SSTInputLayer(nn.Module):
    """models/middle_encoders/sst_input_layer.py:14-364.  `forward` also accepts the `batch_size` third argument that
    DynamicVoxelNet.extract_feat passes (detectors/dynamic_voxelnet.py:43; the reference's v1 signature rejects it)."""

    def __init__(self, drop_info, shifts_list, window_shape, point_cloud_range, voxel_size, shuffle_voxels=True, debug=True):
        super().__init__()
        self.fp16_enabled = False
        self.meta_drop_info = drop_info
        self.shifts_list = shifts_list
        self.point_cloud_range = point_cloud_range
        self.voxel_size = voxel_size
        self.shuffle_voxels = shuffle_voxels
        self.debug = debug
        self.window_shape = window_shape
        wx, wy = window_shape
        for i, (sx, sy) in enumerate(shifts_list):
            if (sx, sy) != ((0, 0) if i == 0 else (wx // 2, wy // 2)) or i > 1:
                raise NotImplementedError(f"shifts_list {shifts_list}: only [(0, 0), (win_x // 2, win_y // 2)] (the reference's own "
                                          "assertion, sst_input_layer.py:312) is built")
        if len(shifts_list) > 1 and (wx % 2 or wy % 2):
            raise NotImplementedError("odd window sizes shift by win - win // 2 in v1 (sst_input_layer.py:313): not built")
        import math
        bev_x = int(math.ceil((point_cloud_range[3] - point_cloud_range[0]) / voxel_size[0]))
        bev_y = int(math.ceil((point_cloud_range[4] - point_cloud_range[1]) / voxel_size[1]))
        self._bev = (bev_x, bev_y)
        # the shared machinery: v2 layer over the same grid (z collapsed), never shuffling by itself
        self._v2 = SSTInputLayerV2(drop_info, (wx, wy, 1), (bev_x, bev_y, 1), shuffle_voxels=False, debug=debug, mute=True)

    def set_drop_info(self):
        if hasattr(self, "drop_info"):
            return
        self._v2.train(self.training)
        self._v2.set_drop_info()
        self.drop_info = self._v2.drop_info
        print(f"drop_info is set to {self.drop_info}, in input_layer")

    def window_partition(self, coors, voxel_info):
        """sst_input_layer.py:298-330 (API parity: the v1 window ids / in-window coordinates, elementwise)."""
        wx, wy = self.window_shape
        bev_x, bev_y = self._bev
        ny_win = -(-bev_y // wy) + 1
        per_sample = (-(-bev_x // wx) + 1) * ny_win
        for i, (sx, sy) in enumerate(self.shifts_list):
            x = coors[:, 3] + (wx - sx if sx > 0 else 0)
            y = coors[:, 2] + (wy - sy if sy > 0 else 0)
            voxel_info[f"batch_win_inds_shift{i}"] = coors[:, 0] * per_sample + (x // wx) * ny_win + y // wy
            voxel_info[f"coors_in_win_shift{i}"] = torch.stack([x % wx, y % wy], dim=-1)
        return voxel_info

    def forward(self, voxel_feat, coors, batch_size=None):
        self.set_drop_info()
        coors = coors.long()
        if self.shuffle_voxels:
            shuffle_inds = torch.randperm(len(voxel_feat), device=voxel_feat.device)
            voxel_feat, coors = voxel_feat[shuffle_inds], coors[shuffle_inds]
        coors = coors.contiguous()
        if batch_size is None:
            batch_size = int(coors[:, 0].max()) + 1 if len(coors) else 1
        plans = self._v2._plans(coors, batch_size)
        num_shifts = len(self.shifts_list)
        p0, p1, keep = plans
        if keep is not None:
            voxel_feat, coors = voxel_feat[keep], coors[keep]
        voxel_info = {"coors": coors,
                      "voxel_keep_inds": keep if keep is not None else torch.arange(len(coors), device=coors.device)}
        self.window_partition(coors, voxel_info)
        tab, ndim, maxw, Lp = self._v2._pos(voxel_feat.size(1), voxel_feat.device)
        flat2win = []
        for i, p in enumerate((p0, p1)[:num_shifts]):
            voxel_info[f"voxel_drop_level_shift{i}"] = p.drop_level
            voxel_info[f"sra_plan_shift{i}"] = dict(plan=p, pos_table=tab, pos_ndim=ndim, pos_maxw=maxw, pos_L=Lp,
                                                    max_tokens=max(v["max_tokens"] for v in self.drop_info.values()))
            flat2win.append(_LazyDict(lambda p=p: {k: v for k, v in self._v2._flat2win_dict(p).items() if not isinstance(k, str)}))
        if self.shuffle_voxels:
            voxel_info["shuffle_inds"] = shuffle_inds
        return voxel_feat, flat2win, voxel_info


@BACKBONES.register_module()
class SSTv1(SSTv2):
    """models/backbones/sst_v1.py:17-270: v1 constructor / forward(input_tuple) on the v2 kernels."""

    def __init__(self, d_model=[], nhead=[], num_blocks=6, dim_feedforward=[], dropout=0.0, activation="gelu", output_shape=None,
                 num_attached_conv=2, conv_in_channel=64, conv_out_channel=64,
                 norm_cfg=dict(type="naiveSyncBN2d", eps=1e-3, momentum=0.01), conv_cfg=dict(type="Conv2d", bias=False), debug=True,
                 drop_info=None, normalize_pos=False, pos_temperature=10000, window_shape=None, in_channel=None,
                 conv_kwargs=dict(kernel_size=3, dilation=2, padding=2, stride=1), checkpoint_blocks=[], precision=None):
        assert drop_info is not None
        super().__init__(d_model=d_model, nhead=nhead, num_blocks=num_blocks, dim_feedforward=dim_feedforward, dropout=dropout,
                         activation=activation, output_shape=output_shape, num_attached_conv=num_attached_conv,
                         conv_in_channel=conv_in_channel, conv_out_channel=conv_out_channel, norm_cfg=norm_cfg, conv_cfg=conv_cfg,
                         debug=debug, in_channel=in_channel, to_bev=True, conv_kwargs=conv_kwargs, checkpoint_blocks=checkpoint_blocks,
                         precision=precision)
        self.meta_drop_info = drop_info
        self.pos_temperature = pos_temperature
        self.window_shape = window_shape
        self.normalize_pos = normalize_pos

    def set_drop_info(self):
        if hasattr(self, "drop_info"):
            return
        meta = self.meta_drop_info
        self.drop_info = (meta[0] if self.training else meta[1]) if isinstance(meta, tuple) else meta
        print(f"drop_info is set to {self.drop_info}, in backbone")

    def forward(self, input_tuple):
        voxel_feat, ind_dict_list, voxel_info = input_tuple
        assert voxel_info["coors"].dtype == torch.int64, "data type of coors should be torch.int64!"
        self.set_drop_info()
        if "sra_plan_shift0" not in voxel_info:
            raise L.SSTB200Error("voxel_info lacks 'sra_plan_shift0': build it with sst_b200's SSTInputLayer")
        plans = [voxel_info[f"sra_plan_shift{i}"] for i in range(len(ind_dict_list))]
        for sp in plans:   # the positional table belongs to the backbone in v1 (pos_temperature / normalize_pos are ITS kwargs)
            tab, ndim, maxw, Lp = _pos_table(tuple(self.window_shape) + (1,), self.d_model[0], self.pos_temperature, self.normalize_pos)
            sp.update(pos_table=tab.to(voxel_feat.device).contiguous(), pos_ndim=ndim, pos_maxw=maxw, pos_L=Lp)
        if len(plans) == 1:
            plans = plans * 2
        precision = self.precision or ("bf16" if self.fp16_enabled else "fp32")
        out = voxel_feat
        if hasattr(self, "linear0"):
            out = ops.linear(out, self.linear0.weight, self.linear0.bias)
        out = self._run_stack(out, plans, precision)
        batch_size = int(voxel_info["coors"][:, 0].max()) + 1
        out = self.recover_bev(out, voxel_info["coors"], batch_size)
        if self.num_attached_conv > 0:
            for conv in self.conv_layer:
                out = conv(out)
        return [out]


@BACKBONES.register_module()
class SST(nn.Module):
    """models/backbones/sst.py: registered in the reference but dead code ("Do not use this file", sst.py:1; it needs the
    undefined SRATensor, sst.py:142, and no config names it).  The name resolves; constructing it says why it cannot run."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        raise NotImplementedError("SST (models/backbones/sst.py) is dead code in the reference - use SSTv1 / SSTv2")
