"""Ragged window attention pinned to a float64 oracle on a window layout chosen to hit every key-chunk, key-tile and window-batch
edge of the four attention kernels:

    win_attn_batch_kernel       csrc/sra_attn.cuh   tensor cores, batches of whole windows, keys in chunks of <= 64
    win_attn_kernel<float>      csrc/sra_attn.cuh   SIMT online softmax, fp32 layers (head dims 8 / 16 / 32 / 64)
    win_attn_kernel<__half>     csrc/sra_bf16.cu    the same SIMT kernel on fp16 q|k|v, bf16 layers the tensor-core kernel refuses
    win_attn_bwd_kernel         csrc/sra_train.cu   training backward

The windows are built so that, for one shift, their token counts in window-id (CSR) order are exactly the list of
`engineered_sizes()`; every GPU test reads back the plan it ran and asserts that layout before it compares anything.  Errors are
also accounted per window-size group, so that a fault confined to, say, the third key chunk of 129..144-token windows cannot hide
in a max-norm over the whole frame."""
import pytest
import torch

from oracle import sst_oracle as O

# csrc/common.cuh:141-146: window batch b holds the windows whose first slot lies in [b * ATT_CHUNK, (b + 1) * ATT_CHUNK); the
# tensor-core kernels take windows of at most ATT_MAXT tokens
ATT_CHUNK, ATT_MAXT = 112, 144
SPARSE = (468, 468, 1)
WIN = (12, 12, 1)
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
DROP_TRAIN = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
              2: {'max_tokens': 100, 'drop_range': (60, 100000)}}
# window sizes at which the tensor-core kernel changes chunk (64 keys), chunk width (rem > 48 / 32 / 16) or masked key tile (8)
EDGES = (16, 17, 32, 33, 48, 49, 56, 57, 63, 64, 65, 80, 81, 112, 113, 120, 121, 128, 129, 144)
GROUPS = ((1, 1), (2, 16), (17, 32), (33, 48), (49, 64), (65, 112), (113, 128), (129, 144))
GROUP_FACTOR = 3.0   # no window-size group's mean error may exceed this multiple of the mean over the other tokens
BF16_REL, FP32_REL, GRAD_REL, TAU_REL = 1e-2, 1e-3, 2e-2, 3e-2
FP32_TIGHT = 5e-6   # see test_simt_fp32_layer


# ------------------------------------------------------------------------------------------------------------------------------
# the engineered layout
# ------------------------------------------------------------------------------------------------------------------------------
def engineered_sizes():
    """Token counts of the windows in CSR order: every size 1..144; every EDGES size once at offset 0 and once at offset 111 of a
    window batch (a 129..144-token window at 111 covers the whole next batch, whose record is then empty: wb == we); a batch that
    stages 111 + 144 = 255 rows; a batch in which 112 one-token windows start (four passes of the kernel's 32-window q-tile table); a last batch that is partly filled."""
    g = torch.Generator().manual_seed(7)
    fill = iter(torch.randint(1, ATT_MAXT + 1, (100000,), generator=g).tolist())
    sizes, pos = [], [0]

    def add(s):
        sizes.append(int(s))
        pos[0] += int(s)

    def goto(off):   # filler windows up to offset `off` of the current (or next) batch
        t = pos[0] // ATT_CHUNK * ATT_CHUNK + off
        if t < pos[0]:
            t += ATT_CHUNK
        while pos[0] < t:
            add(min(next(fill), t - pos[0]))

    for s in (torch.randperm(ATT_MAXT, generator=g) + 1).tolist():
        add(s)
    for e in EDGES:
        goto(0)
        add(e)
        goto(ATT_CHUNK - 1)
        add(e)
    goto(0)   # the fullest batch: 111 + 144 = 255 staged rows
    add(ATT_CHUNK - 1)
    add(ATT_MAXT)
    goto(0)
    for _ in range(ATT_CHUNK):
        add(1)
    add(45)
    return sizes


def _sample_split(sizes):
    """Index of the first window of sample 1: near the middle, where the sample boundary falls inside a window batch."""
    k = len(sizes) // 2
    while sum(sizes[:k]) % ATT_CHUNK in (0, ATT_CHUNK - 1):
        k += 1
    return k


def engineered_coors(sizes, shift, window=12, seed=0):
    """(b, 0, y, x) rows on the 468 x 468 grid whose `window` x `window` windows at `shift` (0 or 1) hold exactly `sizes` tokens in
    CSR (window-id) order, over two samples.  Each window's cells are drawn at random inside it and the rows are shuffled, so that
    positional embeddings vary and flat token order differs from window order."""
    g = torch.Generator().manual_seed(seed)
    off = 0 if shift == 0 else window // 2          # x -> window (x + window - off) // window: shift 0 adds window, shift 1 half
    per = (SPARSE[0] - off) // window               # whole windows per axis inside the grid
    split = _sample_split(sizes)
    rows = []
    for b, part in ((0, sizes[:split]), (1, sizes[split:])):
        assert len(part) <= per * per
        for i, s in enumerate(part):
            x0, y0 = off + window * (i // per), off + window * (i % per)   # window-id order: x window major, then y
            cells = torch.randperm(window * window, generator=g)[:s]
            rows.append(torch.stack([torch.full((s,), b), torch.zeros(s, dtype=torch.long), y0 + cells // window,
                                     x0 + cells % window], 1))
    coors = torch.cat(rows)
    return coors[torch.randperm(coors.shape[0], generator=g)].int()


def batch_records(sizes):
    """{first window, end window, first slot, end slot} of every window batch, as win_batch_kernel (csrc/window.cu) writes them."""
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    starts = torch.tensor(offs[:-1])
    nb = (offs[-1] + ATT_CHUNK - 1) // ATT_CHUNK
    recs = []
    for b in range(nb):
        wb, we = (int(torch.searchsorted(starts, t)) for t in (b * ATT_CHUNK, (b + 1) * ATT_CHUNK))
        recs.append((wb, we, offs[wb], offs[we]))
    return recs


def check_engineered(sizes, recs):
    """The layout covers what the tests claim to cover; `recs` are the batch records of the plan that ran (or the oracle's)."""
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    n = offs[-1]
    assert 15000 <= n <= 25000, n
    assert set(range(1, ATT_MAXT + 1)) <= set(sizes), "a window size in 1..144 is missing"
    placed = {(s, o % ATT_CHUNK) for s, o in zip(sizes, offs)}
    missing = [(e, o) for e in EDGES for o in (0, ATT_CHUNK - 1) if (e, o) not in placed]
    assert not missing, f"edge windows (size, batch offset) missing: {missing}"
    assert max(sizes) <= ATT_MAXT
    assert len(recs) == (n + ATT_CHUNK - 1) // ATT_CHUNK
    empty = [b for b, r in enumerate(recs) if r[0] == r[1]]
    assert any(sizes[recs[b - 1][1] - 1] == ATT_MAXT and offs[recs[b - 1][1] - 1] % ATT_CHUNK == ATT_CHUNK - 1 for b in empty), \
        "no wb == we record behind a 144-token window at batch offset 111"
    assert max(r[1] - r[0] for r in recs) > 32, "no batch with more than 32 windows"
    assert max(r[3] - r[2] for r in recs) == ATT_CHUNK - 1 + ATT_MAXT, "no batch staging the most rows a batch can hold"
    assert 0 < n % ATT_CHUNK < ATT_CHUNK - 16, "the last batch is not partly filled"
    assert offs[_sample_split(sizes)] % ATT_CHUNK != 0


def test_engineered_layout_oracle():
    """CPU: the coordinates give the engineered window sizes, in CSR order, under the oracle's window partition - for shift 0 and
    for the shifted grid of shift 1."""
    sizes = engineered_sizes()
    check_engineered(sizes, batch_records(sizes))
    for shift in (0, 1):
        coors = engineered_coors(sizes, shift).long()
        assert torch.unique(coors, dim=0).shape[0] == coors.shape[0], "duplicate voxels"
        assert 0 <= coors[:, 2:].min() and coors[:, 2:].max() < SPARSE[0]
        win, _ = O.get_window_coors(coors, SPARSE, WIN, shift == 1)
        counts = torch.unique(win, sorted=True, return_counts=True)[1]   # window-id order == CSR order of the plan
        assert counts.tolist() == sizes, shift
        assert not torch.equal(win, win.sort().values), "rows are not shuffled"
        assert (coors[:, 0] == 0).sum() == sum(sizes[:_sample_split(sizes)])
    big = big_window_sizes()
    coors = engineered_coors(big, 0, window=16).long()
    win, _ = O.get_window_coors(coors, SPARSE, (16, 16, 1), False)
    assert torch.unique(win, sorted=True, return_counts=True)[1].tolist() == big


def big_window_sizes():
    """16 x 16 windows for the SIMT fallback beyond ATT_MAXT: 145..256 tokens, and some small ones around them."""
    g = torch.Generator().manual_seed(11)
    big = list(range(145, 257, 3)) + [256]
    small = torch.randint(1, 100, (len(big),), generator=g).tolist()
    return [s for pair in zip(big, small) for s in pair]


# ------------------------------------------------------------------------------------------------------------------------------
# plan read-back, models, float64 oracle, error accounting
# ------------------------------------------------------------------------------------------------------------------------------
def plan_layout(info, shift):
    """(window sizes in CSR order, batch records, per-token window size in flat order) of the plan the kernels ran."""
    p = info[f"sra_plan_shift{shift}"]["plan"]
    cnt = p.counters.cpu()
    R, nb = int(cnt[0]), int(cnt[17])
    offs = p.win_offsets[:R + 1].cpu().long()
    sizes = (offs[1:] - offs[:-1]).tolist()
    recs = [tuple(r) for r in p.win_batch[:4 * nb].cpu().view(nb, 4).tolist()]
    tok_size = torch.tensor(sizes)[p.tok_win.cpu().long()]
    return sizes, recs, tok_size


def assert_engineered_plan(info, shift, sizes):
    got, recs, tok_size = plan_layout(info, shift)
    assert got == sizes, "the window planner no longer produces the engineered layout"
    assert recs == batch_records(sizes), "window batch records differ from the engineered layout's"
    check_engineered(got, recs)
    return tok_size


def _model(d, h, ff, blocks, lc=None, taus=None, seed=0):
    """SSTv2 with non-trivial norms and biases (as test_gpu_sst.py's _sst_pair sets them); taus(layer, tau) -> new tau."""
    from sst_b200.sst_modules import SSTv2
    torch.manual_seed(seed)
    m = SSTv2(d_model=[d] * blocks, nhead=[h] * blocks, num_blocks=blocks, dim_feedforward=[ff] * blocks, output_shape=[468, 468],
              num_attached_conv=0, to_bev=False, layer_cfg=lc or {}).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        li = 0
        for n_, p in m.named_parameters():
            if n_.endswith("tau"):
                p.copy_(taus(li, p) if taus else torch.rand(p.shape, generator=g) * 0.5 + 0.05)
                li += 1
            elif p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
    return m


def _head_rows(m, part, head, fn):
    """Apply fn to the in_proj rows (and bias) of q (part 0) or k (part 1) of `head` in every layer."""
    with torch.no_grad():
        for blk in m.block_list:
            for layer in blk.encoder_list:
                sa = layer.win_attn.self_attn
                d, dh = layer.d_model, layer.d_model // layer.nhead
                r = slice(part * d + head * dh, part * d + (head + 1) * dh)
                sa.in_proj_weight[r] = fn(sa.in_proj_weight[r])
                sa.in_proj_bias[r] = fn(sa.in_proj_bias[r])


def _sharpen(m, f=3.0):
    """q and k rows of in_proj_weight x f: logits x f^2, so that they span tens of units and the running max moves between chunks."""
    with torch.no_grad():
        for blk in m.block_list:
            for layer in blk.encoder_list:
                layer.win_attn.self_attn.in_proj_weight[:2 * layer.d_model] *= f


def _inputs(coors, d, seed=3):
    return torch.randn(coors.shape[0], d, generator=torch.Generator().manual_seed(seed))


def _gpu_info(cuda, feats, coors, drop=DROP_TEST, window=WIN, train=False):
    from sst_b200.sst_modules import SSTInputLayerV2
    il = SSTInputLayerV2(drop, window, SPARSE, shuffle_voxels=False, mute=True).train(train)
    return il(feats.to(cuda), coors.to(cuda), 2)


def _oracle64(m, feats, coors, lc, layer=None, drop=DROP_TEST, window=WIN):
    """float64 oracle: the whole stack of `m`, or only encoder layer `layer` = (block, index) on shift `index`."""
    w = {k: v.detach().double() for k, v in m.state_dict().items()}
    info = O.input_layer_v2(feats.double(), coors, drop, window, SPARSE)
    heads = [blk.encoder_list[0].nhead for blk in m.block_list]
    if layer is None:
        return O.sstv2_forward(info, w, heads, len(heads), "gelu", lc)
    b, i = layer
    return O.encoder_layer(info["voxel_feats"], info[f"pos_dict_shift{i}"], info[f"flat2win_inds_shift{i}"], info[f"key_mask_shift{i}"],
                           w, f"block_list.{b}.encoder_list.{i}.", heads[b], "gelu", lc)


def check_grouped(got, ref, tok_size, rel, what, all_groups=True):
    """Element-wise comparison (max-norm and assert_close at `rel` of the reference's max-abs) plus the per-window-size accounting:
    no group's mean error above GROUP_FACTOR x the mean over the tokens outside that group (not over all tokens: a group holding a
    third of them would pull the overall mean up with its own fault), every group's max error under the global bound.
    Returns (max error / scale, mean error / scale, table)."""
    got = got.detach().cpu().double()
    ref = ref.detach().cpu().double()
    assert got.shape == ref.shape and tok_size.shape[0] == got.shape[0]
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    scale = ref.abs().max().item()
    err = (got - ref).abs() / scale
    mean_all = err.mean().item()
    lines, bad = [f"{what}: scale {scale:.4g}, mean {mean_all:.3e}, max {err.max().item():.3e} (bound {rel:g})",
                  "  group        tokens   mean err    max err   mean / mean outside"], []
    for lo, hi in GROUPS:
        m = (tok_size >= lo) & (tok_size <= hi)
        if not m.any():
            lines.append(f"  {lo:>3}..{hi:<3}   {0:>8}")
            if all_groups:
                bad.append(f"no tokens in windows of {lo}..{hi}")
            continue
        e = err[m]
        gm, gx = e.mean().item(), e.max().item()
        mo = err[~m].mean().item() if (~m).any() else gm
        lines.append(f"  {lo:>3}..{hi:<3}   {int(m.sum()):>8}   {gm:.3e}   {gx:.3e}   {gm / max(mo, 1e-300):.2f}")
        if gm > GROUP_FACTOR * mo:
            bad.append(f"group {lo}..{hi}: mean {gm:.3e} > {GROUP_FACTOR} x {mo:.3e} (mean outside the group)")
        if gx >= rel:
            bad.append(f"group {lo}..{hi}: max {gx:.3e} >= {rel:g}")
    table = "\n".join(lines)
    print(table)
    assert not bad, "\n".join(bad) + "\n" + table
    torch.testing.assert_close(got, ref, rtol=rel, atol=rel * scale, msg=lambda m_: f"{what}: {m_}\n{table}")
    return err.max().item(), mean_all, table


# ------------------------------------------------------------------------------------------------------------------------------
# tensor-core attention, inference
# ------------------------------------------------------------------------------------------------------------------------------
def _taus_per_head_one_below(tau_min):
    """tau ~ U[tau_min, tau_min + 0.5] per head, head 3 at tau_min / 2 (clamped)."""
    def taus(li, p):
        t = torch.rand(p.shape, generator=torch.Generator().manual_seed(50 + li)) * 0.5 + tau_min
        t.view(-1)[3] = tau_min / 2
        return t
    return taus


TC_VARIANTS = {
    "plain": ({}, None, False),
    "cosine_one_tau": (dict(cosine=True, tau_min=0.01), None, False),
    "cosine_tau_per_head": (dict(cosine=True, non_shared_tau=True, tau_min=0.05), _taus_per_head_one_below(0.05), False),
    "sharp": ({}, None, True),
}


def _tc_model(variant, blocks):
    lc, taus, sharp = TC_VARIANTS[variant]
    m = _model(128, 8, 256, blocks, lc, taus)
    if sharp:
        _sharpen(m)
    return m, lc


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(TC_VARIANTS))
@pytest.mark.parametrize("shift", [0, 1])
def test_tensor_core_layer(cuda, shift, variant):
    """One bf16 encoder layer (sstb200_sra_layer_forward -> win_attn_batch_kernel) on the layout engineered for its shift."""
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, shift)
    m, lc = _tc_model(variant, 1)
    feats = _inputs(coors, 128)
    ref = _oracle64(m, feats, coors, lc, layer=(0, shift))
    info = _gpu_info(cuda, feats, coors)
    tok_size = assert_engineered_plan(info, shift, sizes)
    layer = m.block_list[0].encoder_list[shift].to(cuda)
    with torch.no_grad():
        got = layer(info["voxel_feats"], info[f"sra_plan_shift{shift}"], "bf16")
    check_grouped(got, ref, tok_size, BF16_REL, f"bf16 layer, shift {shift}, {variant}")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(TC_VARIANTS))
def test_tensor_core_block(cuda, variant):
    """The fused bf16 stack (2 launches per layer) for one block: shift 0 engineered, shift 1 whatever follows from it."""
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, 0)
    m, lc = _tc_model(variant, 1)
    feats = _inputs(coors, 128)
    ref = _oracle64(m, feats, coors, lc)
    info = _gpu_info(cuda, feats, coors)
    tok_size = assert_engineered_plan(info, 0, sizes)
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        got = m(info)[0]["voxel_feats"]
    check_grouped(got, ref, tok_size, BF16_REL, f"bf16 block, {variant}")


# ------------------------------------------------------------------------------------------------------------------------------
# degenerate and scaled heads, through all three forward kernels
# ------------------------------------------------------------------------------------------------------------------------------
DEGENERATE = {
    # q of head 2 = 0: every score 0, uniform softmax
    "zero_q_plain": ({}, lambda m: _head_rows(m, 0, 2, torch.zeros_like)),
    # cosine, q of head 1 = 0 and k of head 3 = 0: F.normalize's 1e-12 clamp
    "zero_qk_cosine": (dict(cosine=True, tau_min=0.01),
                       lambda m: (_head_rows(m, 0, 1, torch.zeros_like), _head_rows(m, 1, 3, torch.zeros_like))),
    # cosine, q of head 0 and k of head 2 x 1e-2 (still normal in fp16): invariant, and catches a clamp larger than 1e-12
    "scaled_cosine": (dict(cosine=True, tau_min=0.01),
                      lambda m: (_head_rows(m, 0, 0, lambda t: t * 1e-2), _head_rows(m, 1, 2, lambda t: t * 1e-2))),
}
DEGENERATE_PATHS = {"tensor_core": (8, "bf16", BF16_REL), "simt_fp32": (8, "fp32", FP32_REL), "simt_fp16": (4, "bf16", BF16_REL)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(DEGENERATE))
@pytest.mark.parametrize("path", list(DEGENERATE_PATHS))
def test_degenerate_heads(cuda, path, case):
    """Zeroed and 1e-2-scaled q / k heads through one layer of each forward kernel (tensor core, SIMT fp32, SIMT on fp16 operands):
    finite, and equal to the float64 oracle; the scaled cosine heads also equal the unscaled model (cosine attention ignores the
    scale of q and k)."""
    h, prec, rel = DEGENERATE_PATHS[path]
    lc, edit = DEGENERATE[case]
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, 0)
    m = _model(128, h, 256, 1, lc)
    edit(m)
    feats = _inputs(coors, 128)
    ref = _oracle64(m, feats, coors, lc, layer=(0, 0))
    info = _gpu_info(cuda, feats, coors)
    tok_size = assert_engineered_plan(info, 0, sizes)
    with torch.no_grad():
        got = m.block_list[0].encoder_list[0].to(cuda)(info["voxel_feats"], info["sra_plan_shift0"], prec)
    check_grouped(got, ref, tok_size, rel, f"{path}, {case}")
    if case == "scaled_cosine":
        base = _model(128, h, 256, 1, lc)
        with torch.no_grad():
            unscaled = base.block_list[0].encoder_list[0].to(cuda)(info["voxel_feats"], info["sra_plan_shift0"], prec)
        check_grouped(got, unscaled, tok_size, rel, f"{path}, {case} vs the unscaled model")


# ------------------------------------------------------------------------------------------------------------------------------
# SIMT kernel: fp32 layers (every head dim) and fp16 operands in bf16 layers
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cosine", [False, True], ids=["plain", "cosine"])
@pytest.mark.parametrize("d,h", [(128, 16), (128, 8), (128, 4), (128, 2), (192, 12)],
                         ids=["dh8", "dh16", "dh32", "dh64", "192x12heads"])
def test_simt_fp32_layer(cuda, d, h, cosine):
    """fp32 layer (win_attn_kernel<float>) at head dims 8, 16, 32, 64 and the 12-head d_model-192 shape of
    configs/sst/sst_waymoD5_1x_3class_12heads.py: within the fp32 contract (1e-3), and within FP32_TIGHT of the float64 oracle.
    Observed on an H100 80GB HBM3 (700 W power limit): at most 1.33e-6 of the output's max-abs over these ten cases (192 x 12 heads,
    cosine), so FP32_TIGHT = 5e-6 leaves a margin of about 4x."""
    lc = dict(cosine=True, non_shared_tau=True, tau_min=0.01) if cosine else {}
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, 0)
    m = _model(d, h, 2 * d, 1, lc)
    feats = _inputs(coors, d)
    ref = _oracle64(m, feats, coors, lc, layer=(0, 0))
    info = _gpu_info(cuda, feats, coors)
    tok_size = assert_engineered_plan(info, 0, sizes)
    with torch.no_grad():
        got = m.block_list[0].encoder_list[0].to(cuda)(info["voxel_feats"], info["sra_plan_shift0"], "fp32")
    err, _, table = check_grouped(got, ref, tok_size, FP32_REL, f"fp32 layer d {d} heads {h} cosine {cosine}")
    assert err < FP32_TIGHT, f"fp32 error {err:.3e} above the tight bound {FP32_TIGHT:g}\n{table}"


@pytest.mark.gpu
@pytest.mark.parametrize("cosine", [False, True], ids=["plain", "cosine"])
@pytest.mark.parametrize("h", [4, 16])
def test_simt_fp16_fallback_block(cuda, h, cosine):
    """bf16 block with 4 or 16 heads: the fused stack refuses it (the tensor-core kernel is built for 8 heads of 16), the stack falls
    back to per-layer calls and each layer runs win_attn_kernel<__half> on fp16 q|k|v.  The fallback is established from the
    tensor-core preconditions: nhead != 8."""
    lc = dict(cosine=True, non_shared_tau=True, tau_min=0.01) if cosine else {}
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, 0)
    m = _model(128, h, 256, 1, lc)
    assert all(l.nhead != 8 for blk in m.block_list for l in blk.encoder_list)
    feats = _inputs(coors, 128)
    ref = _oracle64(m, feats, coors, lc)
    info = _gpu_info(cuda, feats, coors)
    tok_size = assert_engineered_plan(info, 0, sizes)
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        got = m(info)[0]["voxel_feats"]
    check_grouped(got, ref, tok_size, BF16_REL, f"fp16 SIMT block, {h} heads, cosine {cosine}")


@pytest.mark.gpu
def test_simt_fp16_fallback_windows_beyond_att_maxt(cuda):
    """8 heads but 16 x 16 windows with a drop level of max_tokens 256 and windows of 145..256 tokens: the plan's max_tokens (256)
    exceeds ATT_MAXT, which is the tensor-core precondition that fails, so each bf16 layer runs the SIMT kernel on fp16 operands."""
    drop = dict(DROP_TEST)
    drop[3] = {'max_tokens': 256, 'drop_range': (100, 100000)}
    sizes = big_window_sizes()
    coors = engineered_coors(sizes, 0, window=16)
    m = _model(128, 8, 256, 1)
    feats = _inputs(coors, 128)
    ref = _oracle64(m, feats, coors, {}, drop=drop, window=(16, 16, 1))
    info = _gpu_info(cuda, feats, coors, drop=drop, window=(16, 16, 1))
    got_sizes, _, tok_size = plan_layout(info, 0)
    assert got_sizes == sizes and max(got_sizes) == 256
    assert info["sra_plan_shift0"]["max_tokens"] > ATT_MAXT and info["sra_plan_shift1"]["max_tokens"] > ATT_MAXT
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        got = m(info)[0]["voxel_feats"]
    big = tok_size > ATT_MAXT
    assert big.sum() > 5000
    check_grouped(got, ref, tok_size.clamp(max=ATT_MAXT), BF16_REL, "fp16 SIMT block, windows up to 256 tokens", all_groups=False)
    check_grouped(got[big.to(cuda)], ref[big], tok_size[big], BF16_REL, "tokens of windows > 144", all_groups=False)


# ------------------------------------------------------------------------------------------------------------------------------
# training: forward, dX per token, every parameter gradient and d tau against float64 autograd
# ------------------------------------------------------------------------------------------------------------------------------
def _oracle_leaves(m, heads=8):
    """float64 leaf copies of m's state; a shared tau enters as per-head copies, so the oracle yields every head's share."""
    return {k: (v.detach().double().reshape(-1)[:1].expand(1, heads, 1, 1).clone() if k.endswith("tau") and v.numel() == 1
                else v.detach().double().clone()).requires_grad_(True) for k, v in m.state_dict().items()}


def _tau_err(got, ref_heads):
    """As test_gpu_train_cosine.py: per-head tau against the layer's largest |d tau|; a shared tau (the sum of the heads' shares)
    against the sum of the shares' magnitudes."""
    ref_heads = ref_heads.reshape(-1)
    if got.numel() == ref_heads.numel():
        return (got.reshape(-1) - ref_heads).abs().max().item() / ref_heads.abs().max().item()
    return abs(got.reshape(-1)[0].item() - ref_heads.sum().item()) / ref_heads.abs().sum().item()


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-300)


def _cos_degenerate(m):
    _head_rows(m, 0, 0, torch.zeros_like)
    _head_rows(m, 1, 1, torch.zeros_like)
    _head_rows(m, 0, 2, lambda t: t * 1e-2)
    _head_rows(m, 1, 3, lambda t: t * 1e-2)


TRAIN_CASES = {
    "plain_1block": (1, {}, None, DROP_TEST, None),
    "plain_2blocks": (2, {}, None, DROP_TEST, None),
    "cosine_tau_per_layer_2blocks": (2, dict(cosine=True, tau_min=0.01), None, DROP_TEST, None),
    # temperatures from 0.1 up, as in test_gpu_train_cosine.py: at 0.05 (logits x 20) the bf16 operands of the training GEMMs
    # alone move single dX elements by up to 3% of the max-abs
    "cosine_tau_per_head_1block": (1, dict(cosine=True, non_shared_tau=True, tau_min=0.1), _taus_per_head_one_below(0.1), DROP_TEST,
                                   None),
    "cosine_degenerate_heads": (1, dict(cosine=True, non_shared_tau=True, tau_min=0.01), None, DROP_TEST, _cos_degenerate),
    "plain_drop_train": (1, {}, None, DROP_TRAIN, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_training_gradients(cuda, case):
    """SSTv2(precision='bf16').train() on the engineered layout (shift 0): forward, dX per token (grouped by window size), every
    parameter gradient and d tau against float64 autograd through the oracle, with the bounds of test_gpu_train*.py.  With
    DROP_TRAIN the windows are cut to 100 tokens and the plans come from the kept tokens' levels."""
    blocks, lc, taus, drop, edit = TRAIN_CASES[case]
    sizes = engineered_sizes()
    coors = engineered_coors(sizes, 0)
    m = _model(128, 8, 256, blocks, lc, taus)
    if edit:
        edit(m)
    feats = _inputs(coors, 128)
    w = _oracle_leaves(m)
    xo = feats.double().requires_grad_(True)
    info_o = O.input_layer_v2(xo, coors, drop, WIN, SPARSE)
    yo = O.sstv2_forward(info_o, w, [8] * blocks, blocks, layer_cfg=lc)
    # loss gradient = output + noise: with noise alone, a layer's d tau can cancel to a few percent of its addends, below what
    # bf16 weights alone resolve
    gy = (yo.detach() + torch.randn(yo.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)) / yo.shape[0]
    (yo * gy).sum().backward()

    m = m.to(cuda).train()
    m.precision = "bf16"
    xg = feats.to(cuda).requires_grad_(True)
    info = _gpu_info(cuda, xg, coors, drop=drop, train=True)
    keep = info["voxel_keep_inds"].cpu()
    assert torch.equal(keep, info_o["voxel_keep_inds"])
    if drop is DROP_TEST:
        tok_size = assert_engineered_plan(info, 0, sizes)
    else:
        got_sizes, _, tok_size = plan_layout(info, 0)
        assert keep.numel() < coors.shape[0] and max(got_sizes) == 100
    yg = m(info)[0]["voxel_feats"]
    full = drop is DROP_TEST   # DROP_TRAIN leaves no window above 100 tokens
    check_grouped(yg, yo, tok_size, BF16_REL, f"training forward, {case}", all_groups=full)
    (yg * gy.float().to(cuda)).sum().backward()
    check_grouped(xg.grad[keep.to(cuda)], xo.grad[keep], tok_size, GRAD_REL, f"dX, {case}", all_groups=full)

    # per-head temperatures from 0.1: in float64, perturbing the weights by 2e-3 relative (less than bf16 rounding) already moves
    # this case's first-layer d tau by up to 1.9% of its largest head, so the bf16 training path gets 5% there.  Headroom: on an
    # H100 80GB HBM3 (700 W power limit) that layer's d tau is off by 3.54e-2 (the same in every run: d tau is reduced in a fixed
    # order), 1.4x under the bound; its second layer by 5.6e-3.  The other cosine cases stay under 1e-2 against their 3e-2.
    tau_rel = 5e-2 if taus else TAU_REL
    bad, ntau = {}, 0
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        got, ref = p.grad.cpu().double(), w[name].grad
        if name.endswith("tau"):
            ntau += 1
            r = _tau_err(got, ref)
            print(f"d tau, {case}, {name}: {r:.3e} (bound {tau_rel:g})")
            if r > tau_rel:
                bad[name] = r
        elif edit and "in_proj" in name:
            # the zeroed q / k heads' gradients are 1 / 1e-12 times the others' (F.normalize's clamp): each head's rows on their own.
            # The bias of a zeroed k head sums dk over each window's keys, which cancels to 0 (sum_j g_ij = 0), so its rounding is
            # measured against the same rows' weight gradient.
            wref = w[name.replace("bias", "weight")].grad
            for i, (a, b, bw) in enumerate(zip(got.split(16), ref.split(16), wref.split(16))):
                # (the other half of a zeroed head - k of a zero-q head, q of a zero-k head - has gradient exactly 0)
                r = (a - b).abs().max().item() / max(b.abs().max().item(), bw.abs().max().item(), 1e-300)
                if r > GRAD_REL:
                    bad[f"{name}[{16 * i}:{16 * i + 16}]"] = r
        elif _rel(got, ref) > GRAD_REL:
            bad[name] = _rel(got, ref)
    assert ntau == (2 * blocks if lc.get("cosine") else 0)
    assert not bad, f"gradients off (bf16 tolerance {GRAD_REL} of max-abs, tau {tau_rel}): {bad}"
