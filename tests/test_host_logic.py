"""CPU: host-side logic of the package (no GPU, no compute calls): registry builds, positional table vs the oracle,
drop-possibility check, lazy reference-layout dicts."""

import pytest
import torch

from oracle import sst_oracle as O


def test_registry_builds_flagship_and_deepcopies_lists():
    from sst_b200 import flagship as fl, registry
    vfe, il, bb = fl.build_sst(fl.sst_cfg(num_blocks=2))
    assert len(bb.block_list) == 2 and bb.block_list[0].encoder_list[1].win_attn.self_attn.in_proj_weight.shape == (384, 128)
    # aliasing trap of SIRLayer (voxel_encoder.py:665): `[[16, 32]] * 3` shares one list object
    cfg = dict(type='SIR', num_blocks=3, in_channels=[84, 133, 133], feat_channels=[[128, 128]] * 3,
               rel_mlp_hidden_dims=[[16, 32]] * 3, norm_cfg=dict(type='LN', eps=1e-3), mode='max', xyz_normalizer=[20, 20, 4],
               act='gelu', unique_once=True)
    sir = registry.build_backbone(cfg)
    assert [tuple(b.rel_mlp[2][0].weight.shape) for b in sir.block_list] == [(84, 32), (133, 32), (133, 32)]
    assert cfg['rel_mlp_hidden_dims'][0] == [16, 32], "config must not be mutated"
    assert sir.block_list[0].vfe_layers[1].linear.weight.shape == (128, 256)


def test_pos_table_matches_oracle():
    from sst_b200.sst_modules import _pos_table
    for ws, d in (((12, 12, 1), 128), ((12, 12), 64), ((10, 10, 4), 96)):
        tab, ndim, maxw, L = _pos_table(ws, d, 10000, False)
        g = torch.Generator().manual_seed(0)
        w3 = ws if len(ws) == 3 else (ws[0], ws[1], 1)
        ciw = torch.stack([torch.randint(0, w3[2], (200,), generator=g), torch.randint(0, w3[1], (200,), generator=g),
                           torch.randint(0, w3[0], (200,), generator=g)], 1)
        ref = O.pos_embed_flat(ciw, ws, d, 10000, False)
        parts = [tab[a][ciw[:, 2 - a]] for a in range(ndim)]
        got = torch.cat(parts, 1)
        got = torch.cat([got, got.new_zeros(200, d - got.shape[1])], 1)
        assert torch.equal(got, ref)


def test_may_drop_host_check():
    from sst_b200 import flagship as fl
    from sst_b200.sst_modules import SSTInputLayerV2
    il = SSTInputLayerV2((fl.DROP_TRAIN, fl.DROP_TEST), (12, 12, 1), (468, 468, 1), mute=True)
    il.eval().set_drop_info()
    assert not il._may_drop()          # test drop_info keeps 144 = the whole 12x12 window
    il2 = SSTInputLayerV2((fl.DROP_TRAIN, fl.DROP_TEST), (12, 12, 1), (468, 468, 1), mute=True).train()
    il2.set_drop_info()
    assert il2._may_drop()             # training drop_info caps windows at 100 tokens


def test_lazy_dict_materialises_once():
    from sst_b200.sst_modules import _LazyDict
    calls = []
    d = _LazyDict(lambda: calls.append(1) or {0: "a", "voxel_drop_level": "b"})
    assert not calls
    assert 0 in d and d[0] == "a" and list(d.keys()) == [0, "voxel_drop_level"] and len(d) == 2
    assert len(calls) == 1


def test_product_synth_frame_equals_oracle_generator():
    """bench.py draws its sweeps from sst_b200.flagship.synth_frame; the oracle's generator (SURVEY 8d) is the checker."""
    from sst_b200 import flagship as fl
    for seed, P, extra in ((1000, 5000, 0), (3, 777, 2)):
        assert torch.equal(fl.synth_frame(seed, P, extra), O.synth_frame(seed, P, extra))


def test_strict_config_walk_rejects_missing_hot_path_types():
    """find_hot_path_modules cannot pass by skipping: a reference hot-path type that is not registered is an error, every
    type the reference registers from a hot-path file IS registered, and the dead `SST` name resolves but refuses to build."""
    from sst_b200 import registry, norm  # noqa: F401
    from sst_b200.config import REFERENCE_HOT_PATH_TYPES, find_hot_path_modules
    for t in REFERENCE_HOT_PATH_TYPES:
        assert (t in registry.NORM_LAYERS) if t.startswith("naiveSyncBN") else (t in registry.MODELS), t
    empty = registry.Registry("empty")
    with pytest.raises(KeyError):
        find_hot_path_modules({"backbone": {"type": "SSTv1"}}, empty)
    assert find_hot_path_modules({"backbone": {"type": "SomethingElse"}}, empty) == []
    with pytest.raises(NotImplementedError):
        registry.MODELS.build({"type": "SST"})
    bn = registry.NORM_LAYERS.get("naiveSyncBN3d")(4).eval()
    x = torch.randn(2, 4, 3, 3, 3)
    torch.testing.assert_close(bn(x), torch.nn.functional.batch_norm(x, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.1, bn.eps))
