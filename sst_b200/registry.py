"""Minimal OpenMMLab-style registry so the reference's config dicts build these modules by `type` name when
mmcv/mmdet are absent (mmdet3d/models/builder.py:1-13,86-98).  If real mmcv is importable the same classes are
additionally registered into mmcv's MODELS/BACKBONES registries (see sst_b200/__init__.py)."""
import copy
import inspect


class Registry:
    def __init__(self, name):
        self.name = name
        self._module_dict = {}

    def register_module(self, name=None, force=False, module=None):
        def deco(cls):
            key = name or cls.__name__
            if key in self._module_dict and not force:
                raise KeyError(f"{key} is already registered in {self.name}")
            self._module_dict[key] = cls
            return cls
        if module is not None:
            return deco(module)
        return deco

    def get(self, key):
        return self._module_dict.get(key)

    def build(self, cfg, default_args=None):
        if not isinstance(cfg, dict) or "type" not in cfg:
            raise TypeError(f"cfg must be a dict with a `type` key, got {cfg!r}")
        # deep copy: some reference modules mutate list-valued config entries in place
        # (SIRLayer: rel_mlp_hidden_dims.append, models/voxel_encoders/voxel_encoder.py:665)
        args = copy.deepcopy(dict(cfg))
        if default_args:
            for k, v in default_args.items():
                args.setdefault(k, v)
        t = args.pop("type")
        cls = t if inspect.isclass(t) else self.get(t)
        if cls is None:
            raise KeyError(f"{t} is not in the {self.name} registry")
        return cls(**args)

    def __contains__(self, key):
        return key in self._module_dict


MODELS = Registry("models")
VOXEL_ENCODERS = MIDDLE_ENCODERS = BACKBONES = FUSION_LAYERS = ROI_EXTRACTORS = MODELS
NORM_LAYERS = Registry("norm layer")


def build_voxel_encoder(cfg):
    return VOXEL_ENCODERS.build(cfg)


def build_middle_encoder(cfg):
    return MIDDLE_ENCODERS.build(cfg)


def build_backbone(cfg):
    return BACKBONES.build(cfg)
