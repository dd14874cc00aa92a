"""sst_b200 - H100-native (sm_90a) implementation of the SST / FSD data-parallel hot path behind the reference's
own module / op names (tusen-ai/SST).  The arithmetic lives in libsstb200.so (csrc/*.cu, C ABI in
include/sstb200.h); this package is the host-side mirror of the reference interface.  There is no CPU or
PyTorch fallback: using an op without the built library or without a CUDA device raises."""
from . import registry
from .registry import BACKBONES, MIDDLE_ENCODERS, MODELS, ROI_EXTRACTORS, VOXEL_ENCODERS, build_backbone, build_middle_encoder, build_voxel_encoder  # noqa: F401
from . import norm  # noqa: F401
from . import ops  # noqa: F401
from . import sst_modules, voxel_modules, sir_modules, neck_modules, fsdv2_modules, spconv_modules, fsd_modules, roiaware_modules, dcn_modules, centerhead_modules, anchor3d_modules, voteseg_modules, cluster_head_modules, fsdv2_head_modules, roi_head_modules  # noqa: F401
from .sst_modules import SSTInputLayer, SSTInputLayerV2, SSTv1, SSTv2, SST, PseudoMiddleEncoderForSpconvFSD  # noqa: F401
from .voxel_modules import DynamicVFE, DynamicScatterVFE  # noqa: F401
from .sir_modules import SIR, SIRLayer  # noqa: F401
from .neck_modules import Voxel2PointScatterNeck  # noqa: F401
from .fsdv2_modules import VirtualVoxelFront  # noqa: F401
from .fsd_modules import ClusterAssigner, DynamicPointROIExtractor  # noqa: F401
from .roiaware_modules import Single3DRoIAwareExtractor  # noqa: F401
from .dcn_modules import DeformConv2d, DeformConv2dPack, SeparateHead, DCNSeparateHead  # noqa: F401
from .centerhead_modules import CenterHead  # noqa: F401
from .anchor3d_modules import SECONDFPN, Anchor3DHead  # noqa: F401
from .voteseg_modules import VoteSegHead, VoteSegmentor  # noqa: F401
from .cluster_head_modules import FSDSeparateHead, SparseClusterHeadV2  # noqa: F401
from .fsdv2_head_modules import FSDV2Head  # noqa: F401
from .roi_head_modules import FullySparseBboxHead, GroupCorrectionHead  # noqa: F401
from .spconv_modules import SimpleSparseUNet, SparseUNet, VirtualVoxelMixer, SparseConvTensor  # noqa: F401
# `from mmdet3d.ops import SparseBasicBlock, make_sparse_convmodule` (mmdet3d/ops/__init__.py:21-22) resolves on the op namespace too
ops.SparseBasicBlock, ops.make_sparse_convmodule = spconv_modules.SparseBasicBlock, spconv_modules.make_sparse_convmodule
from . import train  # noqa: F401  (training entry points: autograd bridge, FlatAdamW)

__version__ = "0.1.0"
