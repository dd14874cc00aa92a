"""TEST INFRASTRUCTURE - recipe that compiles the reference's OWN native sources, unmodified and in place, into oracle/_ref/:
  voxel_layer_ref*.so       /root/reference/mmdet3d/ops/voxel/src/*.{cpp,cu}
  sparse_conv_ext_ref*.so   /root/reference/mmdet3d/ops/spconv/src/*.{cc,cu} (+ include/) - the vendored spconv v1

The result is used only by tests (to pin oracle/sst_oracle.py and the CUDA path against the real reference
kernels on a GPU box).  Nothing is copied into the repo; oracle/_ref/ is git-ignored but travels with gpurun.
Runs only where /root/reference exists (the build container).  `python -m oracle.build_ref`
"""
import glob
import os
import sys

REF_SRC = os.path.join(os.environ.get("SST_REFERENCE_ROOT", "/root/reference"), "mmdet3d/ops/voxel/src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


SPCONV_ROOT = os.path.join(os.environ.get("SST_REFERENCE_ROOT", "/root/reference"), "mmdet3d/ops/spconv")


def built(name="voxel_layer_ref"):
    return sorted(glob.glob(os.path.join(OUT, f"{name}*.so")))


def build_spconv(verbose=False):
    name = "sparse_conv_ext_ref"
    if built(name):
        return built(name)[0]
    if not os.path.isdir(SPCONV_ROOT):
        return None
    out = os.path.join(OUT, "spconv_build")
    os.makedirs(out, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils.cpp_extension import load
    srcs = [os.path.join(SPCONV_ROOT, "src", f) for f in ("all.cc", "indice.cc", "indice_cuda.cu", "reordering.cc", "reordering_cuda.cu",
                                                          "maxpool.cc", "maxpool_cuda.cu")]
    load(name=name, sources=srcs, extra_include_paths=[os.path.join(SPCONV_ROOT, "include")], extra_cflags=["-O2", "-w"],
         extra_cuda_cflags=["-O2", "-w", "-gencode", "arch=compute_90a,code=sm_90a"], build_directory=out, verbose=verbose,
         is_python_module=False)
    import shutil
    for f in glob.glob(os.path.join(out, f"{name}*.so")):
        shutil.copy(f, OUT)
    shutil.rmtree(out, ignore_errors=True)   # objects and ninja files do not need to travel
    return built(name)[0] if built(name) else None


def build(verbose=False):
    build_spconv(verbose)
    if built():
        return built()[0]
    if not os.path.isdir(REF_SRC):
        return None
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "6")
    from torch.utils.cpp_extension import load
    srcs = [os.path.join(REF_SRC, f) for f in ("voxelization.cpp", "voxelization_cpu.cpp", "scatter_points_cpu.cpp",
                                               "scatter_points_cuda.cu", "voxelization_cuda.cu")]
    load(name="voxel_layer_ref", sources=srcs, extra_cflags=["-DWITH_CUDA", "-O2"],
         extra_cuda_cflags=["-DWITH_CUDA", "-O2", "-gencode", "arch=compute_90a,code=sm_90a"],
         build_directory=OUT, verbose=verbose, is_python_module=False)
    return built()[0] if built() else None


def load_module(name="voxel_layer_ref"):
    """Import the prebuilt extension (no compilation; works on the GPU box where the sources are absent)."""
    so = built(name)
    if not so:
        return None
    import importlib.util
    import torch  # noqa: F401  (libtorch symbols)
    spec = importlib.util.spec_from_file_location(name, so[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
