"""TEST INFRASTRUCTURE - recipe that compiles the reference's roiaware_pool3d sources, unmodified and in place, into
oracle/_ref/roiaware_pool3d_ext_ref*.so (points_in_boxes_{cpu,gpu,batch}: the box test FSD's RoI point pooling is pinned to):
  /root/reference/mmdet3d/ops/roiaware_pool3d/src/{roiaware_pool3d.cpp, points_in_boxes_cpu.cpp, points_in_boxes_cuda.cu,
                                                  roiaware_pool3d_kernel.cu}
Same conventions as oracle/build_ref.py (sm_90a, objects removed afterwards, nothing copied into the repository); load the result with
build_ref.load_module("roiaware_pool3d_ext_ref").  Runs only where the reference tree exists.  `python -m oracle.build_ref_roiaware`"""
import glob
import os
import shutil
import sys

from oracle.build_ref import OUT, built

NAME = "roiaware_pool3d_ext_ref"
SRC = os.path.join(os.environ.get("SST_REFERENCE_ROOT", "/root/reference"), "mmdet3d/ops/roiaware_pool3d/src")


def build(verbose=False):
    if built(NAME):
        return built(NAME)[0]
    if not os.path.isdir(SRC):
        return None
    out = os.path.join(OUT, "roiaware_build")
    os.makedirs(out, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    srcs = [os.path.join(SRC, f) for f in ("roiaware_pool3d.cpp", "points_in_boxes_cpu.cpp", "points_in_boxes_cuda.cu",
                                           "roiaware_pool3d_kernel.cu")]
    load(name=NAME, sources=srcs, extra_cflags=["-O2", "-w"], extra_cuda_cflags=["-O2", "-w", "-gencode", "arch=compute_90a,code=sm_90a"],
         build_directory=out, verbose=verbose, is_python_module=False)
    for f in glob.glob(os.path.join(out, f"{NAME}*.so")):
        shutil.copy(f, OUT)
    shutil.rmtree(out, ignore_errors=True)   # objects and ninja files do not need to travel
    return built(NAME)[0] if built(NAME) else None


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
