"""CPU: the C-ABI library loads without a GPU and exports every function include/sstb200.h declares;
every declared function also has a ctypes prototype (no un-prototyped, pointer-truncating calls)."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    h = open(os.path.join(ROOT, "include", "sstb200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    return sorted(set(re.findall(r"\b(sstb200_[a-z0-9_]+)\s*\(", h)))


def test_library_builds_and_exports_all_symbols():
    from sst_b200 import build
    so = build.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", so], text=True)
    exported = set(re.findall(r" T (sstb200_[a-z0-9_]+)", out))
    decl = _declared()
    assert len(decl) >= 20
    missing = [d for d in decl if d not in exported]
    assert not missing, f"declared in include/sstb200.h but not exported: {missing}"
    extra = sorted(exported - set(decl))
    assert not extra, f"exported but not declared: {extra}"


def test_every_symbol_has_a_ctypes_prototype():
    import sst_b200  # noqa: F401
    from sst_b200 import _lib, engine, sir_modules  # noqa: F401  (late registrations)
    L = _lib.lib()
    assert L.sstb200_version() >= 100
    for name in _declared():
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature"
        assert getattr(L, name).argtypes is not None


def test_no_cpu_fallback():
    import pytest
    import torch
    from sst_b200 import _lib, ops
    with pytest.raises(_lib.SSTB200Error):
        ops.get_inner_win_inds(torch.zeros(4, dtype=torch.long))
    with pytest.raises(_lib.SSTB200Error):
        ops.scatter_v2(torch.zeros(4, 2), torch.zeros(4, 3, dtype=torch.long), "max")


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "sst_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("# oracle", ""), f"{f} mentions the oracle"


def test_sass_carries_the_hopper_instructions():
    """The built library really contains the sm_90a tensor-core path (no silent SIMT-only build): wgmma.mma_async -> HGMMA,
    cp.async -> LDGSTS, cp.async.bulk.tensor (TMA) -> UTMALDG, mma.sync -> HMMA, redux.sync -> REDUX, tanh.approx -> MUFU.TANH."""
    import shutil
    import pytest
    from sst_b200 import build
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    so = build.build()
    sass = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass and "arch = sm_100" not in sass
    for mnemonic in ("HGMMA.64x128x16.F32", "HGMMA.64x64x16.F32.BF16", "LDGSTS", "UTMALDG", "HMMA.16816.F32", "REDUX", "MUFU.TANH"):
        assert mnemonic in sass, f"{mnemonic} missing from the SASS of {so}"
    # every tensor-core kernel family is present
    for kern in ("sra_chain2_kernel", "wgmma_gemm_kernel", "spconv_wgmma_kernel", "vfe_l1_wgmma_kernel", "sir_a_kernel", "sir_b_kernel"):
        assert kern in sass, kern
