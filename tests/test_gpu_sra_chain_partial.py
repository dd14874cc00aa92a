"""The fused SRA stack's partial last tile, with the row count on the device and buffers 200 rows past it.

The fused chain writes the next layer's q|k|v (a [capacity, 384] fp16 workspace) and y per 128-row tile, each warp copying its 16
rows of q|k|v out through shared memory.  At row counts on every tile and half-tile edge (1, 63, 64, 65, 127, 128, 129) and at
2 x SMs + 2 tiles with 37 rows missing from the last, rows past the count must keep what was there: q|k|v rows in [M, capacity) and
y rows past M keep a sentinel fill, and y matches the float64 oracle within the bf16 bounds of test_gpu_sra_chain.py.

The q|k|v workspace is the first allocation of the stack call in the context's arena, which is reset at the start of each call,
so it starts at the arena's base.  The test reads that base from the context (its fields `int device; cudaStream_t stream;
int num_sms; char* arena;`, checked through num_sms), fills it, and calls the stack again on the same arena.
"""
import ctypes as C

import pytest
import torch

import test_gpu_sra_chain as T

pytestmark = pytest.mark.gpu

COUNTS = [1, 63, 64, 65, 127, 128, 129, T.ODD]
QKV_FILL = -1234.0   # exact in fp16
Y_FILL = 7.0


class _Cuda:
    """Zero-copy view of device memory this test does not own"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def _arena(c, cuda):
    assert C.c_int.from_address(c + 16).value == torch.cuda.get_device_properties(cuda).multi_processor_count, "context layout changed"
    return C.c_uint64.from_address(c + 24).value


@pytest.mark.parametrize("layer_cfg", [T.LN, T.BN_COS], ids=["layernorm", "batchnorm_cosine"])
@pytest.mark.parametrize("n", COUNTS)
def test_fused_stack_partial_tile_keeps_rows_past_count(cuda, n, layer_cfg):
    from sst_b200 import _lib as L
    from sst_b200.sst_modules import PRECISIONS, _SraLayer, make_sra_plan
    n = T._rows(n)
    m, info_g, ref = T._case(cuda, n, layer_cfg)
    layers = [l for blk in m.block_list for l in blk.encoder_list]
    assert len(layers) >= 2   # the first chain carries the q|k|v tail
    arr = (_SraLayer * len(layers))(*[l._struct(PRECISIONS["bf16"]) for l in layers])
    p0, p1 = make_sra_plan(info_g["sra_plan_shift0"]), make_sra_plan(info_g["sra_plan_shift1"])
    cap = n + 200
    x = T._padded(info_g["voxel_feats"].float(), cap, 3.0)
    y, tmp = torch.full_like(x, Y_FILL), torch.empty_like(x)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    c = L.ctx(cuda)

    def run():
        L.check(c, L.lib().sstb200_sra_stack_forward(c, arr, len(layers), C.byref(p0), C.byref(p1), x.data_ptr(), y.data_ptr(),
                                                     tmp.data_ptr(), cap, n_dev.data_ptr(), PRECISIONS["bf16"]))

    run()   # sizes the arena
    torch.cuda.synchronize()
    qkv = torch.as_tensor(_Cuda(_arena(c, cuda), (cap, 384), "<f2"), device=cuda)
    qkv.fill_(QKV_FILL)
    y.fill_(Y_FILL)
    torch.cuda.synchronize()
    run()
    torch.cuda.synchronize()
    assert _arena(c, cuda) == qkv.data_ptr(), "the arena moved"
    assert (qkv[n:] == QKV_FILL).all(), "q|k|v rows past the count were written"
    assert not (qkv[:n] == QKV_FILL).any(), "q|k|v rows below the count were not all written"
    assert (y[n:] == Y_FILL).all()
    T._check(y[:n], ref)
