"""The caller-owned workspace size queries, restated as sums of 256-byte-rounded pieces.

sstb200_sra_train_workspace_bytes and sstb200_sir_layer_train_state_bytes tell a caller how large a buffer to allocate; a change to
either breaks callers that cache the size, so both are pinned here over a grid of shapes.  Neither needs a device."""
import ctypes as C

import pytest

from sst_b200 import _lib as L
from sst_b200 import sir_modules as SM


def al256(b):
    return (b + 255) // 256 * 256


def sra_train_bytes(n, num_layers):
    DM, DFF = 128, 256
    N = max(n, 1)
    layer = (al256(N * DM * 4) + al256(N * 3 * DM * 2) + al256(N * DM * 2) + 2 * al256(N * DM * 4) + al256(N * DM * 2) +
             2 * al256(N * DFF * 2) + al256(N * DM * 4))
    shared = (al256(N * DM * 4) + al256(N * DM * 2) + al256(N * DFF * 2) + al256(N * DM * 2) + al256(N * 3 * DM * 2) +
              3 * al256(N * DM * 4) + al256(N * 8 * 3 * 4))
    return layer * num_layers + shared


def sir_state_bytes(N, G, C0, C1):
    return al256(N * C0 * 4) + al256(N * C1 * 4) + al256(G * C0 * 8) + al256(G * C1 * 8)


@pytest.fixture(scope="module")
def lib():
    lb = L.lib()
    lb.sstb200_sra_train_workspace_bytes.restype = C.c_size_t
    lb.sstb200_sra_train_workspace_bytes.argtypes = [C.c_int, C.c_int]
    return lb


@pytest.mark.parametrize("num_layers", [1, 2, 3, 6])
@pytest.mark.parametrize("n", [-3, 0, 1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000, 4097, 20011, 150000])
def test_sra_train_workspace_bytes(lib, n, num_layers):
    assert lib.sstb200_sra_train_workspace_bytes(n, num_layers) == sra_train_bytes(n, num_layers)


@pytest.mark.parametrize("C0,C1", [(32, 0), (64, 0), (32, 64), (64, 64), (128, 128), (96, 256)])
@pytest.mark.parametrize("N,G", [(0, 0), (1, 1), (7, 3), (33, 1), (64, 64), (1000, 17), (4097, 4097), (150001, 9000)])
def test_sir_layer_train_state_bytes(N, G, C0, C1):
    s = SM._SirLayer()
    s.num_vfe = 2 if C1 else 1
    s.feat_channels[0], s.feat_channels[1] = C0, C1
    assert L.lib().sstb200_sir_layer_train_state_bytes(C.byref(s), N, G) == sir_state_bytes(N, G, C0, C1)


def test_sir_layer_train_state_bytes_refuses():
    s = SM._SirLayer()
    s.num_vfe, s.feat_channels[0] = 1, 32
    assert L.lib().sstb200_sir_layer_train_state_bytes(C.byref(s), -1, 4) == 0
    s.num_vfe = 3
    assert L.lib().sstb200_sir_layer_train_state_bytes(C.byref(s), 8, 4) == 0
