"""CPU, build container only: the gradients of the oracle's recover_bev and voxel2point_neck (what the GPU backward tests compare
against) pinned to autograd through the reference's own SSTv2.recover_bev and Voxel2PointScatterNeck (unmodified, through
oracle/ref_shim.py).  Skipped where /root/reference does not exist (e.g. the GPU box)."""
import pytest
import torch

from oracle import ref_shim, sst_oracle as O

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]


@pytest.fixture(scope="module")
def R():
    return ref_shim.load()


@pytest.mark.parametrize("B,C,ny,nx,M,dup", [(1, 16, 60, 70, 900, 0), (2, 37, 50, 45, 700, 0), (2, 8, 20, 30, 300, 80), (2, 8, 10, 10, 0, 0)])
def test_recover_bev_gradients(R, B, C, ny, nx, M, dup):
    """Rows sharing a cell each receive that cell's gradient, in the reference's per-sample loop as in the oracle."""
    g = torch.Generator().manual_seed(M + C + dup)
    cells = torch.randperm(B * ny * nx, generator=g)[:M]
    if dup:
        cells = torch.cat([cells, cells[torch.randint(0, M, (dup,), generator=g)]])
        cells = cells[torch.randperm(cells.numel(), generator=g)]
    b, rem = cells // (ny * nx), cells % (ny * nx)
    coors = torch.stack([b, torch.zeros_like(b), rem // nx, rem % nx], 1)
    feat = torch.randn(cells.numel(), C, generator=g)
    probe = torch.randn(B, C, ny, nx, generator=g)
    bb = R.SSTv2(d_model=[C], nhead=[1], num_blocks=0, dim_feedforward=[C], output_shape=[ny, nx], num_attached_conv=0, to_bev=True)
    xr = feat.clone().requires_grad_(True)
    (bb.recover_bev(xr, coors, B) * probe).sum().backward()
    xo = feat.clone().requires_grad_(True)
    (O.recover_bev(xo, coors, B, (ny, nx)) * probe).sum().backward()
    assert torch.equal(xo.grad, xr.grad)
    if dup:  # duplicated rows: each copy carries the full gradient of its cell
        flat = b * ny * nx + rem
        assert torch.equal(xo.grad, probe.permute(0, 2, 3, 1).reshape(-1, C)[flat])


@pytest.mark.parametrize("with_xyz,norm", [(True, False), (True, True), (False, False)])
def test_voxel2point_neck_gradients(R, with_xyz, norm):
    g = torch.Generator().manual_seed(6)
    N, M, C = 5000, 700, 16
    pts = O.synth_frame(3, N, extra_dims=1)
    coors = torch.nn.functional.pad(O.dynamic_voxelize(pts, VS, RNG), (1, 0), value=0).long()
    vf = torch.randn(M, C, generator=g)
    vf[::7] = -1.0
    inds = torch.randint(0, M, (N,), generator=g)
    neck = R.Voxel2PointScatterNeck(point_cloud_range=RNG, voxel_size=VS, with_xyz=with_xyz, normalize_local_xyz=norm).eval()
    xr = vf.clone().requires_grad_(True)
    r_out, r_mask = neck(pts, coors, xr, inds)
    probe = torch.randn(r_out.shape, generator=g)
    (r_out * probe).sum().backward()
    xo = vf.clone().requires_grad_(True)
    o_out, o_mask = O.voxel2point_neck(pts, coors, xo, inds, VS, RNG, with_xyz, norm)
    assert torch.equal(o_mask, r_mask)
    (o_out * probe).sum().backward()
    assert (xo.grad - xr.grad).abs().max().item() <= 1e-6 * xr.grad.abs().max().item()
    assert int((xo.grad[::7] != 0).sum()) == 0
