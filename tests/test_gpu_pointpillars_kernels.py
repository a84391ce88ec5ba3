"""The fused pillar feature net + BEV scatter (voxelize.cu pp_pfn_scatter_kernel) against the reference's
PillarFeatureNet + PFNLayer + PointPillarsScatter in float64: dense [M, max_points, C] pillars gathered from the voxel
CSR, decorated by the torch port (oracle/models_torch.pp_decorate), then the layer in the kernel's folded-BN form.  The
voxel CSR comes from the CUDA voxelize, which is bit-exact against the oracle (test_gpu_ops.py)."""
import numpy as np
import pytest
import torch

from open3d_ml_b200 import _lib as L
from open3d_ml_b200 import ops
from oracle import models_torch as MT

from conftest import rel_err

pytestmark = pytest.mark.gpu

COUT = 64
VOXEL = (0.25, 0.25, 4.0)
RANGE = (0.0, 0.0, -3.0, 32.0, 32.0, 1.0)
NX = NY = 128
# Against float64 on an H100 80GB HBM3 (400 W power limit), the largest rel_err of the pillar features over the
# cases below was 3.3e-7; the bound keeps about 5x of margin.
PFN_TOL = 1.7e-6


def _frame(n, C, max_pts, g):
    """n background points in y < 30 (about 14 000 pillars over two frames, more than the kernel's grid-stride loop
    covers in one pass on an H100), pillars of exactly 1, max_pts - 1, max_pts and max_pts + 5 points in the strip
    y in [30, 32), and points on x == 32 or y == 32, the range's upper faces, whose pillars sit at cx == nx or
    cy == ny: outside the canvas."""
    bg = torch.rand(n, 3, generator=g) * torch.tensor([32.0, 30.0, 3.9]) + torch.tensor([0.0, 0.0, -2.95])
    parts = [bg]
    for j, cnt in enumerate((1, max(max_pts - 1, 1), max_pts, max_pts + 5)):
        cell = torch.tensor([0.25 * (3 * j + 1), 30.25 + 0.5 * (j % 3)])
        xy = cell + torch.rand(cnt, 2, generator=g) * 0.2 + 0.02
        parts.append(torch.cat([xy, torch.rand(cnt, 1, generator=g) * 3.0 - 2.5], 1))
    edge = torch.rand(6, 3, generator=g) * torch.tensor([31.0, 31.0, 3.0]) + torch.tensor([0.5, 0.5, -2.5])
    edge[:3, 0] = 32.0
    edge[3:, 1] = 32.0
    parts.append(edge)
    xyz = torch.cat(parts)
    extra = torch.randn(xyz.shape[0], C - 3, generator=g)
    return torch.cat([xyz, extra], 1)


def pillar_decoration(pts, coords, vrs, pidx, M, max_pts, vx, vy, x_off, y_off):
    """The first M pillars of the voxel CSR as dense float64 [M, P, C] pillars (padded slots zero), decorated by the
    torch port: -> ([M, P, C+5] with the padded slots zeroed, the slot mask [M, P])."""
    rs = vrs[:M + 1].long()
    cnt = rs[1:] - rs[:-1]
    slot = torch.arange(max_pts, device=pts.device).view(1, -1)
    mask = slot < cnt.view(-1, 1)
    src = torch.where(mask, pidx[(rs[:-1].view(-1, 1) + slot).clamp_max(pidx.numel() - 1)], -1)
    pillars = torch.cat([torch.zeros_like(pts[:1]), pts]).double()[src + 1]
    c = coords[:M].double()
    return MT.pp_decorate(pillars, cnt, c[:, 0], c[:, 1], vx, vy, x_off, y_off), mask


def pfn_reference(pts, coords, vrs, pidx, M, max_pts, wt, scale, shift, vx, vy, x_off, y_off):
    """[M, 64] float64 pillar features (point_pillars.py PillarFeatureNet / PFNLayer)."""
    f, _ = pillar_decoration(pts, coords, vrs, pidx, M, max_pts, vx, vy, x_off, y_off)
    y = torch.relu((f @ wt.double()) * scale.double() + shift.double())
    return y.max(1)[0]


def scatter_reference(feat, coords, bid, B):
    """NCHW canvas, NaN where no in-grid pillar lands (point_pillars.py PointPillarsScatter, on a NaN canvas)."""
    canvas = torch.full((B, COUT, NY, NX), float("nan"), dtype=torch.float64, device=feat.device)
    c = coords[:feat.shape[0]].long()
    ok = (c[:, 0] < NX) & (c[:, 1] < NY)
    b = bid[:feat.shape[0]].long()
    canvas[b[ok], :, c[ok, 1], c[ok, 0]] = feat[ok]
    return canvas


@pytest.mark.parametrize("max_pts", [1, 20, 32])
@pytest.mark.parametrize("C", [3, 4, 5, 11])
def test_pfn_scatter_vs_float64(C, max_pts):
    g = torch.Generator().manual_seed(100 + 10 * C + max_pts)
    frames = [_frame(20000, C, max_pts, g), torch.zeros(0, C), _frame(20000, C, max_pts, g)]   # B = 3, frame 1 empty
    B = len(frames)
    pts = torch.cat(frames).cuda().contiguous()
    rs = torch.tensor(np.cumsum([0] + [f.shape[0] for f in frames]), dtype=torch.int64).cuda()
    coords, pidx, vrs, _, bid, counts = ops.voxelize_raw(pts[:, :3], rs, VOXEL, RANGE[:3], RANGE[3:], max_pts,
                                                         10 ** 6, want_batch_id=True)
    M = int(counts[0])
    bound = pts.shape[0]
    assert M < bound and M > 132 * 64
    wt = (torch.randn(C + 5, COUT, generator=g) * 0.3).cuda()
    scale = (torch.randn(COUT, generator=g) * 0.5 + 1.0).cuda()
    shift = torch.randn(COUT, generator=g).cuda()                        # both signs: relu(shift) of padded slots
    assert float(shift.min()) < 0 < float(shift.max())
    vx, vy = VOXEL[0], VOXEL[1]
    x_off, y_off = float(np.float32(vx / 2 + RANGE[0])), float(np.float32(vy / 2 + RANGE[1]))

    def run(feat, canvas, nchw):
        n0 = L.lib().o3dml_launch_count()
        L.check(L.lib().o3dml_pp_pfn_scatter(
            L.ptr(pts), pts.stride(0), C, L.ptr(coords), L.ptr(vrs), L.ptr(pidx), L.ptr(bid), L.ptr(counts), bound,
            L.ptr(wt), L.ptr(scale), L.ptr(shift), COUT, vx, vy, x_off, y_off, NX, NY, max_pts, L.ptr(feat),
            L.ptr(canvas), nchw, L.stream()))
        assert L.lib().o3dml_launch_count() == n0 + 1

    nan = float("nan")
    feat = torch.full((bound, COUT), nan).cuda()
    nhwc = torch.full((B, NY, NX, COUT), nan).cuda()
    run(feat, nhwc, 0)
    nchw = torch.full((B, COUT, NY, NX), nan).cuda()
    run(None, nchw, 1)                                                  # canvas without feat_out
    feat2 = torch.full((bound, COUT), nan).cuda()
    run(feat2, None, 0)                                                 # feat_out without canvas
    torch.cuda.synchronize()

    ref = pfn_reference(pts, coords, vrs, pidx, M, max_pts, wt, scale, shift, vx, vy, x_off, y_off)
    err = rel_err(feat[:M], ref)
    assert err < PFN_TOL, err
    assert bool(feat[M:].isnan().all()), "rows of feat_out past the device voxel count were written"
    assert torch.equal(feat2[:M], feat[:M]) and bool(feat2[M:].isnan().all())
    # pillars of every size the case builds, including some outside the canvas
    cnt = (vrs[1:M + 1] - vrs[:M])
    for k in {1, max(max_pts - 1, 1), max_pts}:
        assert bool((cnt == k).any()), k
    c = coords[:M].long()
    assert bool((c[:, 0] == NX).any()) and bool((c[:, 1] == NY).any())

    cref = scatter_reference(feat[:M].double(), coords, bid, B)
    assert torch.equal(nchw.isnan(), cref.isnan()), "written canvas cells differ from the in-grid pillars"
    assert torch.equal(nchw.nan_to_num(0.0), cref.float().nan_to_num(0.0))          # the scattered rows of feat_out
    assert bool(nchw[1].isnan().all())                                                 # the empty frame
    assert torch.equal(nhwc.permute(0, 3, 1, 2).nan_to_num(0.0), nchw.nan_to_num(0.0))
    assert torch.equal(nhwc.permute(0, 3, 1, 2).isnan(), nchw.isnan())
