"""Seeded synthetic clouds for the BASELINE.json configs (SURVEY.md section 8d).

No dataset can be downloaded here, so the bench and the parity tests run on
clouds with the shapes and rough statistics of KITTI / SemanticKITTI / S3DIS /
Waymo frames.  Everything is a pure function of (kind, n, seed).
"""
import numpy as np

KITTI_RANGE = (0.0, -39.68, -3.0, 69.12, 39.68, 1.0)
WAYMO_RANGE = (-74.88, -74.88, -2.0, 74.88, 74.88, 4.0)


def lidar_frame(n, seed, pc_range=KITTI_RANGE, with_intensity=True):
    """LiDAR-like frame inside ``pc_range``: 64 elevation rings hitting a noisy
    ground plane (z ~ -1.7 +- 0.1) with |N(0,15)|+2 m ranges, plus 10 % of the
    points on box-shaped clusters.  Returns float32 [n, 4] (x, y, z, intensity)
    or [n, 3]."""
    rng = np.random.default_rng(seed)
    x0, y0, z0, x1, y1, z1 = pc_range
    n_box = n // 10
    pts = np.empty((0, 3), np.float64)
    need = n - n_box
    while len(pts) < need:
        m = int((need - len(pts)) * 1.6) + 64
        r = np.abs(rng.normal(0.0, 15.0, m)) + 2.0
        ring = rng.integers(0, 64, m)
        az = rng.uniform(-np.pi, np.pi, m)
        r = r * (1.0 + 0.02 * ring)  # farther rings reach farther
        x, y = r * np.cos(az), r * np.sin(az)
        z = -1.7 + rng.normal(0.0, 0.1, m) + 0.002 * r * (ring - 32) / 32.0
        p = np.stack([x, y, z], 1)
        ok = ((p[:, 0] >= x0) & (p[:, 0] < x1) & (p[:, 1] >= y0) & (p[:, 1] < y1) &
              (p[:, 2] >= z0) & (p[:, 2] < z1))
        pts = np.concatenate([pts, p[ok]])
    pts = pts[:need]
    nb = max(n_box // 200, 1)
    cx = rng.uniform(x0 * 0.5 + 3, min(x1, 40.0), nb) if x0 >= 0 else rng.uniform(-35, 35, nb)
    cy = rng.uniform(max(y0, -25.0), min(y1, 25.0), nb)
    which = rng.integers(0, nb, n_box)
    size = np.array([4.0, 1.8, 1.6])
    face = rng.uniform(-0.5, 0.5, (n_box, 3))
    ax = rng.integers(0, 3, n_box)
    face[np.arange(n_box), ax] = np.sign(face[np.arange(n_box), ax] + 1e-9) * 0.5
    box = np.stack([cx[which], cy[which], np.full(n_box, -0.9)], 1) + face * size
    box[:, 0] = np.clip(box[:, 0], x0, np.nextafter(np.float32(x1), np.float32(-1e9)))
    box[:, 1] = np.clip(box[:, 1], y0, np.nextafter(np.float32(y1), np.float32(-1e9)))
    box[:, 2] = np.clip(box[:, 2], z0, np.nextafter(np.float32(z1), np.float32(-1e9)))
    out = np.concatenate([pts, box]).astype(np.float32)
    out = out[rng.permutation(n)]
    # float32 rounding may touch the open upper bound; keep strictly inside
    for d, hi in enumerate((x1, y1, z1)):
        out[:, d] = np.minimum(out[:, d], np.nextafter(np.float32(hi), np.float32(-1e9)))
    if with_intensity:
        out = np.concatenate([out, rng.uniform(0, 1, (n, 1)).astype(np.float32)], 1)
    return out


def semantickitti_cloud(n, seed):
    """RandLA-Net input: xyz only, recentred in x,y (randlanet_semantickitti.yml:31-33)."""
    p = lidar_frame(n, seed, (-50.0, -50.0, -3.0, 50.0, 50.0, 1.0), with_intensity=False)
    p[:, :2] -= p[:, :2].mean(0, keepdims=True)
    return p


def uniform_cloud(n, seed, lo=0.0, hi=10.0, dims=3):
    rng = np.random.default_rng(seed)
    return rng.uniform(lo, hi, (n, dims)).astype(np.float32)


def uniform_frame(n, seed, pc_range=KITTI_RANGE):
    """Worst case for PointPillars: uniform points -> ~one pillar per point."""
    rng = np.random.default_rng(seed)
    lo, hi = np.array(pc_range[:3]), np.array(pc_range[3:])
    p = rng.uniform(lo, hi, (n, 3))
    out = np.concatenate([p, rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
    for d in range(3):
        out[:, d] = np.minimum(out[:, d], np.nextafter(np.float32(hi[d]), np.float32(-1e9)))
    return out


def room_cloud(n, seed, dl=0.04, room=(6.0, 5.0, 2.7), feat_dim=5):
    """S3DIS-like room surfaces (walls, floor, ceiling, furniture boxes), snapped
    to a ``dl`` grid and de-duplicated, n points; features [n, feat_dim]
    (constant 1, rgb, height) like KPFCNN.transform builds them."""
    rng = np.random.default_rng(seed)
    lx, ly, lz = room
    pts = np.empty((0, 3))
    while len(pts) < n:
        m = 2 * n
        kind = rng.integers(0, 8, m)
        u, v = rng.uniform(0, 1, m), rng.uniform(0, 1, m)
        p = np.zeros((m, 3))
        for kd, (a, b, c) in enumerate([(0, 1, 0.0), (0, 1, lz), (0, 2, 0.0), (0, 2, ly),
                                        (1, 2, 0.0), (1, 2, lx)]):
            s = kind == kd
            dims = [lx, ly, lz]
            fixed = ({0, 1, 2} - {a, b}).pop()
            p[s, a], p[s, b], p[s, fixed] = u[s] * dims[a], v[s] * dims[b], c
        s = kind >= 6  # furniture: box surfaces
        nb = 6
        centers = rng.uniform([lx / 6, ly / 5, lz * 0.15], [lx * 5 / 6, ly * 4 / 5, lz * 0.3], (nb, 3))
        w = rng.integers(0, nb, m)
        f = rng.uniform(-0.5, 0.5, (m, 3))
        ax = rng.integers(0, 3, m)
        f[np.arange(m), ax] = np.sign(f[np.arange(m), ax] + 1e-9) * 0.5
        p[s] = (centers[w] + f * np.array([lx * 0.2, ly * 0.14, lz * 0.3]))[s]
        q = np.round(p / dl).astype(np.int64)
        _, first = np.unique(q, axis=0, return_index=True)
        pts = np.concatenate([pts, (q[np.sort(first)] * dl)])
        q = np.round(pts / dl).astype(np.int64)
        _, first = np.unique(q, axis=0, return_index=True)
        pts = pts[np.sort(first)]
    pts = pts[rng.permutation(len(pts))[:n]].astype(np.float32)
    feats = np.ones((n, feat_dim), np.float32)
    if feat_dim >= 4:
        feats[:, 1:4] = rng.uniform(0, 1, (n, 3))
    if feat_dim >= 5:
        feats[:, 4] = pts[:, 2]
    return pts, feats


def pvcnn_s3dis_input(n, seed):
    """PVCNN's S3DIS input by the arithmetic of PVCNN.preprocess (pvcnn.py:203-223) on a room_cloud: min-shifted xyz,
    colour in [0, 1], xyz over its per-axis maximum.  -> (point [n, 3], feat [n, 9]) float32 rows."""
    pts, f = room_cloud(n, seed)
    pts = pts - pts.min(0)
    feat = np.concatenate([pts, f[:, 1:4], pts / pts.max(0)], 1)
    return pts.astype(np.float32), feat.astype(np.float32)


def sparseconvunet_scannet_input(n, seed, voxel_size=0.02, grid_size=4096):
    """SparseConvUnet's test-split input by the arithmetic of SparseConvUnet.preprocess (sparseconvnet.py:106-145) on a
    room_cloud sampled at 1 cm: xyz over voxel_size, shifted to a random place inside the grid and moved to the voxel
    centre k + 0.5; colour in [0, 1].  -> (point [n, 3], feat [n, 3]) float32 rows."""
    pts, f = room_cloud(n, seed, dl=0.01)
    rng = np.random.default_rng(seed + 1)
    p = pts / np.float32(voxel_size)
    p = p - p.min(0) + np.clip(grid_size - (p.max(0) - p.min(0)) - 0.001, 0, None) * rng.random(3)
    return (p.astype(np.int32) + 0.5).astype(np.float32), f[:, 1:4].copy()


def grid_subsample(points, dl):
    """Barycentre grid subsampling (stand-in for `open3d.ml.contrib.subsample`,
    kpconv.py:2037-2164; a "next" row of SURVEY.md 8f).  Deterministic."""
    q = np.floor(points / dl).astype(np.int64)
    _, inv, cnt = np.unique(q, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    out = np.zeros((len(cnt), 3), np.float64)
    np.add.at(out, inv, points.astype(np.float64))
    return (out / cnt[:, None]).astype(np.float32)
