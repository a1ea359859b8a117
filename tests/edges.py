"""Inputs at the edges where the kernels' exactness claims matter, and plain numpy references for them.

The synthetic room of synthetic.py is well conditioned by construction: no exact distance ties, no collinear,
duplicated or exactly coplanar neighbourhoods, no coordinate beyond ~35 m, no coarsened grid, no repeated curvature.
Real maps reach all of these (kilometre-scale map frames, VoxelGrid centroids of walls, poles, small cells).  The
generators here build them on purpose, mostly from exactly representable coordinates, so that a tie is a real tie in
float and not an accident of rounding.  numpy only: the GPU tests (test_gpu_edges.py) and the CPU tests of the
generators themselves (test_edges_cpu.py) both use this module.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32


def cloud(xyz, intensity=None) -> np.ndarray:
    """[n, 3] coordinates (+ optional intensity) -> float32 [n, 4]."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    w = np.zeros((xyz.shape[0], 1), np.float32) if intensity is None else np.asarray(intensity, np.float32).reshape(-1, 1)
    return np.ascontiguousarray(np.concatenate([xyz, w], 1))


def rot_z(yaw: float) -> np.ndarray:
    c, s = math.cos(yaw), math.sin(yaw)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


# ------------------------------------------------------------------------------------------------ kNN reference
def sqdist_f32(map_xyz: np.ndarray, q_xyz: np.ndarray) -> np.ndarray:
    """[nq, m] squared distances in float32, in FLANN's L2_Simple order: (dx*dx + dy*dy) + dz*dz."""
    d = map_xyz[None, :, :3].astype(np.float32) - q_xyz[:, None, :3].astype(np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn_brute(map_: np.ndarray, q: np.ndarray, k: int, max_sqdist: float, extra: int = 0, chunk: int = 256):
    """Exact kNN: ascending (d2, original index) over the finite map points, d2 < max_sqdist; missing slots -1 / +inf.
    With extra > 0 the (k + extra) nearest are returned without the radius cut (to see what lies past the K-th)."""
    map_ = np.asarray(map_, np.float32)
    q = np.asarray(q, np.float32)
    fin = np.nonzero(np.all(np.isfinite(map_[:, :3]), axis=1))[0]
    mp = map_[fin]
    kk = k + extra
    idx = np.full((q.shape[0], kk), -1, np.int64)
    sqd = np.full((q.shape[0], kk), np.inf, np.float32)
    qfin = np.all(np.isfinite(q[:, :3]), axis=1)
    for a in range(0, q.shape[0], chunk):
        b = min(a + chunk, q.shape[0])
        sel = np.nonzero(qfin[a:b])[0] + a
        if sel.size == 0 or mp.shape[0] == 0:
            continue
        d2 = sqdist_f32(mp, q[sel])
        order = np.argsort(d2, axis=1, kind="stable")[:, :kk]  # stable: equal d2 keep ascending original index
        dd = np.take_along_axis(d2, order, 1)
        n = order.shape[1]
        idx[sel, :n] = fin[order]
        sqd[sel, :n] = dd
    if extra == 0:
        out = ~(sqd < np.float32(max_sqdist))
        idx[out], sqd[out] = -1, np.inf
    return idx.astype(np.int32), sqd


def boundary_ties(sqd_k1: np.ndarray, k: int) -> np.ndarray:
    """Per query: the K-th and the (K+1)-th distance are equal (a tie that the index has to break)."""
    return np.isfinite(sqd_k1[:, k - 1]) & (sqd_k1[:, k - 1] == sqd_k1[:, k])


# ------------------------------------------------------------------------------------------------ kNN maps
def lattice(shape, spacing=0.125, origin=(0.0, 0.0, 0.0)) -> np.ndarray:
    """Points of an axis-aligned lattice (spacing and origin exactly representable: every coordinate is exact)."""
    g = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), -1).reshape(-1, 3)
    return cloud(np.asarray(origin, np.float64) + g * spacing)


def lattice_queries(shape, spacing=0.125, origin=(0.0, 0.0, 0.0), rng=None, n=600) -> np.ndarray:
    """Queries at interior lattice points and at half-steps (body centres, face centres): exact equidistant neighbours."""
    rng = np.random.default_rng(0) if rng is None else rng
    lo, hi = np.array([2, 2, 2]), np.array(shape) - 3
    base = rng.integers(lo, np.maximum(hi, lo + 1), (n, 3)).astype(np.float64)
    half = np.zeros((n, 3))
    kind = np.arange(n) % 3  # 0: lattice point, 1: body centre, 2: face centre
    half[kind == 1] = 0.5
    half[kind == 2, :2] = 0.5
    return cloud(np.asarray(origin) + (base + half) * spacing)


def duplicated(base: np.ndarray, rng, lo=2, hi=40):
    """Every point repeated lo..hi times, then shuffled.  Returns (map, number of copies per base point)."""
    reps = rng.integers(lo, hi + 1, base.shape[0])
    m = np.repeat(base, reps, axis=0)
    return np.ascontiguousarray(m[rng.permutation(m.shape[0])]), reps


def dense_cell(rng, n_dense=3200, cell=0.5, n_background=20000):
    """n_dense points inside the one cell [0, cell)^3 plus a sparse background: a ring-1 run of many TMA tiles."""
    d = rng.uniform(0.02 * cell, 0.98 * cell, (n_dense, 3))
    b = rng.uniform(-5, 5, (n_background, 3))
    m = cloud(np.concatenate([d, b]))
    return np.ascontiguousarray(m[rng.permutation(m.shape[0])])


def cell_counts(map_: np.ndarray, cell: float) -> np.ndarray:
    """Number of map points in each occupied cell (cell index floor(p * (1 / cell)) in float, as the grid computes it)."""
    inv = np.float32(1.0) / np.float32(cell)
    c = np.floor(map_[:, :3].astype(np.float32) * inv).astype(np.int64)
    _, cnt = np.unique(c, axis=0, return_counts=True)
    return cnt


def grid_level(map_: np.ndarray, cell: float) -> tuple[int, float]:
    """(level, cell edge) of the dense grid a map is built on: the edge doubles until the bounding box fits the capacity
    (16 cells per point, between 2^22 and 2^28 cells)."""
    m = map_.shape[0]
    cap = min(max(16 * max(m, 1), 1 << 22), 1 << 28)
    fin = np.all(np.isfinite(map_[:, :3]), axis=1)
    lo, hi = map_[fin, :3].min(0), map_[fin, :3].max(0)
    c = np.float32(cell)
    for level in range(101):
        inv = np.float32(1.0) / c
        a, b = np.floor(lo * inv).astype(np.int64), np.floor(hi * inv).astype(np.int64)
        n = b - a + 1
        if n[0] * n[1] <= cap and n[0] * n[1] * n[2] <= cap:
            return level, float(c)
        c = np.float32(c * 2)
    raise AssertionError("grid does not fit")


def wide_ball_line(cell=0.002, length=20.0):
    """A straight line of points along y every `cell` metres: with cell 0.002 the grid is 1 x 10001 x 1 cells."""
    n = int(round(length / cell)) + 1
    y = np.arange(n) * cell
    return cloud(np.stack([np.zeros(n), y, np.zeros(n)], 1))


def wide_ball_queries(rng, n=256):
    """Queries 0.3-4 m off the middle of the line (y in 6..14 m), in x or in z: their 5 m ball spans > 4096 cell rows."""
    off = rng.uniform(0.3, 4.0, n)
    y = rng.uniform(6.0, 14.0, n)
    in_x = rng.random(n) < 0.5
    x = np.where(in_x, off, 0.0)
    z = np.where(in_x, 0.0, -off)
    return cloud(np.stack([x, y, z], 1))


# ------------------------------------------------------------------------------------------------ matcher maps
def coplanar_patches(rotated: bool, spacing=0.125, n=24, rng=None) -> np.ndarray:
    """Three families of planar lattice patches (floor z = 0.5, wall x = 6.25, wall y = -5.75), each lattice-exact;
    with rotated the whole map is turned about z by 30 degrees (then the walls are only nearly planar in float)."""
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2) * spacing
    floor = np.stack([g[:, 0] - 1.5, g[:, 1] - 1.5, np.full(len(g), 0.5)], 1)
    wall_x = np.stack([np.full(len(g), 6.25), g[:, 0] - 1.5, g[:, 1] + 0.25], 1)
    wall_y = np.stack([g[:, 0] - 1.5, np.full(len(g), -5.75), g[:, 1] + 0.25], 1)
    xyz = np.concatenate([floor, wall_x, wall_y])
    if rotated:
        xyz = xyz @ rot_z(math.pi / 6).T
    return cloud(xyz)


def rods(spacing=0.125, length=48, sep=1.0, grid=4) -> np.ndarray:
    """Straight rows of points along x, y and z (grid x grid rods per direction, sep apart): collinear neighbour sets."""
    t = np.arange(length) * spacing - length * spacing / 2
    out = []
    for a in range(grid):
        for b in range(grid):
            u, v = (a - grid / 2) * sep + 0.25, (b - grid / 2) * sep + 0.25
            out.append(np.stack([t, np.full_like(t, u), np.full_like(t, v + 10.0)], 1))
            out.append(np.stack([np.full_like(t, u + 10.0), t, np.full_like(t, v)], 1))
            out.append(np.stack([np.full_like(t, u - 10.0), np.full_like(t, v), t], 1))
    return cloud(np.concatenate(out))


def near(map_: np.ndarray, rng, n: int, jitter: float) -> np.ndarray:
    """n queries at map points (with replacement) moved by a uniform jitter of +-jitter per axis."""
    sel = map_[rng.integers(0, map_.shape[0], n), :3].astype(np.float64)
    return cloud(sel + rng.uniform(-jitter, jitter, sel.shape))


def neighbour_rank(map_: np.ndarray, nn: np.ndarray, tol: float = 1e-9) -> np.ndarray:
    """Rank of the centred neighbour coordinates of every row of nn (float64)."""
    P = map_[nn, :3].astype(np.float64)
    C = P - P.mean(1, keepdims=True)
    s = np.linalg.svd(C, compute_uv=False)
    scale = np.maximum(np.abs(P).max(axis=(1, 2)), 1.0)
    return (s > tol * scale[:, None]).sum(1)


def scatter_is_diagonal(map_: np.ndarray, nn: np.ndarray) -> np.ndarray:
    """The line fit's scatter matrix of every neighbour set is exactly diagonal (float32 centring, as the fit does)."""
    P = map_[nn, :3].astype(np.float32)
    C = P - P.mean(1, keepdims=True, dtype=np.float32)
    S = np.einsum("nki,nkj->nij", C.astype(np.float64), C.astype(np.float64))
    off = S[:, [0, 0, 1], [1, 2, 2]]
    return np.all(off == 0.0, axis=1)


def plane_residual_zero(map_: np.ndarray, nn: np.ndarray, coeffs: np.ndarray) -> np.ndarray:
    """Every neighbour lies exactly on the fitted plane n . p + d = 0 (coeffs = [n, d] per row, float64)."""
    P = map_[nn, :3].astype(np.float64)
    r = np.einsum("nki,ni->nk", P, coeffs[:, :3]) + coeffs[:, 3:4]
    return np.all(r == 0.0, axis=1)


# ------------------------------------------------------------------------------------------------ voxel filters
def heavy_voxel_cloud(rng, n=2049, leaf=0.4) -> np.ndarray:
    """A cloud that puts most of its points in a handful of voxels (and the rest in many), intensity 0..63."""
    hot = rng.integers(0, 6, n)
    centres = (np.arange(6)[:, None] * np.array([1.0, 0.5, 0.25]) - 1.0) * leaf * 3
    xyz = centres[hot] + rng.uniform(0.05 * leaf, 0.95 * leaf, (n, 3))
    cold = rng.random(n) < 0.1
    xyz[cold] = rng.uniform(-4, 4, (int(cold.sum()), 3))
    return cloud(xyz, rng.integers(0, 64, n))


def voxel_face_cloud(rng, leaf: float, n=3000, kmax=20) -> np.ndarray:
    """Points whose coordinates are float(k) * leaf (k in -kmax..kmax), i.e. exactly on voxel faces, mixed with points
    that have only one or two such coordinates."""
    k = rng.integers(-kmax, kmax + 1, (n, 3)).astype(np.float32)
    xyz = k * np.float32(leaf)
    free = rng.random((n, 3)) < 0.3
    xyz[free] = rng.uniform(-kmax * leaf, kmax * leaf, int(free.sum())).astype(np.float32)
    return cloud(xyz, rng.integers(0, 64, n))


def index_space_cloud(rng, n: int, span: int, leaf=1.0) -> np.ndarray:
    """Points whose bounding box is span x span x 1 voxels at leaf 1.0: (span - 1) * leaf apart in x and y.
    span 46340 fits PCL's int32 index space (46340^2 < 2^31), span 46341 does not."""
    assert n >= 2
    ext = (span - 1) * leaf
    xyz = np.empty((n, 3))
    xyz[:, :2] = rng.uniform(0, ext, (n, 2))
    xyz[n // 10:, :2] = np.floor(rng.uniform(0, 8, (n - n // 10, 2))) * (ext / 8)  # most points share 64 voxels
    xyz[:, 2] = rng.uniform(0.1, 0.9, n) * leaf
    xyz[0, :2], xyz[1, :2] = 0.0, ext
    return cloud(xyz, rng.integers(0, 64, n))


def voxel_index_extent(pts: np.ndarray, leaf: float) -> int:
    """dx * dy * dz of PCL's VoxelGrid over the finite points (float arithmetic of applyFilter)."""
    p = pts[np.all(np.isfinite(pts[:, :3]), axis=1), :3].astype(np.float32)
    inv = np.float32(1.0) / np.float32(leaf)
    d = ((p.max(0) - p.min(0)) * inv).astype(np.int64) + 1
    return int(d[0] * d[1] * d[2])


# ------------------------------------------------------------------------------------------------ extraction
def rings_cloud(lengths, rng, pattern=None):
    """One ring per entry of `lengths`, scan_end - scan_start = length (5 leading and 6 trailing points as ScanInfo
    leaves them).  Default: a noisy circle with steps (corners and flats).  pattern: an exactly representable repeating
    sequence of radii (multiples of 1/64) on an axis-aligned zig-zag, so that curvature values repeat exactly."""
    pts, ss, se = [], [], []
    off = 0
    for r, L in enumerate(lengths):
        m = L + 11
        if pattern is None:
            a = np.linspace(0, 2 * np.pi, m, endpoint=False)
            rad = 8.0 + np.where((np.arange(m) // 37) % 3 == 0, 1.5, 0.0) + rng.normal(0, 0.02, m)
            xyz = np.stack([rad * np.cos(a), rad * np.sin(a), np.full(m, 0.1 * r)], 1)
        else:
            p = np.asarray(pattern, np.float64)
            x = np.arange(m) / 64.0 * 4
            y = p[np.arange(m) % len(p)]
            xyz = np.stack([x, y, np.full(m, r / 64.0)], 1)
        pts.append(cloud(xyz, np.full(m, r, np.float32)))
        ss.append(off + 5)
        se.append(off + m - 6)
        off += m
    return np.ascontiguousarray(np.concatenate(pts)), np.array(ss, np.int32), np.array(se, np.int32)


def curvature_f32(pts: np.ndarray, i: int) -> np.float32:
    """extractCloud's curvature of point i (float32, left-to-right sum of the 11-point stencil)."""
    s = np.zeros(3, np.float32)
    for k in range(-5, 6):
        c = np.float32(-10.0) if k == 0 else np.float32(1.0)
        s = (s + c * pts[i + k, :3]).astype(np.float32)
    return np.float32(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])


# ------------------------------------------------------------------------------------------------ normal equations
def normal_eq_fsum(types, points, coeffs, sqrt_info, huber_a, x7, factor_eval, huber):
    """Loss-corrected normal equations of map factors from per-row residuals and Jacobians, each entry an exactly rounded
    sum (math.fsum).  Ceres' Corrector for HuberLoss scales J and r by sqrt(rho') (rho'' <= 0), so
    H_ab = sum rho'_i J_ia J_ib, g_a = sum rho'_i J_ia r_i, cost = 1/2 sum rho_i.  Also returns the sums of the absolute
    terms, which scale the rounding error bound of any other summation order.
    factor_eval(kind, point, coeffs, sqrt_info, x7) -> (r, J[7...]); huber(a, s) -> (rho, rho')."""
    n = len(types)
    HT = [[[] for _ in range(6)] for _ in range(6)]
    gT = [[] for _ in range(6)]
    cT = []
    for i in range(n):
        kind = 0 if types[i] == ord("s") else 1
        r, J = factor_eval(kind, points[i], coeffs[i], sqrt_info, x7)
        s = r[0] * r[0]
        rho, rho1 = huber(huber_a, s) if huber_a > 0 else (s, 1.0)
        cT.append(rho)
        for a in range(6):
            gT[a].append(rho1 * J[a] * r[0])
            for b in range(6):
                HT[a][b].append(rho1 * J[a] * J[b])
    H = np.array([[math.fsum(HT[a][b]) for b in range(6)] for a in range(6)])
    Habs = np.array([[math.fsum(abs(t) for t in HT[a][b]) for b in range(6)] for a in range(6)])
    g = np.array([math.fsum(t) for t in gT])
    gabs = np.array([math.fsum(abs(t) for t in tt) for tt in gT])
    return H, g, 0.5 * math.fsum(cT), Habs, gabs, 0.5 * math.fsum(abs(t) for t in cT)


def sum_error_bound(n: int, abs_sum):
    """|computed - exact| <= 16 (n + 10) 2^-53 sum |terms|: a recursive or blocked summation of n double products,
    with slack for the products and the per-block partial sums."""
    return 16.0 * (n + 10) * 2.0 ** -53 * np.asarray(abs_sum)
