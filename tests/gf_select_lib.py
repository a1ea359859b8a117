"""Good-feature selection (ActiveFeatureSelection::goodFeatureMatching, lidar_mapper.h:229-573) stated in plain Python, and scans
that drive the selection to its edges.

`select` restates the reference's four loops with its own data structures: the candidate pool is a list that loses the
erased element (`all_feature_idx.erase`), `feature_visited` is erased alongside it, fps keeps a float32 min-distance table
and the greedy round keeps every pushed candidate like the priority queue does.  Only what the reference leaves to chance is
made explicit, as the oracle does it (oracle/orc_gf.hpp): PCG32 with multiply-shift range reduction instead of
mt19937(random_device), no wall-clock cap, fps stops once every point is visited, and priority-queue ties go to the candidate
pushed first.  It shares no code with the oracle, so agreeing with `orc.good_features` pins the oracle's Fenwick-free
restatement (and through it the kernel) to the reference's loops.  It also reports which edges a run went through.

Every generator returns a dict: kind ('s' / 'c'), scan (n x 4 float32), map, pose7 and, where it matters, cov6 / seed.
"""
import functools
import math

import numpy as np

import oracle_lib as orc
import synthetic as syn

MASK64 = (1 << 64) - 1
MAX_RANDOM_QUEUE_TIME = 20  # lidar_mapper.h:83
BATCH = 32                  # candidates one draw batch of the device's greedy round holds
IDENTITY7 = np.array([0, 0, 0, 0, 0, 0, 1], np.float64)


# ------------------------------------------------------------------------------------------------ PCG32 and the uniform draw
class Pcg32:
    def __init__(self, seed):
        self.s = (int(seed) * 0x9E3779B97F4A7C15 + 0xDA3E39CB94B95BDB) & MASK64
        self.next()

    def next(self):
        old = self.s
        self.s = (old * 6364136223846793005 + 1442695040888963407) & MASK64
        xorshifted = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        return ((xorshifted >> rot) | (xorshifted << ((32 - rot) & 31))) & 0xFFFFFFFF

    def uniform(self, lo, hi):
        """geneRandUniform(lo, hi): an integer in [lo, hi] by multiply-shift range reduction."""
        return lo + ((self.next() * (hi - lo + 1)) >> 32)


def first_draw(seed, n):
    """Index of the first draw of a selection over n features (fps: the start point)."""
    return Pcg32(seed).uniform(0, n - 1)


# ------------------------------------------------------------------------------------------------ log det(M) by Cholesky
def logdet(M):
    """common::logDet(M, true) as the oracle's logdet_chol computes it: column-wise Cholesky, then 2 * sum log diag."""
    L = list(M)
    for j in range(6):
        d = L[j * 6 + j]
        for k in range(j):
            d -= L[j * 6 + k] * L[j * 6 + k]
        if not d > 0.0:
            return -math.inf
        d = math.sqrt(d)
        L[j * 6 + j] = d
        for i in range(j + 1, 6):
            s = L[i * 6 + j]
            for k in range(j):
                s -= L[i * 6 + k] * L[j * 6 + k]
            L[i * 6 + j] = s / d
    s = 0.0
    for i in range(6):
        s += math.log(L[i * 6 + i])
    return 2.0 * s


def _add_outer(H, j):
    for a in range(6):
        for b in range(6):
            H[a * 6 + b] += j[a] * j[b]


def num_use_of(n, ratio):
    return int(n * ratio)  # static_cast<size_t>(num_all_features * gf_ratio), :248


def subset_of(n, ratio):
    """size_rnd_subset of the greedy round (:474)."""
    k = num_use_of(n, ratio)
    return int(1.0 * n / k) if k > 0 else None


# ------------------------------------------------------------------------------------------------ goodFeatureMatching's loops
def select(method, ratio, seed, matched, jaco, xyz):
    """Returns (sel, H 6x6, info).  method 0 wo_gf, 1 rnd, 2 fps, 3 gd; matched[n], jaco (n, 6), xyz (n, >= 3) float32."""
    matched = [bool(m) for m in np.asarray(matched)]
    rows = [tuple(r) for r in np.asarray(jaco, np.float64).tolist()]
    n = len(matched)
    H = [1e-6 if i % 7 == 0 else 0.0 for i in range(36)]  # sub_mat_H = I * 1e-6 (:504, :519)
    num_use = num_use_of(n, ratio)
    rng = Pcg32(seed)
    pool = list(range(n))          # all_feature_idx
    visited = [-1] * n             # feature_visited
    sel = []
    info = {"exit": None, "erased": 0, "ties": [], "fallback": 0, "start": None, "fps_ties": [], "empty_mid_round": False,
            "max_heap": 0}
    if method == 0:  # wo_gf (:257-299)
        for q in range(n):
            if matched[q]:
                _add_outer(H, rows[q])
                sel.append(q)
        info["exit"] = "all"
    elif method == 1:  # rnd (:300-352)
        while True:
            if len(sel) >= num_use or len(pool) == 0:
                info["exit"] = "quota" if len(sel) >= num_use else "empty"
                break
            j = rng.uniform(0, len(pool) - 1)
            q = pool[j]
            if matched[q]:
                _add_outer(H, rows[q])
                sel.append(q)
            del pool[j]
    elif method == 2 and n > 0:  # fps (:353-457)
        xyz = np.ascontiguousarray(np.asarray(xyz)[:, :3], np.float32)
        x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        k = rng.uniform(0, len(pool) - 1)
        vis = np.zeros(n, bool)
        vis[k] = True
        cnt_visited = 1
        old = k
        info["start"] = k
        if matched[k]:
            sel.append(k)  # selected, never added to sub_mat_H (:383-387)
        dist = np.full(n, 1e5, np.float32)
        while True:
            # the reference's exits are the quota, an empty pool (never: fps erases nothing) and its time cap; without the cap
            # the loop stops once every point has been visited (the condition commented out at :396-399)
            if len(sel) >= num_use or len(pool) == 0 or cnt_visited >= n:
                info["exit"] = "quota" if len(sel) >= num_use else "visited"
                break
            dx, dy, dz = x[old] - x, y[old] - y, z[old] - z
            d = np.sqrt((dx * dx + dy * dy) + dz * dz)
            d2 = np.where(dist < d, dist, d)  # std::min(d, dist[j]) is (dist[j] < d) ? dist[j] : d: a NaN d stays NaN
            unv = ~vis
            dist[unv] = d2[unv]
            ok = unv & (d2 > -1)  # best_j moves only on d2 > best_d, which a NaN never passes
            if not ok.any():
                best_j = 1  # size_t best_j = 1 (:402), visited or not
                info["fallback"] += 1
            else:
                cand = np.where(ok, d2, np.float32(-np.inf))
                best_j = int(np.argmax(cand))  # the first maximum in index order
                tied = np.flatnonzero(cand == cand[best_j])
                if tied.size > 1:
                    info["fps_ties"].append(tied)
            q = best_j
            old = q
            vis[q] = True
            cnt_visited += 1
            if matched[q]:
                _add_outer(H, rows[q])
                sel.append(q)
    elif method == 3:  # gd_fix / gd_float (:458-563)
        num_rnd_que = 0
        while True:
            if len(sel) >= num_use or len(pool) == 0:
                info["exit"] = "quota" if len(sel) >= num_use else "empty"
                break
            size_rnd_subset = int(1.0 * n / num_use)
            heap = []  # (score, idx) in push order; the top is the largest score, the first pushed among equals
            while True:
                if len(pool) == 0:
                    info["empty_mid_round"] = True
                    break
                num_rnd_que = 0
                while num_rnd_que < MAX_RANDOM_QUEUE_TIME:
                    j = rng.uniform(0, len(pool) - 1)
                    if visited[j] < len(sel):
                        visited[j] = len(sel)
                        break
                    num_rnd_que += 1
                if num_rnd_que >= MAX_RANDOM_QUEUE_TIME:
                    break
                q = pool[j]
                if not matched[q]:  # "not found constraints or outlier constraints" (:529-534)
                    del pool[j]
                    del visited[j]
                    info["erased"] += 1
                    continue
                r = rows[q]
                M = [H[a * 6 + b] + r[a] * r[b] for a in range(6) for b in range(6)]
                heap.append((logdet(M), q))
                info["max_heap"] = max(info["max_heap"], len(heap))
                if len(heap) >= size_rnd_subset:
                    top = 0
                    for p in range(1, len(heap)):
                        if heap[p][0] > heap[top][0]:
                            top = p
                    tied = [p for p in range(len(heap)) if heap[p][0] == heap[top][0]]
                    if len(tied) > 1:
                        info["ties"].append(tied)  # push positions of the candidates that share the top score
                    best = heap[top][1]
                    pos = pool.index(best)
                    _add_outer(H, rows[best])
                    del pool[pos]
                    del visited[pos]
                    sel.append(best)
                    break
            if num_rnd_que >= MAX_RANDOM_QUEUE_TIME:
                info["exit"] = "repeat"
                break
    return np.array(sel, np.int32), np.array(H).reshape(6, 6), info


# ------------------------------------------------------------------------------------------------ scans
@functools.lru_cache(maxsize=1)
def c1():
    """The 16-ring x 1024 sweep against the 50k-point submap: down-sampled surf (~4k) and corner (~1.7k) scans."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
    matched = orc.good_features("s", surf_map, sf, init, orc.GF_WO, 1.0, 0)["matched"]
    return dict(surf_map=surf_map, corner_map=corner_map, surf_scan=sf, corner_scan=cs, init=init, surf_matched=matched)


def _surf(scan, **kw):
    c = c1()
    return dict(kind="s", scan=np.ascontiguousarray(scan, np.float32), map=c["surf_map"], pose7=c["init"], **kw)


def pool_scan(n, seed=0):
    """n surf features: c1's surf scan tiled, every copy after the first moved by millimetre jitter, so most of them match."""
    sf = c1()["surf_scan"]
    rng = np.random.default_rng(seed)
    reps = -(-n // sf.shape[0])
    tiles = [sf] + [sf + np.concatenate([rng.normal(0, 1e-3, (sf.shape[0], 3)), np.zeros((sf.shape[0], 1))], 1) for _ in range(reps - 1)]
    return _surf(np.concatenate(tiles)[:n])


def prefix_scan(n):
    """The first n features of c1's surf scan (n <= its size)."""
    return _surf(c1()["surf_scan"][:n])


def tie_scan(distinct, copies, seed=0):
    """`distinct` matched surf features, each repeated exactly `copies` times in a shuffled order: equal rows, equal log dets."""
    c = c1()
    idx = np.flatnonzero(c["surf_matched"])[:: 37][:distinct]
    order = np.random.default_rng(seed).permutation(distinct * copies)
    return _surf(np.repeat(c["surf_scan"][idx], copies, axis=0)[order])


def mixed_scan(n_matched, n_far, seed=0, matched_at=()):
    """n_matched matched surf features and n_far features 1 km from the map (never matched), shuffled; the positions in
    matched_at hold matched features."""
    c = c1()
    rng = np.random.default_rng(seed)
    good = c["surf_scan"][np.flatnonzero(c["surf_matched"])[:n_matched]]
    far = c["surf_scan"][:n_far].copy()
    far[:, 0] += 1000.0
    pts = np.concatenate([good, far])
    is_good = np.r_[np.ones(n_matched, bool), np.zeros(n_far, bool)]
    order = rng.permutation(pts.shape[0])
    pts, is_good = pts[order], is_good[order]
    for p in matched_at:
        if not is_good[p]:
            g = int(np.flatnonzero(is_good)[-1])
            pts[[p, g]], is_good[[p, g]] = pts[[g, p]], is_good[[g, p]]
    return _surf(pts, is_matched=is_good)


def lattice_scan(half=20):
    """Points of the integer lattice on the plane z = -2 (row-major, (2 half + 1)^2 of them) against a dense random map of that
    plane (the plane fit n.p + 1 = 0 cannot hold a plane through the origin): integer x and y give exact float32 distances, so
    many points are equidistant from every pick."""
    rng = np.random.default_rng(5)
    g = np.arange(-half, half + 1, dtype=np.float32)
    xx, yy = np.meshgrid(g, g)
    scan = np.stack([xx.ravel(), yy.ravel(), np.full(xx.size, -2.0), np.zeros(xx.size)], 1).astype(np.float32)
    m = rng.uniform(-half - 2, half + 2, (120000, 2))
    mp = np.concatenate([m, np.full((m.shape[0], 1), -2.0), np.zeros((m.shape[0], 1))], 1).astype(np.float32)
    return dict(kind="s", scan=scan, map=mp, pose7=IDENTITY7.copy())


def nan_scan(nan_at=(137,)):
    """c1's surf scan with the points at nan_at made NaN."""
    sc = c1()["surf_scan"].copy()
    sc[list(nan_at), :3] = np.nan
    return _surf(sc, nan_at=np.array(nan_at))


def nan_tail_scan(n_finite=300, n_nan=700):
    """n_finite features of c1's surf scan (index 1 matched), then n_nan NaN points."""
    c = c1()
    fin = c["surf_scan"][:n_finite].copy()
    assert c["surf_matched"][1]
    tail = np.full((n_nan, 4), np.nan, np.float32)
    tail[:, 3] = 0
    return _surf(np.concatenate([fin, tail]), nan_at=np.arange(n_finite, n_finite + n_nan))


def nan_mixed_scan(nan_at=150):
    """mixed_scan(100, 200) (index 1 matched) with one NaN point: fps visits every finite point before the quota, and then only
    the NaN point is left."""
    c = mixed_scan(100, 200, matched_at=(1,))
    c["scan"][nan_at, :3] = np.nan
    c["is_matched"][nan_at] = False
    c["nan_at"] = np.array([nan_at])
    return c


def seed_with_first_draw(n, want, start=0):
    """The smallest seed >= start whose first draw over n features is `want` (a predicate on the index)."""
    s = start
    while not want(first_draw(s, n)):
        s += 1
    return s


def odom_corner_case():
    """Corner features for Estimator::goodFeatureMatching: every matched row is [1 0 0 0 0 0], so every candidate ties."""
    c = c1()
    return dict(kind="c", scan=c["corner_scan"], map=c["corner_map"], pivot=IDENTITY7.copy(), pose_i=c["init"], ext=IDENTITY7.copy())


def f32_triple(trace):
    """Three float32 values whose double sum, left to right, is exactly `trace` (a double)."""
    a = np.float32(trace)
    r = trace - float(a)
    b = np.float32(r)
    c = np.float32(r - float(b))
    assert (float(a) + float(b)) + float(c) == trace or (math.isinf(trace) and float(a) == trace)
    return a, b, c


def clamp_traces():
    """Traces around the sqrt_info clamp of lidar_map_factor.hpp:34,41 (sqrt(1 / trace) >= 3 -> 1): the double nearest 1/9, one
    ulp either side, the first trace above it whose sqrt(1 / trace) falls below 3, 0 and +inf."""
    t9 = 1.0 / 9.0
    above = t9
    while math.sqrt(1 / above) >= 3.0:
        above = float(np.nextafter(above, 1.0))
    return [t9, float(np.nextafter(t9, 0.0)), float(np.nextafter(t9, 1.0)), above, 0.0, math.inf]


def clamp_scan():
    """c1's surf scan with per-point covariances whose traces cycle through clamp_traces()."""
    sc = c1()["surf_scan"]
    traces = clamp_traces()
    cov6 = np.zeros((sc.shape[0], 6), np.float32)
    for i in range(sc.shape[0]):
        t = traces[i % len(traces)]
        cov6[i, 0], cov6[i, 3], cov6[i, 5] = (np.float32(t), np.float32(0), np.float32(0)) if math.isinf(t) else f32_triple(t)
    return _surf(sc, cov6=cov6, traces=traces)
