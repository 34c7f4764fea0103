"""A synthetic street drive for the association's slab path, and numpy restatements of its root counts and slab plan.

street_scans: lidar-like scans of a straight street (two facades, the ground, poles and clutter) along a trajectory
that crosses the origin -- so root voxels on both sides of the key's 2^18 bias fall in different slabs -- and that ends
by driving the first stretch again, so that one slab holds points of frames far apart in time."""
import numpy as np

import assoc_ref
import scenes

HALF_WIDTH = 8.0      # facades at y = +-8 m
POLE_Y = 6.0          # poles at y = +-6 m, every 12 m
SENSOR_H = 1.8        # sensor above the ground


def _surface(rng, n, p, rng_m):
    """n world points of the street around the sensor position p, within rng_m metres along x"""
    kind = rng.choice(5, n, p=[0.3, 0.3, 0.25, 0.05, 0.1])
    x = p[0] + rng.uniform(-rng_m, rng_m, n)
    w = np.zeros((n, 3))
    m = kind < 2                                    # the two facades, 0 to 12 m high
    w[m] = np.stack([x[m], np.where(kind[m] == 0, -HALF_WIDTH, HALF_WIDTH), rng.uniform(0.0, 12.0, m.sum())], axis=1)
    m = kind == 2                                   # the ground
    w[m] = np.stack([x[m], rng.uniform(-HALF_WIDTH, HALF_WIDTH, m.sum()), np.zeros(m.sum())], axis=1)
    m = kind == 3                                   # poles: radius 0.15 m, 5 m high
    px = np.round(x[m] / 12.0) * 12.0
    a = rng.uniform(0, 2 * np.pi, m.sum())
    side = np.where(rng.random(m.sum()) < 0.5, -POLE_Y, POLE_Y)
    w[m] = np.stack([px + 0.15 * np.cos(a), side + 0.15 * np.sin(a), rng.uniform(0.0, 5.0, m.sum())], axis=1)
    m = kind == 4                                   # clutter: blobs on the pavement
    cx = np.round(x[m] / 7.0) * 7.0 + 1.3
    w[m] = np.stack([cx, rng.choice([-4.5, 3.5], m.sum()), np.full(m.sum(), 0.8)], axis=1) + rng.normal(0, 0.5, (m.sum(), 3))
    return w


def street_scans(n_forward=24, n_revisit=6, pts_per_scan=4000, seed=11, step=4.0, rng_m=20.0):
    """-> (points_body n x 3 float64 rounded to float32, frames n int32, poses [(R, p)] at which to cut: the noisy
    initial poses, pose 0 exact). The forward drive runs along x from -(n_forward - 1) step / 2 through the origin; the
    revisit drives the first n_revisit forward positions again in the other lane, facing back."""
    rng = np.random.default_rng(seed)
    x0 = -(n_forward - 1) * step / 2
    poses = [(scenes.exp_so3(np.array([0.0, 0.0, 0.01 * np.sin(i)])), np.array([x0 + step * i, -2.0, SENSOR_H]))
             for i in range(n_forward)]
    poses += [(scenes.exp_so3(np.array([0.0, 0.0, np.pi + 0.01 * i])), np.array([x0 + step * i + 1.0, 2.0, SENSOR_H]))
              for i in range(n_revisit)]
    pts, frs = [], []
    for i, (R, p) in enumerate(poses):
        w = _surface(rng, pts_per_scan, p, rng_m) + rng.normal(0, 0.01, (pts_per_scan, 3))
        pts.append(((w - p) @ R).astype(np.float32).astype(np.float64))  # R^T (w - p)
        frs.append(np.full(pts_per_scan, i, dtype=np.int32))
    noisy = [(R @ scenes.exp_so3(rng.normal(0, 0.002, 3)), p + rng.normal(0, 0.01, 3)) for R, p in poses]
    noisy[0] = poses[0]
    return np.concatenate(pts), np.concatenate(frs), noisy


def root_counts(points_body, frames, poses, voxel_size):
    """points of every root voxel, in ascending key order (x, then y, then z) -> int64 counts"""
    R = np.stack([r for r, _ in poses])
    t = np.stack([p for _, p in poses])
    world = np.einsum("nij,nj->ni", R[frames], points_body) + t[frames]
    key = assoc_ref.root_index(world, voxel_size)
    _, counts = np.unique(key, axis=0, return_counts=True)  # rows sorted lexicographically: the key order
    return counts.astype(np.int64)


def greedy_slabs(counts, cap):
    """slab count of the plan: roots in ascending key order, a slab closed before the root that would take it past
    cap points; None when one root alone holds more than cap points"""
    if counts.max() > cap:
        return None
    slabs, cur = 1, 0
    for c in counts:
        if cur + c > cap:
            slabs, cur = slabs + 1, 0
        cur += c
    return slabs
