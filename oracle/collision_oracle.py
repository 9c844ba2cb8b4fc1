"""collision_oracle.py — CPU restatement (numpy, FP64) of the reference's footprint collision check. TEST
INFRASTRUCTURE: imported only by tests/ and bench_collision.py; the product path is the CUDA kernel
collision_check_kernel in path_optimizer_2_b200/csrc/pqp_bounds.cu and never calls this.

PARITY UNPINNED: the reference never calls CollisionChecker and has no test for it, so this restatement is checked
against closed-form cases (tests/test_collision.py: the circle table, wall sweeps), not against reference output.

Follows, relative to /root/reference/:
  car_geometry            src/tools/car_geometry.cpp:10-55 (CarGeometry constructor, setCircles)
  local2global            src/tools/tools.cpp:50-55
  state_free_exact        src/tools/collision_checker.cpp:17-39 (isSingleStateCollisionFree)
  state_free_improved     src/tools/collision_checker.cpp:41-59 (isSingleStateCollisionFreeImproved)
  CollisionChecker(map)   src/tools/collision_checker.cpp:9-15: CarGeometry(car_width, fabs(rear_length), front_length)
over bounds_oracle.map_distance (Map::getObstacleDistance, src/tools/Map.cpp:16-22).
"""
import math

import numpy as np

from oracle.bounds_oracle import CAR_WIDTH, FRONT_LENGTH, REAR_LENGTH, map_distance

CIRCLE_NAMES = ("rr", "rl", "fr", "fl", "fm", "rm")


def car_geometry(width=CAR_WIDTH, back_length=abs(REAR_LENGTH), front_length=FRONT_LENGTH):
    """-> (bounding circle (x, y, r), the six circles [(x, y, r)] in CIRCLE_NAMES order) in the rear-axle frame."""
    length = front_length + back_length
    fl, fr = (front_length, width / 2.0), (front_length, -width / 2.0)
    rl, rr = (-back_length, width / 2.0), (-back_length, -width / 2.0)
    bx = (front_length - back_length) / 2.0
    bounding = (bx, 0.0, math.sqrt(math.pow(length / 2, 2) + math.pow(width / 2, 2)))
    shift = width / 4.0
    small = math.sqrt(2 * math.pow(shift, 2))
    large = math.sqrt(math.pow(width, 2) + math.pow((length - width) / 2.0, 2)) / 2
    circles = [(rr[0] + shift, rr[1] + shift, small), (rl[0] + shift, rl[1] - shift, small),
               (fr[0] - shift, fr[1] + shift, small), (fl[0] - shift, fl[1] - shift, small),
               (bx + (length - width) / 4, 0.0, large), (bx - (length - width) / 4, 0.0, large)]
    return bounding, circles


def local2global(x, y, heading, cx, cy):
    """The point (cx, cy) of the car frame at the pose (x, y, heading) in the map frame."""
    c, s = np.cos(heading), np.sin(heading)
    return cx * c - cy * s + x, cx * s + cy * c + y


def inside(dist, res, x, y, center=(0.0, 0.0)):
    """grid_map isInside: strictly inside the map's rectangle (False for NaN)."""
    rows, cols = dist.shape
    with np.errstate(invalid="ignore"):
        return (np.abs(x - center[0]) < 0.5 * rows * res) & (np.abs(y - center[1]) < 0.5 * cols * res)


def _lookups(dist, res, x, y, heading, geometry, center):
    """(inside, distance) of the bounding circle and of each of the six circles: arrays [7, ...]."""
    bounding, circles = geometry
    ins, d = [], []
    for cx, cy, _ in [bounding] + circles:
        gx, gy = local2global(x, y, heading, cx, cy)
        ins.append(inside(dist, res, gx, gy, center))
        d.append(map_distance(dist, res, gx, gy, *center))
    return np.array(ins), np.array(d)


def state_free_exact(dist, res, x, y, heading, geometry=None, center=(0.0, 0.0)):
    """isSingleStateCollisionFree over arrays of poses: every circle inside and not closer than its radius."""
    geometry = geometry or car_geometry()
    ins, d = _lookups(dist, res, np.asarray(x, float), np.asarray(y, float), np.asarray(heading, float), geometry,
                      center)
    r = np.array([c[2] for c in geometry[1]]).reshape((6,) + (1,) * (d.ndim - 1))
    with np.errstate(invalid="ignore"):
        return np.all(ins[1:] & ~(d[1:] < r), axis=0)


def state_free_improved(dist, res, x, y, heading, geometry=None, center=(0.0, 0.0)):
    """isSingleStateCollisionFreeImproved over arrays of poses -> (free, clearance): free when the bounding circle's
    centre is inside and its distance is not below R, else the exact test; clearance = min over the six circles of
    d_i - r_i, NaN terms skipped."""
    geometry = geometry or car_geometry()
    ins, d = _lookups(dist, res, np.asarray(x, float), np.asarray(y, float), np.asarray(heading, float), geometry,
                      center)
    R = geometry[0][2]
    r = np.array([c[2] for c in geometry[1]]).reshape((6,) + (1,) * (d.ndim - 1))
    with np.errstate(invalid="ignore"):
        exact = np.all(ins[1:] & ~(d[1:] < r), axis=0)
        free = ins[0] & (~(d[0] < R) | exact)
    return free, np.fmin.reduce(d[1:] - r, axis=0)


def margins(dist, res, x, y, heading, geometry=None, center=(0.0, 0.0)):
    """d - r of the bounding circle and of each of the six circles: [7, ...]."""
    geometry = geometry or car_geometry()
    _, d = _lookups(dist, res, np.asarray(x, float), np.asarray(y, float), np.asarray(heading, float), geometry, center)
    r = np.array([c[2] for c in [geometry[0]] + geometry[1]]).reshape((7,) + (1,) * (d.ndim - 1))
    return d - r


def check(dist, res, poses, n, *, geometry=None, center=(0.0, 0.0)):
    """poses [B, rows >= 3, n_max] (x, y, heading in rows 0-2), n [B] clamped to [0, n_max] -> (first_hit [B],
    state_free [B, n_max] uint8, clearance [B, n_max]; both 0 at i >= n[b])."""
    poses = np.asarray(poses, dtype=np.float64)
    B, _, n_max = poses.shape
    nb = np.clip(np.asarray(n, dtype=np.int64), 0, n_max)
    free, clear = state_free_improved(dist, res, poses[:, 0], poses[:, 1], poses[:, 2], geometry, center)
    valid = np.arange(n_max)[None, :] < nb[:, None]
    free = free & valid
    clear = np.where(valid, clear, 0.0)
    hit = np.array([int(np.argmax(~free[b, :nb[b]])) if not free[b, :nb[b]].all() else int(nb[b]) for b in range(B)],
                   dtype=np.int32)
    return hit, free.astype(np.uint8), clear
