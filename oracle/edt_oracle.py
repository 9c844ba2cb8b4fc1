"""The exact Euclidean distance transform of an occupancy image, in numpy: what pqp_bounds_set_occupancy computes on
the GPU (include/pqp_bounds.h) and what sharedmap.DistanceMap computes with scipy / OpenCV.

    d2(i, j) = min over obstacle cells (i', j') of (i - i')^2 + (j - j')^2     (exact, integer)
    layer    = float32(sqrt(float64(d2))) * float32(resolution)

A cell is an obstacle when its value is <= obstacle_max. An image without any obstacle gives float32(2^64) *
float32(resolution) per cell, OpenCV's value for that case (scipy's result there is not a distance).

`transform` is the separable algorithm (integer column pass, then the lower envelope of parabolas per row, Meijster
et al. 2000) vectorised over columns resp. rows; `brute_force` is the O(cells^2) definition for small grids.
"""
import numpy as np

NO_OBSTACLE = np.float32(2.0 ** 64)


def obstacles(img, obstacle_max=0):
    return np.asarray(img).astype(np.int64) <= int(obstacle_max)


def layer_from_d2(d2, res, any_obstacle=True):
    if not any_obstacle:
        return np.full(np.shape(d2), NO_OBSTACLE * np.float32(res), dtype=np.float32)
    return np.sqrt(np.asarray(d2, dtype=np.float64)).astype(np.float32) * np.float32(res)


def column_distance(obst):
    """g(i, j): distance along column j to its nearest obstacle, rows + cols where the column has none."""
    rows, cols = obst.shape
    inf = rows + cols
    g = np.empty((rows, cols), dtype=np.int64)
    d = np.full(cols, inf, dtype=np.int64)
    for i in range(rows):
        d = np.where(obst[i], 0, np.minimum(d + 1, inf))
        g[i] = d
    d = np.full(cols, inf, dtype=np.int64)
    for i in range(rows - 1, -1, -1):
        d = np.where(g[i] == 0, 0, np.minimum(d + 1, inf))
        g[i] = np.minimum(g[i], d)
    return g


def row_envelope(g):
    """min over j' of (j - j')^2 + g(i, j')^2 per row, from the lower envelope of the parabolas; all rows at once."""
    R, cols = g.shape
    f = g.astype(np.int64) ** 2
    ar = np.arange(R)
    s = np.zeros((R, cols), dtype=np.int64)   # vertex of envelope parabola k
    t = np.zeros((R, cols), dtype=np.int64)   # first column where parabola k is the lowest
    q = np.zeros(R, dtype=np.int64)           # index of the last parabola; -1: envelope empty
    for u in range(1, cols):
        fu = f[:, u]
        while True:
            qq = np.maximum(q, 0)
            tq, sq = t[ar, qq], s[ar, qq]
            pop = (q >= 0) & ((tq - sq) ** 2 + f[ar, sq] > (tq - u) ** 2 + fu)
            if not pop.any():
                break
            q = q - pop
        empty = q < 0
        sq = s[ar, np.maximum(q, 0)]
        # the first column where u is strictly lower than the last parabola: 1 + floor(num / den)
        w = 1 + np.floor_divide(u * u - sq * sq + fu - f[ar, sq], 2 * (u - sq))
        push = ~empty & (w < cols)
        q = np.where(push, q + 1, np.where(empty, 0, q))
        s[ar[push], q[push]] = u
        t[ar[push], q[push]] = w[push]
        s[empty, 0] = u
        t[empty, 0] = 0
    # column -> envelope parabola: scatter each parabola's index at its first column, running maximum along the row
    k_of = np.zeros((R, cols), dtype=np.int64)
    n = q + 1
    kk = np.arange(cols)[None, :]
    live = kk < n[:, None]
    rr, ks = np.nonzero(live)
    k_of[rr, t[rr, ks]] = ks
    k_of = np.maximum.accumulate(k_of, axis=1)
    sv = s[ar[:, None], k_of]
    return (kk - sv) ** 2 + f[ar[:, None], sv]


def transform(img, res, obstacle_max=0):
    """-> (d2 int64 [rows, cols], layer float32 [rows, cols]); d2 is undefined (rows + cols)^2 without obstacles."""
    obst = obstacles(img, obstacle_max)
    d2 = row_envelope(column_distance(obst))
    return d2, layer_from_d2(d2, res, bool(obst.any()))


def brute_force(img, res, obstacle_max=0):
    """The definition, O(cells^2): -> (d2, layer) as `transform`; d2 is None without obstacles."""
    obst = obstacles(img, obstacle_max)
    rows, cols = obst.shape
    oi, oj = np.nonzero(obst)
    if len(oi) == 0:
        return None, layer_from_d2(np.zeros((rows, cols)), res, False)
    ii, jj = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    d2 = ((ii[..., None] - oi) ** 2 + (jj[..., None] - oj) ** 2).min(axis=-1)
    return d2, layer_from_d2(d2, res)
