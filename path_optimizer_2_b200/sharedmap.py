"""Shared-obstacle-map workload (BASELINE configs[0] and configs[1], SURVEY.md §8d configs 1-2).

Workload synthesis only (host side, numpy): reference lines through the free space of
`tests/golden/gridmap.png`, as spline coefficients + reference states — the inputs of the
clearance-bounds kernel (include/pqp_bounds.h, `bounds.PathBounds`), whose output then feeds the
solver. What is restated from the reference here is only what produces those inputs:

  distance layer      src/test/demo.cpp:98-113  (cv2.distanceTransform(DIST_L2, MASK_PRECISE), float, * 0.2 m)
  reference spline    src/tools/spline.cpp:163-247  (natural cubic spline over arc length)
  reference states    src/data_struct/reference_path_impl.cpp:314-338, src/tools/tools.cpp:32-44

The reference line itself comes from a greedy clearance-following walk that stands in for the
reference's hybrid A* + smoother (out of scope, SURVEY.md §8).
"""
import math
import os

import numpy as np

from . import abi

RES = 0.2
SPLINE_ROWS, STATE_ROWS, BOUND_ROWS = 9, 4, 6
_MAP_PNG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "gridmap.png")


class DistanceMap:
    """grid_map "distance" layer of the demo (float32): cell (i, j) = image pixel (row i, col j),
    centred at (+Lx/2 - (i + 1/2) res, +Ly/2 - (j + 1/2) res), Lx = rows * res, Ly = cols * res."""

    def __init__(self, png_path=_MAP_PNG, dist=None, res=RES):
        self.res = res
        if dist is None:
            if not os.path.exists(png_path):
                raise FileNotFoundError(png_path)
            try:
                import cv2
                img = cv2.imread(png_path, cv2.IMREAD_GRAYSCALE)
                free = (img > 127).astype(np.uint8)  # OCCUPY = 0, FREE = 255 (demo.cpp:103-106)
                dist = cv2.distanceTransform(free, cv2.DIST_L2, cv2.DIST_MASK_PRECISE)
            except ImportError:  # same exact Euclidean transform without OpenCV
                from PIL import Image
                from scipy.ndimage import distance_transform_edt
                img = np.asarray(Image.open(png_path).convert("L"))
                dist = distance_transform_edt(img > 127)
            dist = dist.astype(np.float32) * np.float32(res)  # MatrixXf *= resolution (demo.cpp:113)
        self.dist = np.ascontiguousarray(dist, dtype=np.float32)
        self.rows, self.cols = self.dist.shape
        self.lx, self.ly = self.rows * res, self.cols * res

    def lookup(self, x, y):
        """Bilinear lookup for the walk below (the kernel has its own, pqp_bounds_core.cuh)."""
        x = np.asarray(x, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        inside = (np.abs(x) < self.lx / 2) & (np.abs(y) < self.ly / 2)
        fi = (self.lx / 2 - np.where(inside, x, 0.0)) / self.res - 0.5
        fj = (self.ly / 2 - np.where(inside, y, 0.0)) / self.res - 0.5
        i0 = np.clip(np.floor(fi).astype(np.int64), 0, self.rows - 2)
        j0 = np.clip(np.floor(fj).astype(np.int64), 0, self.cols - 2)
        ti, tj = np.clip(fi - i0, 0.0, 1.0), np.clip(fj - j0, 0.0, 1.0)
        d = self.dist
        v = (d[i0, j0] * (1 - ti) * (1 - tj) + d[i0 + 1, j0] * ti * (1 - tj) +
             d[i0, j0 + 1] * (1 - ti) * tj + d[i0 + 1, j0 + 1] * ti * tj)
        return np.where(inside, v, 0.0)


def natural_spline_rows(s, x, y):
    """Rows (abscissa; a, b, c, y of x(s); a, b, c, y of y(s)) in tk::spline's convention
    f_i(h) = ((a_i h + b_i) h + c_i) h + y_i, incl. its right-end entries (spline.cpp:241-246)."""
    from scipy.interpolate import CubicSpline
    rows = [np.asarray(s, dtype=np.float64)]
    for v in (x, y):
        cs = CubicSpline(s, v, bc_type="natural")
        k = len(s)
        a, b, c = np.zeros(k), np.zeros(k), np.zeros(k)
        a[:-1], b[:-1], c[:-1] = cs.c[0], cs.c[1], cs.c[2]
        b[0] = 0.0  # natural end: the reference's first equation is 2 b0 = 0 exactly
        c[-1] = float(cs(s[-1], 1))
        rows += [a, b, c, np.asarray(v, dtype=np.float64)]
    return np.stack(rows)


def _eval(rows, s, which):
    """value, first and second derivative of x(s) (which = 0) or y(s) (which = 1) inside the range."""
    sx = rows[0]
    a, b, c, y = rows[1 + 4 * which:5 + 4 * which]
    idx = np.clip(np.searchsorted(sx, s, side="left") - 1, 0, len(sx) - 2)
    h = s - sx[idx]
    return (((a[idx] * h + b[idx]) * h + c[idx]) * h + y[idx], (3 * a[idx] * h + 2 * b[idx]) * h + c[idx],
            6 * a[idx] * h + 2 * b[idx])


def reference_states(rows, n):
    """buildReferenceFromSpline(0.15, 0.3) (reference_path_impl.cpp:314-338): the first n states as
    (s, x, y, heading, curvature), or None when the spline is too short."""
    max_s = float(rows[0][-1])
    s_list, s = [], 0.0
    while s <= max_s and len(s_list) < n:
        s_list.append(s)
        _, dx, ddx = _eval(rows, s, 0)
        _, dy, ddy = _eval(rows, s, 1)
        k = abs(float((dx * ddy - dy * ddx) / math.pow(dx * dx + dy * dy, 1.5)))  # tools.cpp:38-44
        share = 1.0 if k > 0.2 else (0.0 if k < 0.08 else (k - 0.08) / 0.12)
        s += 0.3 - share * 0.15
    if len(s_list) < n:
        return None
    s = np.array(s_list)
    x, dx, ddx = _eval(rows, s, 0)
    y, dy, ddy = _eval(rows, s, 1)
    return s, x, y, np.arctan2(dy, dx), (dx * ddy - dy * ddx) / np.power(dx * dx + dy * dy, 1.5)


def _walk_free_line(dmap, rng, x0, y0, total, step=1.5, min_clear=1.6):
    """Walk from (x0, y0) in 1.5 m arcs, each time taking the curvature whose 6 m look-ahead keeps
    the most clearance; returns control points (s, x, y) or None when the corridor closes."""
    cand = np.linspace(-0.12, 0.12, 9)
    look = step * np.arange(1, 5)
    best_h, best_c = 0.0, -1.0
    for h in rng.uniform(-math.pi, math.pi, size=8):  # start along the most open direction
        c = float(dmap.lookup(x0 + look * math.cos(h), y0 + look * math.sin(h)).min())
        if c > best_c:
            best_h, best_c = h, c
    x, y, h, k_prev = x0, y0, best_h, 0.0
    xs, ys = [x], [y]
    for _ in range(int(math.ceil(total / step))):
        hh = h + 0.5 * cand[:, None] * look[None, :]
        px, py = x + look[None, :] * np.cos(hh), y + look[None, :] * np.sin(hh)
        score = np.minimum(dmap.lookup(px, py).min(axis=1), 2.5) - 4.0 * np.abs(cand - k_prev) - 2.0 * np.abs(cand)
        k = float(cand[int(np.argmax(score))])
        x, y = x + step * math.cos(h + 0.5 * step * k), y + step * math.sin(h + 0.5 * step * k)
        h, k_prev = h + step * k, k
        if dmap.lookup(x, y) < min_clear:
            return None
        xs.append(x)
        ys.append(y)
    xs, ys = np.array(xs), np.array(ys)
    sc = np.concatenate(([0.0], np.cumsum(np.hypot(np.diff(xs), np.diff(ys)))))
    return sc, xs, ys


class LineBatch:
    """`batch` reference lines: what ReferencePathImpl holds before updateBoundsImproved — the
    splines x_s_, y_s_ and reference_states_ — in the layout of include/pqp_bounds.h."""

    def __init__(self, batch, n, k_max):
        self.batch, self.n_max, self.k_max = batch, n, k_max
        self.spline = np.zeros((batch, SPLINE_ROWS, k_max))
        self.k = np.zeros(batch, dtype=np.int32)
        self.states = np.zeros((batch, STATE_ROWS, n))
        self.kref = np.zeros((batch, n))
        self.n = np.full(batch, n, dtype=np.int32)
        self.inst = np.zeros((batch, abi.NINST))

    def spline_rows(self, b):
        return self.spline[b, :, :int(self.k[b])]

    def to_host_batch(self, bounds, n_valid=None):
        """Solver input: knots from the states, the front/rear rows of `bounds[b][6][n]`;
        n = n_valid (the reference cuts reference_states_ at the first blocked state)."""
        knots = np.zeros((self.batch, abi.NFIELDS, self.n_max))
        knots[:, abi.F_S] = self.states[:, 0]
        knots[:, abi.F_KREF] = knots[:, abi.F_K] = self.kref
        knots[:, abi.F_B0_LB:abi.F_B1_UB + 1] = bounds[:, 0:4]
        n = self.n.copy() if n_valid is None else np.asarray(n_valid, dtype=np.int32).copy()
        return abi.HostBatch(knots, self.inst.copy(), n)

    @property
    def ref_xyh(self):
        return np.ascontiguousarray(self.states[:, 1:4])


def make_plan_inputs(batch, n=120, first=0, dmap=None, seed=11, noise=0.03, lines=None):
    """Inputs of a whole plan (include/pqp_plan.h) from the lines of `make_lines`: the line sampled about every 1 m
    with `noise` m of noise stands in for bSpline()'s samples; the start lies up to 1 m beside the line at s = 0.5
    with its heading and curvature, the target on the line 1 m before its end. `lines`: make_lines(batch, n, first,
    dmap=dmap) when already built. -> (raw_x, raw_y lists, start [B][4], target [B][3])."""
    if lines is None:
        lines = make_lines(batch, n, first=first, dmap=dmap)
    rng = np.random.default_rng(seed + first)
    raw_x, raw_y = [], []
    start, target = np.zeros((batch, 4)), np.zeros((batch, 3))
    for b in range(batch):
        rows = lines.spline_rows(b)
        end = float(rows[0, -1])
        s = np.arange(0.0, end, 1.0)
        x, dx, ddx = _eval(rows, s, 0)
        y, dy, ddy = _eval(rows, s, 1)
        raw_x.append(x + rng.normal(0, noise, len(s)))
        raw_y.append(y + rng.normal(0, noise, len(s)))
        x0, dx0, ddx0 = (float(v) for v in _eval(rows, 0.5, 0))
        y0, dy0, ddy0 = (float(v) for v in _eval(rows, 0.5, 1))
        h = math.atan2(dy0, dx0)
        off = rng.uniform(-1.0, 1.0)
        start[b] = x0 - off * math.sin(h), y0 + off * math.cos(h), h, (dx0 * ddy0 - dy0 * ddx0) / math.pow(dx0 * dx0 + dy0 * dy0, 1.5)
        xe, dxe, _ = (float(v) for v in _eval(rows, end - 1.0, 0))
        ye, dye, _ = (float(v) for v in _eval(rows, end - 1.0, 1))
        target[b] = xe, ye, math.atan2(dye, dxe)
    return raw_x, raw_y, start, target


def make_plan_points(batch, n=120, first=0, dmap=None, seed=11, spacing=(3.0, 14.0), noise=0.2):
    """Inputs of a whole plan from the reference points (pqp_plan_points): "clicked" points along the lines of
    `make_lines`, evenly spaced per path at a spacing drawn from `spacing` (m) - so that the B-spline degrees 3
    (average spacing above 10 m), 4 (above 5 m) and 5 all occur - from the line's start to its end, each moved up to
    `noise` m (normal, sigma noise / 2) sideways. Start and target are those of `make_plan_inputs`.
    -> (ref_x, ref_y lists, start [B][4], target [B][3])."""
    dmap = dmap or DistanceMap()
    lines = make_lines(batch, n, first=first, dmap=dmap)
    _, _, start, target = make_plan_inputs(batch, n, first=first, dmap=dmap, seed=seed, lines=lines)
    rng = np.random.default_rng(seed + 7919 + first)
    ref_x, ref_y = [], []
    for b in range(batch):
        rows = lines.spline_rows(b)
        end = float(rows[0, -1])
        m = max(int(round(end / rng.uniform(*spacing))), 3) + 1
        s = np.linspace(0.0, end, m)
        x, dx, _ = _eval(rows, s, 0)
        y, dy, _ = _eval(rows, s, 1)
        h = np.arctan2(dy, dx)
        off = np.clip(rng.normal(0.0, noise / 2, m), -noise, noise)
        ref_x.append(x - off * np.sin(h))
        ref_y.append(y + off * np.cos(h))
    return ref_x, ref_y, start, target


def make_lines(batch, n=120, first=0, cfg_id=2, dmap=None):
    """Lines [first, first + batch) of the shared-map config; line i depends only on (cfg_id, i)."""
    dmap = dmap or DistanceMap()
    total = 0.3 * n + 8.0
    lb = LineBatch(batch, n, int(math.ceil(total / 1.5)) + 1)
    for b in range(batch):
        rng = np.random.default_rng(cfg_id * 1_000_003 + first + b)
        for _ in range(400):
            x0 = rng.uniform(-dmap.lx / 2 + 5, dmap.lx / 2 - 5)
            y0 = rng.uniform(-dmap.ly / 2 + 5, dmap.ly / 2 - 5)
            if dmap.lookup(x0, y0) < 2.0:
                continue
            line = _walk_free_line(dmap, rng, x0, y0, total)
            if line is None:
                continue
            rows = natural_spline_rows(*line)
            st = reference_states(rows, n)
            if st is None:
                continue
            break
        else:
            raise RuntimeError("no free reference line found for line %d" % (first + b))
        k = rows.shape[1]
        lb.spline[b, :, :k], lb.k[b] = rows, k
        lb.spline[b, 0, k:] = rows[0, -1] + 1.0 + np.arange(lb.k_max - k)  # padding keeps abscissae increasing
        lb.states[b] = np.stack(st[:4])
        lb.kref[b] = st[4]
        inst = lb.inst[b]
        inst[abi.I_L0] = rng.uniform(-0.3, 0.3)
        inst[abi.I_PSI0] = rng.uniform(-0.08, 0.08)
        inst[abi.I_K0] = st[4][0]
        inst[abi.I_EPSI_LO], inst[abi.I_EPSI_HI] = -abi.INFTY, abi.INFTY
        if rng.uniform() < 0.5:
            e = rng.uniform(-0.05, 0.05)
            inst[abi.I_EPSI_LO], inst[abi.I_EPSI_HI] = e - 0.087, e + 0.087
    return lb
