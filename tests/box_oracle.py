"""The obstacle set of pqp_bounds_set_occupancy_boxes (include/pqp_bounds.h), in numpy, on top of the exact distance
transform of oracle/edt_oracle.py. TEST ONLY.

`stamp_boxes` is the base image's obstacles plus every cell whose centre lies in or on an oriented box (x, y, heading,
length, width), by the header's predicate in float64 with its operation order (numpy rounds each operation on its own);
`edge_distance` is each cell's distance to the nearest box edge, which says where a last-bit difference in cos / sin
could decide a cell.
"""
import numpy as np

from oracle.edt_oracle import obstacles


def cell_centres(shape, res, center):
    """(px [rows, 1], py [1, cols]) of the cell centres, as pqp_bounds_map places them (half_lx = 0.5 * rows * res)."""
    rows, cols = shape
    half_lx, half_ly = 0.5 * rows * float(res), 0.5 * cols * float(res)
    px = float(center[0]) + (half_lx - (np.arange(rows, dtype=np.float64) + 0.5) * float(res))
    py = float(center[1]) + (half_ly - (np.arange(cols, dtype=np.float64) + 0.5) * float(res))
    return px[:, None], py[None, :]


def _box_uv(px, py, box):
    x, y, heading, length, width = (float(v) for v in box)
    with np.errstate(invalid="ignore", over="ignore"):  # an infinite heading has a NaN cosine, as on the device
        c, s = np.cos(np.float64(heading)), np.sin(np.float64(heading))
        dx, dy = px - x, py - y
        return dx * c + dy * s, dy * c - dx * s, 0.5 * length, 0.5 * width


def stamp_boxes(img, res, center, boxes, obstacle_max=0):
    """The obstacle mask (bool [rows, cols]) of a base image plus boxes [k, 5]."""
    obst = obstacles(img, obstacle_max)
    px, py = cell_centres(obst.shape, res, center)
    for box in np.asarray(boxes, dtype=np.float64).reshape(-1, 5):
        u, v, hl, hw = _box_uv(px, py, box)
        with np.errstate(invalid="ignore"):
            obst |= (np.abs(u) <= hl) & (np.abs(v) <= hw)
    return obst


def stamped_image(img, res, center, boxes, obstacle_max=0):
    """A uint8 image (0: obstacle, 255: free) of the stamped obstacle set, for `transform(..., obstacle_max=0)` and for
    set_occupancy_slots."""
    return np.where(stamp_boxes(img, res, center, boxes, obstacle_max), 0, 255).astype(np.uint8)


def edge_distance(shape, res, center, boxes):
    """Each cell centre's Euclidean distance to the boundary of the nearest box (inf without boxes), in the box's own
    frame: inside min(hl - |u|, hw - |v|), outside the distance to the rectangle."""
    px, py = cell_centres(shape, res, center)
    out = np.full(shape, np.inf)
    for box in np.asarray(boxes, dtype=np.float64).reshape(-1, 5):
        u, v, hl, hw = _box_uv(px, py, box)
        au, av = np.abs(u), np.abs(v)
        inside = (au <= hl) & (av <= hw)
        d = np.where(inside, np.minimum(hl - au, hw - av),
                     np.hypot(np.maximum(au - hl, 0.0), np.maximum(av - hw, 0.0)))
        out = np.minimum(out, np.where(np.isnan(d), np.inf, d))
    return out
