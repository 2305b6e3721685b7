"""float64 restatement of hvn_inst_features (include/hvn.h HVN_FEAT_*): the oracle of tests/test_features_*.py.

Every column is computed as the device computes it, operation for operation in IEEE double (Python floats), from
exact integer sums; the convex hull is Andrew's monotone chain here, and tests/test_features_cpu.py checks it and the
other contour quantities against cv2's own contourArea, arcLength, convexHull and moments."""
import math

import numpy as np

NAMES = ("area", "contour_area", "perimeter", "convex_area", "solidity", "circularity", "major_axis_length",
         "minor_axis_length", "eccentricity", "orientation", "feret_max", "mean_r", "mean_g", "mean_b", "std_r",
         "std_g", "std_b", "np_prob_mean")


def shoelace2(P):
    """Twice the signed shoelace area of the closed polygon P [n,2] (x, y), exact."""
    s = 0
    n = len(P)
    for i in range(n):
        (x0, y0), (x1, y1) = P[i - 1], P[i]
        s += int(x0) * int(y1) - int(y0) * int(x1)
    return s


def arc_length(P):
    """cv2.arcLength(P, True): fp32 segment lengths from the closing segment on, added in fp64 in point order."""
    n = len(P)
    if n <= 1:
        return 0.0
    P = np.asarray(P, dtype=np.int64)
    prev = np.roll(P, 1, axis=0)
    d = (P - prev).astype(np.float32)
    seg = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])  # float32 throughout
    s = 0.0
    for v in seg:
        s += float(v)
    return s


def hull(P):
    """Convex hull vertices of the point set P (Andrew's monotone chain, collinear points dropped), counter-clockwise
    in image axes; one point for a single distinct point, two for a segment."""
    pts = sorted(set((int(x), int(y)) for x, y in P))
    if len(pts) <= 1:
        return pts

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    lower, upper = [], []
    for p in pts:
        while len(lower) >= 2 and cross(lower[-2], lower[-1], p) <= 0:
            lower.pop()
        lower.append(p)
    for p in reversed(pts):
        while len(upper) >= 2 and cross(upper[-2], upper[-1], p) <= 0:
            upper.pop()
        upper.append(p)
    return lower[:-1] + upper[:-1]


def moments(crop):
    """(A, m10, m01, mu20, mu11, mu02) of the binary crop: exact integer raw moments, the central ones completed in
    OpenCV's order (cx = m10 * (1 / m00), mu20 = m20 - m10 * cx, mu11 = m11 - m10 * cy, mu02 = m02 - m01 * cy)."""
    ys, xs = np.nonzero(crop)
    xs, ys = xs.astype(np.int64), ys.astype(np.int64)
    A, m10, m01 = int(xs.size), int(xs.sum()), int(ys.sum())
    m20, m11, m02 = int((xs * xs).sum()), int((xs * ys).sum()), int((ys * ys).sum())
    if A == 0:
        return 0, 0, 0, 0.0, 0.0, 0.0
    inv = 1.0 / float(A)
    cx, cy = float(m10) * inv, float(m01) * inv
    return A, m10, m01, float(m20) - float(m10) * cx, float(m11) - float(m10) * cy, float(m02) - float(m01) * cy


def pop_std(A, S, Q):
    return math.sqrt(float(A * Q - S * S) / (float(A) * float(A)))


def row_features(inst, table_row, P, img=None, np_map=None):
    """The HVN_FEAT_LEN columns of one instance-table row.  inst [H,W]; table_row (id, rmin, cmin, rmax, cmax, ...);
    P [n,2] (x, y) map coordinates; img u8 [H,W,3] or None; np_map float32 [H,W] (the NP channel) or None."""
    iid, rmin, cmin, rmax, cmax = (int(v) for v in table_row[:5])
    crop = np.asarray(inst)[rmin:rmax, cmin:cmax] == iid
    A, _, _, mu20, mu11, mu02 = moments(crop)
    P = np.asarray(P, dtype=np.int64).reshape(-1, 2)
    f = [0.0] * len(NAMES)
    f[0] = float(A)
    carea = abs(shoelace2(P)) * 0.5
    perim = arc_length(P)
    H = hull(P)
    harea = abs(shoelace2(H)) * 0.5 if len(H) >= 3 else 0.0
    f[1], f[2], f[3] = float(carea), perim, float(harea)
    f[4] = carea / harea if harea != 0.0 else 0.0
    f[5] = 4.0 * math.pi * carea / (perim * perim) if perim != 0.0 else 0.0
    if A > 0:
        a_px = float(A)
        a, b, c = mu20 / a_px, mu11 / a_px, mu02 / a_px
        hd, mid = (a - c) / 2.0, (a + c) / 2.0
        rr = math.sqrt(hd * hd + b * b)
        l1, l2 = mid + rr, max(mid - rr, 0.0)
        f[6], f[7] = 4.0 * math.sqrt(l1), 4.0 * math.sqrt(l2)
        f[8] = math.sqrt(1.0 - l2 / l1) if l1 != 0.0 else 0.0
        f[9] = 0.5 * math.atan2(2.0 * b, a - c)
    fer2 = 0
    for i in range(len(H)):
        for j in range(i + 1, len(H)):
            dx, dy = H[j][0] - H[i][0], H[j][1] - H[i][1]
            fer2 = max(fer2, dx * dx + dy * dy)
    f[10] = math.sqrt(float(fer2))
    if img is None:
        f[11:17] = [math.nan] * 6
    else:
        v = np.asarray(img)[rmin:rmax, cmin:cmax][crop].astype(np.int64)
        for ch in range(3):
            S, Q = int(v[:, ch].sum()), int((v[:, ch] * v[:, ch]).sum())
            f[11 + ch] = float(S) / float(A) if A else 0.0
            f[14 + ch] = pop_std(A, S, Q) if A else 0.0
    if np_map is None:
        f[17] = math.nan
    else:
        vals = np.asarray(np_map, dtype=np.float32)[rmin:rmax, cmin:cmax][crop].astype(np.float64)
        f[17] = float(vals.sum()) / float(A) if A else 0.0
    return np.array(f, dtype=np.float64)


def features(inst, table, pts, offs, img=None, pred=None):
    """row_features over every row of a one-map call (offs: the point range of row r is pts[offs[r]:offs[r+1]]);
    pred [H,W,C] with NP at channel C - 3."""
    np_map = None if pred is None else np.asarray(pred)[..., np.asarray(pred).shape[-1] - 3]
    return np.stack([row_features(inst, table[r], pts[int(offs[r]):int(offs[r + 1])], img, np_map)
                     for r in range(len(table))]) if len(table) else np.zeros((0, len(NAMES)))


# ---- test inputs ---------------------------------------------------------------------------------------------------
def table_of(inst):
    """Instance-table rows [n,10] of every id > 0 of inst, ascending (id, rmin, cmin, rmax, cmax exclusive, area; the
    other columns 0): what hvn_postproc's table holds for these columns."""
    rows = []
    for iid in np.unique(inst):
        if iid <= 0:
            continue
        ys, xs = np.nonzero(inst == iid)
        rows.append([iid, ys.min(), xs.min(), ys.max() + 1, xs.max() + 1, ys.size, 0, 0, 0, 0])
    return np.array(rows, dtype=np.int64).reshape(-1, 10)


def cv2_contours(inst, table):
    """(pts [m,2] int32, offs [n+1]): per row the reference's contour, cv2.findContours(crop == id, RETR_TREE,
    CHAIN_APPROX_SIMPLE)[0][0] + (cmin, rmin)."""
    import cv2
    parts, offs = [], [0]
    for r in table:
        iid, rmin, cmin, rmax, cmax = (int(v) for v in r[:5])
        crop = (inst[rmin:rmax, cmin:cmax] == iid).astype(np.uint8)
        c = cv2.findContours(crop, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)[0][0].reshape(-1, 2) + [cmin, rmin]
        parts.append(c.astype(np.int32))
        offs.append(offs[-1] + len(c))
    pts = np.concatenate(parts) if parts else np.zeros((0, 2), np.int32)
    return pts.astype(np.int32), np.array(offs, dtype=np.int32)


def rhombus(r):
    """A filled rhombus |x| + 2 |y| <= 2 r, [2r+1, 4r+1]: its border steps E, NE, E, NE, ..., so its contour has 8 r
    CHAIN_APPROX_SIMPLE points."""
    y, x = np.mgrid[-r:r + 1, -2 * r:2 * r + 1]
    return np.abs(x) + 2 * np.abs(y) <= 2 * r


def edge_maps():
    """(name, inst int32) maps with the shapes the measurements must get right."""
    out = []
    m = np.zeros((12, 14), np.int32)
    m[2, 3] = 1                      # 1 pixel
    m[5, 5:7] = 2                    # 2 pixels, horizontal
    m[8, 1] = m[9, 2] = 3            # 2 pixels, diagonal
    m[1:9, 10] = 4                   # a vertical line: collinear contour, convex_area 0
    m[10, 3:12] = 5                  # a horizontal line
    out.append(("small", m))
    m = np.zeros((20, 20), np.int32)
    for k in range(8):               # a diagonal line of 8-connected pixels
        m[2 + k, 2 + k] = 1
    m[3:8, 11:16] = 2                # two blobs joined by a one-pixel neck
    m[8, 13] = 2
    m[9:14, 11:16] = 2
    m[14:19, 1:8] = 3                # a ring with a hole
    m[16, 3:6] = 0
    m[15:18, 4] = 0
    out.append(("necks_rings", m))
    m = np.zeros((16, 18), np.int32)
    m[0, 2:6] = 1                    # bboxes on every edge and corner
    m[15, 4:9] = 2
    m[3:9, 0] = 3
    m[5:12, 17] = 4
    m[0:2, 15:18] = 5
    m[13:16, 0:3] = 6
    m[6:9, 6:11] = 7
    out.append(("edges", m))
    out.append(("w1", np.array([[0], [3], [3], [0], [7], [7], [7]], np.int32)))
    out.append(("h1", np.array([[2, 2, 0, 5, 5, 5, 5, 0, 9]], np.int32)))
    # contours of 504, 512 (the device's shared-memory cap) and 520 points, and one of 1200
    m = np.zeros((135, 820), np.int32)
    m[2:129, 1:254][rhombus(63)] = 1
    m[2:131, 270:527][rhombus(64)] = 2
    m[1:132, 545:806][rhombus(65)] = 3
    out.append(("rhombus_cap", m))
    m = np.zeros((305, 610), np.int32)
    m[2:303, 3:604][rhombus(150)] = 4
    out.append(("rhombus_big", m))
    return out


def seeded_map(h, w, seed, n=40):
    """A map of n random ellipses (overlaps overwrite), ids 1..n."""
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), np.int32)
    y, x = np.mgrid[0:h, 0:w]
    for k in range(1, n + 1):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        a, b, t = rng.uniform(2, 12), rng.uniform(2, 9), rng.uniform(0, np.pi)
        u = (x - cx) * np.cos(t) + (y - cy) * np.sin(t)
        v = -(x - cx) * np.sin(t) + (y - cy) * np.cos(t)
        m[(u / a) ** 2 + (v / b) ** 2 <= 1] = k
    return m
