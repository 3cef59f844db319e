"""numpy restatement of the HPatches statistics (patch2pix_b200/hpatches.py, p2p_homography_errors), for the tests.

Every product and sum is a separate fp64 numpy operation in the order the kernel uses ((h0 x + h1 y) + h2), so the
distances agree bit for bit with the device's, whose arithmetic has no fused multiply-add.
"""
import numpy as np


def project(H, x, y):
    """(px, py, w) of pi(H [x, y, 1]^T), elementwise over arrays x, y."""
    H = np.asarray(H, dtype=np.float64).reshape(9)
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(all='ignore'):
        u = (H[0] * x + H[1] * y) + H[2]
        v = (H[3] * x + H[4] * y) + H[5]
        w = (H[6] * x + H[7] * y) + H[8]
        return u / w, v / w, w


def _dist(ax, ay, bx, by):
    with np.errstate(all='ignore'):
        dx, dy = ax - bx, ay - by
        return np.sqrt(dx * dx + dy * dy)


def reprojection_errors(rows, H_gt):
    """d = |pi(H_gt [x1, y1, 1]^T) - (x2, y2)| per row of [N, >=4] float64 rows."""
    rows = np.asarray(rows, dtype=np.float64)
    rows = rows.reshape(0, 4) if rows.size == 0 else rows.reshape(len(rows), -1)
    px, py, _ = project(H_gt, rows[:, 0], rows[:, 1])
    return _dist(px, py, rows[:, 2], rows[:, 3])


def counts(d, thresholds):
    """int32 [len(thresholds) + 1]: #(d <= t) per threshold (NaN and inf never count), then len(d)."""
    d = np.asarray(d, dtype=np.float64)
    with np.errstate(invalid='ignore'):
        c = [int(np.count_nonzero(d <= t)) for t in thresholds]
    return np.array(c + [len(d)], dtype=np.int32)


def corner_error(H_gt, H_pred, n_inliers, width, height):
    """Mean over the corners (0, 0), (w-1, 0), (0, h-1), (w-1, h-1) of |pi(H_gt c) - pi(H_pred c)|, summed in that
    order; +inf when n_inliers <= 0 (no model), a corner has w = 0 under either H, or the mean is not finite."""
    if n_inliers <= 0:
        return np.inf
    cx = np.array([0.0, width - 1.0, 0.0, width - 1.0])
    cy = np.array([0.0, 0.0, height - 1.0, height - 1.0])
    gx, gy, wg = project(H_gt, cx, cy)
    ex, ey, we = project(H_pred, cx, cy)
    if np.any(wg == 0) or np.any(we == 0):
        return np.inf
    d = _dist(gx, gy, ex, ey)
    s = 0.0
    for v in d:
        s = s + float(v)
    e = s / 4.0
    return e if np.isfinite(e) else np.inf


def pair_mma(c):
    """Per-pair accuracy at each threshold from counts(...): correct / N, all 0 when N = 0."""
    c = np.asarray(c)
    n = int(c[-1])
    return np.zeros(len(c) - 1) if n == 0 else c[:-1].astype(np.float64) / n


def split_summary(seqs, pair_mmas, corner_errs, h_thresholds):
    """({'all', 'i', 'v'} -> mean per-pair MMA, {'all', 'i', 'v'} -> share of pairs with corner error <= t), one entry
    per pair; seqs are the sequence names (split = name[0]).  An empty split gives NaN."""
    seqs = list(seqs)
    pm = np.asarray(pair_mmas, dtype=np.float64).reshape(len(seqs), -1)
    ce = np.asarray(corner_errs, dtype=np.float64).reshape(-1)
    mma, hacc = {}, {}
    for split in ('all', 'i', 'v'):
        sel = np.array([split == 'all' or s.startswith(split + '_') for s in seqs], dtype=bool)
        if not sel.any():
            mma[split] = np.full(pm.shape[1], np.nan)
            hacc[split] = np.full(len(h_thresholds), np.nan)
            continue
        mma[split] = pm[sel].mean(0)
        hacc[split] = np.array([np.mean(ce[sel] <= t) for t in h_thresholds])
    return mma, hacc
