"""numpy restatement of the relative-pose statistics (patch2pix_b200/relpose.py, p2p_relpose_errors_batch), for the tests.

Every product, sum, quotient and square root is a separate fp64 numpy operation in the order csrc/relpose.cu uses, so
the cosines and the epipolar errors agree bit for bit with the device's, whose arithmetic has no fused multiply-add.
The host statistics (arccos, the E ambiguity fold, the AUC and the precision) are restated from the protocol of
SuperGlue / LoFTR's relative-pose evaluation.
"""
import numpy as np


def essential_from_pose(Rt):
    """E = [t]x R of a [12] pose (R row-major, then t), row by row as the kernel: -t2 R1 + t1 R2, t2 R0 - t0 R2,
    t0 R1 - t1 R0."""
    Rt = np.asarray(Rt, dtype=np.float64).reshape(12)
    R = Rt[:9].reshape(3, 3)
    t0, t1, t2 = Rt[9], Rt[10], Rt[11]
    return np.stack([t1 * R[2] - t2 * R[1], t2 * R[0] - t0 * R[2], t0 * R[1] - t1 * R[0]])


def _dot3(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def epipolar_errors(rows, intr, Rt_gt):
    """Symmetric epipolar error in camera coordinates of each row (x0, y0, x1, y1 in columns 0..3) under
    E = [t_gt]x R_gt: (x1^T E x0)^2 (1 / ((E x0)_0^2 + (E x0)_1^2) + 1 / ((E^T x1)_0^2 + (E^T x1)_1^2)).
    intr: (fx0, fy0, cx0, cy0, fx1, fy1, cx1, cy1)."""
    rows = np.asarray(rows, dtype=np.float64)
    rows = rows.reshape(0, 4) if rows.size == 0 else rows.reshape(len(rows), -1)
    fx0, fy0, cx0, cy0, fx1, fy1, cx1, cy1 = (float(v) for v in np.asarray(intr, dtype=np.float64).reshape(8))
    E = essential_from_pose(Rt_gt).reshape(9)
    with np.errstate(all='ignore'):
        u0, v0 = (rows[:, 0] - cx0) / fx0, (rows[:, 1] - cy0) / fy0
        u1, v1 = (rows[:, 2] - cx1) / fx1, (rows[:, 3] - cy1) / fy1
        l0 = _dot3(E[0], E[1], E[2], u0, v0, 1.0)
        l1 = _dot3(E[3], E[4], E[5], u0, v0, 1.0)
        l2 = _dot3(E[6], E[7], E[8], u0, v0, 1.0)
        m0 = _dot3(E[0], E[3], E[6], u1, v1, 1.0)
        m1 = _dot3(E[1], E[4], E[7], u1, v1, 1.0)
        num = _dot3(u1, v1, 1.0, l0, l1, l2)
        d0 = l0 * l0 + l1 * l1
        d1 = m0 * m0 + m1 * m1
        return (num * num) * (1.0 / d0 + 1.0 / d1)


def counts(err, thresholds):
    """int32 [len(thresholds) + 1]: #(err < t) per threshold (NaN never counts), then len(err)."""
    err = np.asarray(err, dtype=np.float64)
    with np.errstate(invalid='ignore'):
        c = [int(np.count_nonzero(err < t)) for t in thresholds]
    return np.array(c + [len(err)], dtype=np.int32)


def _clip1(c):
    return 1.0 if c > 1.0 else (-1.0 if c < -1.0 else c)       # keeps NaN


def pose_cosines(Rt_gt, Rt_est, n_inliers):
    """(cos of the rotation error, cos of the translation-direction error) as the kernel computes them: (tr(R_gt^T R) -
    1) / 2 with the nine products summed in row-major order, t_gt . t / (|t_gt| |t|), each clipped to [-1, 1]; NaN for
    both when n_inliers <= 0."""
    if n_inliers <= 0:
        return np.nan, np.nan
    g = np.asarray(Rt_gt, dtype=np.float64).reshape(12)
    e = np.asarray(Rt_est, dtype=np.float64).reshape(12)
    with np.errstate(all='ignore'):
        tr = np.float64(0.0)
        for j in range(9):
            tr = tr + g[j] * e[j]
        cr = _clip1((tr - 1.0) / 2.0)
        dot = _dot3(g[9], g[10], g[11], e[9], e[10], e[11])
        ng = np.sqrt(_dot3(g[9], g[10], g[11], g[9], g[10], g[11]))
        ne = np.sqrt(_dot3(e[9], e[10], e[11], e[9], e[10], e[11]))
        ct = _clip1(dot / (ng * ne))
    return float(cr), float(ct)


def pose_errors(cos_R, cos_t, failed=False):
    """(R_err, t_err) in degrees from the cosines: arccos, t_err folded to min(t_err, 180 - t_err) (E fixes t up to
    sign); both +inf when the pair failed or a cosine is not finite (no model)."""
    if failed or not (np.isfinite(cos_R) and np.isfinite(cos_t)):
        return np.inf, np.inf
    r = float(np.degrees(np.arccos(cos_R)))
    t = float(np.degrees(np.arccos(cos_t)))
    return r, min(t, 180.0 - t)


def pose_auc(errors, thresholds):
    """Area under the recall curve of the pose errors up to each threshold, divided by it: errors sorted, recall
    (i + 1) / N, (0, 0) prepended, the curve cut at the threshold (errors equal to it fall outside), trapezoid rule.  An
    empty list gives NaN."""
    errors = np.sort(np.asarray(errors, dtype=np.float64).reshape(-1))
    if errors.size == 0:
        return {t: float('nan') for t in thresholds}
    recall = np.r_[0.0, (np.arange(errors.size) + 1) / errors.size]
    errors = np.r_[0.0, errors]
    out = {}
    for t in thresholds:
        last = int(np.searchsorted(errors, t))
        r = np.r_[recall[:last], recall[last - 1]]
        e = np.r_[errors[:last], t]
        out[t] = float(np.trapezoid(r, x=e) / t)
    return out


def precision(count_rows, thresholds):
    """Mean over pairs of correct(t) / N per threshold (0 for a pair with N = 0) from counts(...) rows; NaN without
    pairs."""
    c = np.asarray(count_rows, dtype=np.float64).reshape(-1, len(thresholds) + 1)
    if c.shape[0] == 0:
        return {t: float('nan') for t in thresholds}
    n = c[:, -1]
    with np.errstate(all='ignore'):
        p = np.where(n[:, None] > 0, c[:, :-1] / np.where(n > 0, n, 1.0)[:, None], 0.0)
    return {t: float(p[:, j].mean()) for j, t in enumerate(thresholds)}
