"""numpy fp64 restatement of patch2pix_b200/csrc/abspose.cu (p2p_find_absolute_pose_batch, p2p_lift_scan), for tests
only.

Same sample generator (verify_oracle's), centring of the world points, P3P solver (Grunert's quartic, Ferrari with the
resolvent's largest root, two Newton steps per root, ascending roots, the same validity rules), rounds of 1024
hypotheses with the same stopping bound and tie rule, and Gauss-Newton local optimisation.  Differences from the
device: scoring is fp64 here (fp32 there), the centroid and the normal equations are summed in another order, and the
lift is the same arithmetic (every operation rounded on its own) so it agrees bit for bit.
"""
import numpy as np

from . import verify_oracle as V

ROUND = 1024
SAMPLE = 3
SLOTS = 4
MIN_ROWS = 4
LO_ITERS = 4
GN_STEPS = 3


# ---- P3P -------------------------------------------------------------------------------------------------------------
def cubic_max_root(b, c, d):
    p = c - b * b / 3.0
    q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    shift = -b / 3.0
    disc = q * q / 4.0 + p * p * p / 27.0
    if disc > 0:
        sq = np.sqrt(disc)
        return np.cbrt(-q / 2.0 + sq) + np.cbrt(-q / 2.0 - sq) + shift
    if p >= 0:
        return shift
    rr = 2.0 * np.sqrt(-p / 3.0)
    phi = np.arccos(min(1.0, max(-1.0, 1.5 * q / p * np.sqrt(-3.0 / p)))) / 3.0
    return rr * np.cos(phi) + shift


def quartic_roots(A):
    """Real roots of A[4] v^4 + ... + A[0], polished and ascending (abspose.cu quartic_roots)."""
    A = [float(a) for a in A]
    if not abs(A[4]) > 1e-12 * max(abs(a) for a in A):
        return []
    b, c, d, e = A[3] / A[4], A[2] / A[4], A[1] / A[4], A[0] / A[4]
    p = c - 3.0 * b * b / 8.0
    q = b * b * b / 8.0 - b * c / 2.0 + d
    rr = -3.0 * b * b * b * b / 256.0 + b * b * c / 16.0 - b * d / 4.0 + e
    m = cubic_max_root(p, p * p / 4.0 - rr, -q * q / 8.0)
    if not m > 0:
        return []
    s = np.sqrt(2.0 * m)
    r = []
    for sg in (1.0, -1.0):
        B, C = -sg * s, p / 2.0 + m + sg * q / (2.0 * s)
        D = B * B - 4.0 * C
        if not D >= 0:
            continue
        sd = np.sqrt(D)
        r += [(-B + sd) / 2.0 - b / 4.0, (-B - sd) / 2.0 - b / 4.0]
    out = []
    for v in r:
        for _ in range(2):
            f = (((A[4] * v + A[3]) * v + A[2]) * v + A[1]) * v + A[0]
            df = ((4.0 * A[4] * v + 3.0 * A[3]) * v + 2.0 * A[2]) * v + A[1]
            if df != 0:
                v = v - f / df
        out.append(v)
    return sorted(out)


def _frame(Q):
    e1 = Q[1] - Q[0]
    e3 = np.cross(e1, Q[2] - Q[0])
    n1, n3 = np.linalg.norm(e1), np.linalg.norm(e3)
    if not (n1 > 0 and n3 > 0):
        return None
    e1, e3 = e1 / n1, e3 / n3
    return np.stack([e1, np.cross(e3, e1), e3], 1)


def p3p_quartic(j, X):
    """Grunert's quartic of a sample -> (A0 .. A4, (b2, ca, cb, cg, amc)), or None when |X0 - X2| = 0."""
    a2, b2, c2 = (float(np.sum((X[i] - X[k]) ** 2)) for i, k in ((1, 2), (0, 2), (0, 1)))
    if not b2 > 0:
        return None
    ca, cb, cg = float(j[1] @ j[2]), float(j[0] @ j[2]), float(j[0] @ j[1])
    amc, apc, bmc, bma = (a2 - c2) / b2, (a2 + c2) / b2, (b2 - c2) / b2, (b2 - a2) / b2
    c2b, a2b = c2 / b2, a2 / b2
    return [(1.0 + amc) * (1.0 + amc) - 4.0 * a2b * cg * cg,
            4.0 * (-amc * (1.0 + amc) * cb + 2.0 * a2b * cg * cg * cb - (1.0 - apc) * ca * cg),
            2.0 * (amc * amc - 1.0 + 2.0 * amc * amc * cb * cb + 2.0 * bmc * ca * ca - 4.0 * apc * ca * cb * cg
                   + 2.0 * bma * cg * cg),
            4.0 * (amc * (1.0 - amc) * cb - (1.0 - apc) * ca * cg + 2.0 * c2b * ca * ca * cb),
            (amc - 1.0) * (amc - 1.0) - 4.0 * c2b * ca * ca], (b2, ca, cb, cg, amc)


def solve_p3p(j, X):
    """Bearings j [3, 3] (unit rows) and world points X [3, 3] -> list of [12] poses (R row-major, t; s_i j_i = R X_i +
    t), ascending in the quartic's root."""
    q = p3p_quartic(j, X)
    if q is None:
        return []
    A, (b2, ca, cb, cg, amc) = q
    roots = quartic_roots(A)
    FX = _frame(X)
    if FX is None:
        return []
    out = []
    with np.errstate(all='ignore'):
        for v in roots:
            u = ((-1.0 + amc) * v * v - 2.0 * amc * cb * v + 1.0 + amc) / (2.0 * (cg - v * ca))
            s1sq = b2 / (1.0 + v * v - 2.0 * v * cb)
            if not (u > 0 and v > 0 and s1sq > 0):
                continue
            s1 = np.sqrt(s1sq)
            P = np.stack([s1 * j[0], u * s1 * j[1], v * s1 * j[2]])
            FP = _frame(P)
            if FP is None:
                continue
            R = FP @ FX.T
            t = P[0] - R @ X[0]
            m = np.concatenate([R.reshape(9), t])
            if np.all(np.isfinite(m)):
                out.append(m)
    return out


# ---- prep, scoring ---------------------------------------------------------------------------------------------------
def bearings(rows, intr):
    fx, fy, cx, cy = (float(v) for v in intr)
    x, y = (rows[:, 0] - cx) / fx, (rows[:, 1] - cy) / fy
    nj = np.sqrt(x * x + y * y + 1.0)
    return np.stack([x / nj, y / nj, 1.0 / nj], 1)


def hypotheses(rows, intr, hyps, seed, mean=None):
    """Poses of the given hypotheses in the centred frame -> (models [len(hyps) * 4, 12], valid [len(hyps) * 4]), a
    sample's poses in its first slots."""
    rows = np.asarray(rows, dtype=np.float64)
    mean = rows[:, 2:5].mean(0) if mean is None else mean
    idx, ok = V.draw_samples(seed, hyps, rows.shape[0], SAMPLE)
    J, X = bearings(rows, intr), rows[:, 2:5] - mean
    B = len(hyps)
    models, valid = np.zeros((B * SLOTS, 12)), np.zeros(B * SLOTS, dtype=bool)
    for i in range(B):
        if not ok[i]:
            continue
        for k, m in enumerate(solve_p3p(J[idx[i]], X[idx[i]])):
            models[i * SLOTS + k], valid[i * SLOTS + k] = m, True
    return models, valid


def errors(models, rows, intr, mean):
    """Per (model, row) squared reprojection error in pixels, inf where the depth is not positive."""
    fx, fy, cx, cy = (float(v) for v in intr)
    M = np.asarray(models, dtype=np.float64).reshape(-1, 12)
    X = rows[:, 2:5] - mean
    P = np.einsum('mij,nj->mni', M[:, :9].reshape(-1, 3, 3), X) + M[:, None, 9:]
    with np.errstate(all='ignore'):
        eu = fx * P[..., 0] / P[..., 2] + cx - rows[None, :, 0]
        ev = fy * P[..., 1] / P[..., 2] + cy - rows[None, :, 1]
        return np.where(P[..., 2] > 0, eu * eu + ev * ev, np.inf)


def count_inliers(models, rows, intr, mean, th2, chunk=64):
    M = np.asarray(models).reshape(-1, 12)
    return np.concatenate([(errors(M[i:i + chunk], rows, intr, mean) < th2).sum(1)
                           for i in range(0, max(len(M), 1), chunk)])


def _expm(w):
    th2 = float(w @ w)
    if th2 < 1e-12:
        a, b = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        th = np.sqrt(th2)
        a, b = np.sin(th) / th, (1.0 - np.cos(th)) / th2
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.eye(3) + a * K + b * (K @ K)


def gauss_newton(m, rows, mask, intr, mean):
    """kAbsGnSteps Gauss-Newton steps on the squared reprojection error of the rows under `mask` -> pose or None."""
    fx, fy, cx, cy = (float(v) for v in intr)
    X = rows[mask, 2:5] - mean
    uv = rows[mask, 0:2]
    m = np.asarray(m, dtype=np.float64).copy()
    for _ in range(GN_STEPS):
        R, t = m[:9].reshape(3, 3), m[9:]
        P = X @ R.T
        x, y, z = (P + t).T
        ok = z > 0
        P, x, y, z, u = P[ok], x[ok], y[ok], z[ok], uv[ok]
        iz = 1.0 / z
        r = np.stack([fx * x * iz + cx - u[:, 0], fy * y * iz + cy - u[:, 1]], 1)
        Jp = np.zeros((len(z), 2, 3))
        Jp[:, 0, 0], Jp[:, 0, 2] = fx * iz, -fx * x * iz * iz
        Jp[:, 1, 1], Jp[:, 1, 2] = fy * iz, -fy * y * iz * iz
        nPx = np.zeros((len(z), 3, 3))                           # -[P]x
        nPx[:, 0, 1], nPx[:, 0, 2] = P[:, 2], -P[:, 1]
        nPx[:, 1, 0], nPx[:, 1, 2] = -P[:, 2], P[:, 0]
        nPx[:, 2, 0], nPx[:, 2, 1] = P[:, 1], -P[:, 0]
        J = np.concatenate([Jp @ nPx, Jp], 2).reshape(-1, 6)
        H, g = J.T @ J, J.T @ r.reshape(-1)
        try:
            L = np.linalg.cholesky(H)
        except np.linalg.LinAlgError:
            return None
        dx = np.linalg.solve(L.T, np.linalg.solve(L, g))
        nm = np.concatenate([(_expm(-dx[:3]) @ R).reshape(9), t - dx[3:]])
        if not np.all(np.isfinite(nm)):
            return None
        m = nm
    return m


def to_world(m, mean):
    """Centred-frame pose -> world pose [12] (t - R mean)."""
    R = m[:9].reshape(3, 3)
    return np.concatenate([m[:9], m[9:] - R @ mean])


def find_absolute_pose(rows, intr, px_th, conf=0.99999, max_iters=10000, seed=0, trace=None):
    """-> (pose [12] world frame or None, bool mask [n], inlier count; -1 and a NaN pose for a non-finite value).
    `trace` (a dict, optional) receives the winner's slot, its count before LO, its margin over the runner-up and the
    hypotheses drawn."""
    rows = np.asarray(rows, dtype=np.float64)
    n = rows.shape[0]
    if not np.all(np.isfinite(rows[:, :5])):
        return np.full(12, np.nan), np.zeros(n, dtype=bool), -1
    if n < MIN_ROWS:
        return None, np.zeros(n, dtype=bool), 0
    th2 = float(px_th) ** 2
    mean = rows[:, 2:5].mean(0)
    best, best_count, best_slot, done, top = None, 0, -1, 0, [0, 0]
    for first in range(0, max_iters, ROUND):
        count = min(ROUND, max_iters - first)
        models, valid = hypotheses(rows, intr, np.arange(first, first + count), seed, mean)
        counts = np.where(valid, count_inliers(models, rows, intr, mean, th2), -1)
        c = int(counts.max())
        top = sorted(top + sorted(counts.tolist())[-2:])[-2:]
        if c > best_count:
            k = int(np.argmax(counts))
            best, best_count, best_slot = models[k], c, first * SLOTS + k
        done = first + count
        needed = np.inf
        if best_count > 0:
            ws = (best_count / n) ** SAMPLE
            needed = 0.0 if ws >= 1 else np.log(1.0 - conf) / np.log1p(-ws)
        if done >= max_iters or done >= needed:
            break
    if trace is not None:
        trace.update(slot=best_slot, ransac_count=best_count, margin=top[1] - top[0], hypotheses=done)
    if best is None:
        return None, np.zeros(n, dtype=bool), 0
    cur = best
    cur_mask = errors(cur, rows, intr, mean)[0] < th2
    cur_count = int(cur_mask.sum())
    for _ in range(LO_ITERS):
        if cur_count < MIN_ROWS:
            break
        cand = gauss_newton(cur, rows, cur_mask, intr, mean)
        if cand is None:
            break
        cand_mask = errors(cand, rows, intr, mean)[0] < th2
        if int(cand_mask.sum()) <= cur_count:
            break
        cur, cur_mask, cur_count = cand, cand_mask, int(cand_mask.sum())
    return to_world(cur, mean), cur_mask, cur_count


# ---- the scan lift ---------------------------------------------------------------------------------------------------
def sample_scan(scan, x, y):
    """grid_sample(align_corners=True) of scan [H, W, 3] at pixels (x, y) [N]: bilinear over the in-bounds corners
    (nw, ne, sw, se, summed in that order), NaN channels from the nearest pixel (round half to even).  The points must
    lie in [0, W-1] x [0, H-1]."""
    H, W, _ = scan.shape
    x0, y0 = np.floor(x), np.floor(y)
    x1, y1 = x0 + 1.0, y0 + 1.0
    corners = ((x0, y0, (x1 - x) * (y1 - y)), (x1, y0, (x - x0) * (y1 - y)), (x0, y1, (x1 - x) * (y - y0)),
               (x1, y1, (x - x0) * (y - y0)))
    v = np.zeros((x.shape[0], 3))
    for cx, cy, w in corners:
        inb = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
        xi, yi = np.where(inb, cx, 0).astype(np.int64), np.where(inb, cy, 0).astype(np.int64)
        v = np.where(inb[:, None], v + scan[yi, xi] * w[:, None], v)
    nn = scan[np.rint(y).astype(np.int64), np.rint(x).astype(np.int64)]
    return np.where(np.isnan(v), nn, v)


def lift_scan(scan, align, matches):
    """Rows (xq, yq, X, Y, Z) [m, 5] of the matches [N, >= 4] (xq, yq, xdb, ydb) that p2p_lift_scan keeps, in match
    order."""
    scan = np.asarray(scan, dtype=np.float64)
    A = np.asarray(align, dtype=np.float64).reshape(4, 4)
    mt = np.asarray(matches, dtype=np.float64).reshape(-1, matches.shape[-1] if np.ndim(matches) == 2 else 4)
    H, W, _ = scan.shape
    x, y = mt[:, 2], mt[:, 3]
    inside = (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)
    p = sample_scan(scan, x[inside], y[inside])
    keep = np.all(np.isfinite(p), 1)
    p = p[keep]
    X = [((A[i, 0] * p[:, 0] + A[i, 1] * p[:, 1]) + A[i, 2] * p[:, 2]) + A[i, 3] for i in range(3)]
    q = mt[inside][keep]
    return np.stack([q[:, 0], q[:, 1]] + X, 1)
