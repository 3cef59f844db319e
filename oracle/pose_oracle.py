"""numpy fp64 restatement of patch2pix_b200/csrc/pose.cu (p2p_find_essential, p2p_recover_pose), for tests only.

Same normalisation to camera coordinates, sample generator (verify_oracle's, s = 5), 5-point solver (null space of the
5 x 9 epipolar system, the 10 cubic constraints over 20 monomials, Gauss-Jordan with partial pivoting, the degree-10
polynomial in z, Sturm sequence + bisection + Newton, back-substitution), rounds of 1024 hypotheses with the same
stopping bound, tie rule and local optimisation, and the same pose recovery.  Differences from the device: scoring is
fp64 here (fp32 there), and SVDs / smallest eigenvectors come from numpy (Jacobi there).
"""
import numpy as np

from . import verify_oracle as V

ROUND = V.ROUND
SAMPLE = 5
SLOTS = 10
LO_ITERS = V.LO_ITERS
LO_MIN = 8
BISECT = 64                   # bisection steps per root
NEWTON = 2                    # guarded Newton steps per root
ZMAX = 1e6                    # roots are searched in (-ZMAX, ZMAX]
DIST_TH = 50.0                # cv2.recoverPose's default distanceThresh

# Monomials of degree <= 3 in (x, y, z): the 10 eliminated ones first, then x * (z^2, z, 1), y * (z^2, z, 1), z^3 .. 1.
MON3 = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
        (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]
MON2 = [(2, 0, 0), (1, 1, 0), (1, 0, 1), (0, 2, 0), (0, 1, 1), (0, 0, 2), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
VAR = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]      # x, y, z, 1


def _add(a, b):
    return tuple(i + j for i, j in zip(a, b))


MUL11 = [[MON2.index(_add(VAR[i], VAR[j])) for j in range(4)] for i in range(4)]    # var i * var j -> MON2 index
MUL21 = [[MON3.index(_add(MON2[i], VAR[j])) for j in range(4)] for i in range(10)]  # MON2 i * var j -> MON3 index


def to_camera(rows, intr):
    """Pixel rows [n, 4] -> normalised camera coordinates ((x - cx) / fx, (y - cy) / fy) per view."""
    fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2 = (float(v) for v in intr)
    return np.stack([(rows[..., 0] - cx1) / fx1, (rows[..., 1] - cy1) / fy1,
                     (rows[..., 2] - cx2) / fx2, (rows[..., 3] - cy2) / fy2], -1)


def _mul11(a, b):
    out = np.zeros(a.shape[:-1] + (10,))
    for i in range(4):
        for j in range(4):
            out[..., MUL11[i][j]] += a[..., i] * b[..., j]
    return out


def _mul21(a, b):
    out = np.zeros(a.shape[:-1] + (20,))
    for i in range(10):
        for j in range(4):
            out[..., MUL21[i][j]] += a[..., i] * b[..., j]
    return out


def constraints(ns):
    """Null spaces [B, 4, 9] (E = x X + y Y + z Z + W) -> [B, 10, 20]: det E = 0, then 2 E E^T E - tr(E E^T) E = 0
    row-major, over MON3."""
    e = np.transpose(ns, (0, 2, 1))                          # [B, 9, 4]: entry (i, j) of E as a polynomial in x, y, z
    E = lambda i, j: e[:, 3 * i + j]
    eet = {}
    for i in range(3):
        for j in range(i, 3):
            eet[i, j] = eet[j, i] = _mul11(E(i, 0), E(j, 0)) + _mul11(E(i, 1), E(j, 1)) + _mul11(E(i, 2), E(j, 2))
    tr = eet[0, 0] + eet[1, 1] + eet[2, 2]
    rows = [_mul21(_mul11(E(1, 1), E(2, 2)) - _mul11(E(1, 2), E(2, 1)), E(0, 0))
            - _mul21(_mul11(E(1, 0), E(2, 2)) - _mul11(E(1, 2), E(2, 0)), E(0, 1))
            + _mul21(_mul11(E(1, 0), E(2, 1)) - _mul11(E(1, 1), E(2, 0)), E(0, 2))]
    for i in range(3):
        for j in range(3):
            acc = _mul21(eet[i, 0], E(0, j)) + _mul21(eet[i, 1], E(1, j)) + _mul21(eet[i, 2], E(2, j))
            rows.append(2.0 * acc - _mul21(tr, E(i, j)))
    return np.stack(rows, 1)


def gauss_jordan(M):
    """[B, 10, 20] -> ([B, 10, 10] right block after reducing the left block to I with partial pivoting, ok [B])."""
    M = np.array(M, dtype=np.float64)
    B = M.shape[0]
    bi = np.arange(B)
    amax0 = np.abs(M).reshape(B, -1).max(1)
    ok = amax0 > 0
    for c in range(10):
        p = c + np.abs(M[:, c:, c]).argmax(1)
        ok &= np.abs(M[bi, p, c]) > 1e-12 * amax0
        rc = M[bi, c].copy()
        M[bi, c] = M[bi, p]
        M[bi, p] = rc
        piv = np.where(ok, M[:, c, c], 1.0)
        M[:, c] /= piv[:, None]
        f = M[:, :, c].copy()
        f[:, c] = 0.0
        M -= f[:, :, None] * M[:, c:c + 1, :]
    return M[:, :, 10:], ok


def _row_polys(Bm, e, f):
    """<e> - z <f> as polynomials (ascending in z) multiplying x (deg 3), y (deg 3) and 1 (deg 4)."""
    X = lambda r: [Bm[:, r, 2], Bm[:, r, 1], Bm[:, r, 0]]
    Y = lambda r: [Bm[:, r, 5], Bm[:, r, 4], Bm[:, r, 3]]
    Cz = lambda r: [Bm[:, r, 9], Bm[:, r, 8], Bm[:, r, 7], Bm[:, r, 6]]
    def sub(pe, pf):
        out = list(pe) + [np.zeros_like(pe[0])]
        for k, c in enumerate(pf):
            out[k + 1] = out[k + 1] - c
        return np.stack(out, -1)
    return sub(X(e), X(f)), sub(Y(e), Y(f)), sub(Cz(e), Cz(f))


def _pmul(a, b):
    out = np.zeros(a.shape[:-1] + (a.shape[-1] + b.shape[-1] - 1,))
    for i in range(a.shape[-1]):
        for j in range(b.shape[-1]):
            out[..., i + j] += a[..., i] * b[..., j]
    return out


def _psub(a, b):
    n = max(a.shape[-1], b.shape[-1])
    pa = np.zeros(a.shape[:-1] + (n,))
    pb = np.zeros(b.shape[:-1] + (n,))
    pa[..., :a.shape[-1]] = a
    pb[..., :b.shape[-1]] = b
    return pa - pb


def degree10(Bm):
    """The three rows <k>, <l>, <m> of Nister's elimination and det of their 3x3 polynomial matrix ->
    (rows [(k1, k2, k3), (l1, l2, l3), (m1, m2, m3)], d [B, 11] ascending in z)."""
    k = _row_polys(Bm, 4, 5)
    l = _row_polys(Bm, 6, 7)
    m = _row_polys(Bm, 8, 9)
    c1 = _psub(_pmul(l[1], m[2]), _pmul(l[2], m[1]))
    c2 = _psub(_pmul(l[0], m[2]), _pmul(l[2], m[0]))
    c3 = _psub(_pmul(l[0], m[1]), _pmul(l[1], m[0]))
    d = _psub(_psub(_pmul(k[0], c1), _pmul(k[1], c2)), -_pmul(k[2], c3))
    return (k, l, m), d


def _peval(p, z):
    """Ascending coefficients [B, n], points [B] -> [B] (Horner)."""
    v = p[:, -1].copy()
    for i in range(p.shape[1] - 2, -1, -1):
        v = v * z + p[:, i]
    return v


def sturm(d):
    """Sturm chain of d (ascending [B, 11]) assuming every remainder has full degree, each scaled to max |coef| = 1
    -> (list of 11 descending arrays of length 11 .. 1, ok [B])."""
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        p0 = d[:, ::-1]
        p1 = p0[:, :-1] * np.arange(10, 0, -1)[None, :]
        chain = []
        for p in (p0, p1):
            s = np.abs(p).max(1, keepdims=True)
            chain.append(p / np.where(s > 0, s, 1.0))
        for _ in range(9):
            a, b = chain[-2], chain[-1]
            q1 = a[:, 0] / b[:, 0]
            t = a[:, 1:] - q1[:, None] * np.concatenate([b[:, 1:], np.zeros((b.shape[0], 1))], 1)
            q0 = t[:, 0] / b[:, 0]
            r = -(t[:, 1:] - q0[:, None] * b[:, 1:])
            s = np.abs(r).max(1, keepdims=True)
            chain.append(r / np.where(s > 0, s, 1.0))
        ok = np.ones(d.shape[0], dtype=bool)
        for p in chain:
            ok &= np.isfinite(p).all(1) & (p[:, 0] != 0)
    return chain, ok


def _sign_changes(chain, z):
    """Sign changes of the chain at z [B] (zeros skipped)."""
    cnt = np.zeros(z.shape[0], dtype=np.int64)
    last = np.zeros(z.shape[0])
    with np.errstate(over='ignore', invalid='ignore'):
        for p in chain:
            v = p[:, 0].copy()
            for i in range(1, p.shape[1]):
                v = v * z + p[:, i]
            s = np.sign(v)
            cnt += (s != 0) & (last != 0) & (s != last)
            last = np.where(s != 0, s, last)
    return cnt


def real_roots(d):
    """Real roots of d (ascending [B, 11]) in (-zb, zb], zb = min(Cauchy bound, ZMAX) -> [B, 10] ascending (NaN = none)."""
    B = d.shape[0]
    out = np.full((B, 10), np.nan)
    chain, ok = sturm(d)
    with np.errstate(divide='ignore', invalid='ignore'):
        zb = np.minimum(1.0 + (np.abs(d[:, :10]) / np.abs(d[:, 10:11])).max(1), ZMAX)
    ok &= np.isfinite(zb)
    zb = np.where(ok, zb, 1.0)
    v_lo = _sign_changes(chain, -zb)
    nr = np.where(ok, v_lo - _sign_changes(chain, zb), 0)
    dd = d[:, 1:] * np.arange(1, 11)[None, :]
    for k in range(10):
        act = nr > k
        if not act.any():
            break
        lo, hi = -zb.copy(), zb.copy()
        for _ in range(BISECT):
            mid = 0.5 * (lo + hi)
            left = (v_lo - _sign_changes(chain, mid)) >= k + 1
            hi = np.where(left, mid, hi)
            lo = np.where(left, lo, mid)
        z = 0.5 * (lo + hi)
        w = hi - lo
        with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
            for _ in range(NEWTON):
                f, df = _peval(d, z), _peval(dd, z)
                step = f / df
                z = np.where((df != 0) & (np.abs(step) <= w), z - step, z)
        out[act, k] = z[act]
    return out


def solve_e5(P):
    """Normalised 5-point samples [B, 5, 4] -> (models [B, 10, 9] unit Frobenius norm, ascending z, valid [B, 10])."""
    B = P.shape[0]
    ns, ok = V.null_space(V.f7_rows(P))
    Bm, ok2 = gauss_jordan(constraints(ns))
    ok &= ok2
    (k, l, m), d = degree10(np.where(ok[:, None, None], Bm, 0.0))
    d = np.where(ok[:, None], d, 0.0)
    z = real_roots(d)
    models = np.zeros((B, 10, 9))
    valid = np.zeros((B, 10), dtype=bool)
    for r in range(10):
        zr = np.where(np.isnan(z[:, r]), 0.0, z[:, r])
        rows = np.stack([np.stack([_peval(p, zr) for p in q], -1) for q in (k, l, m)], 1)   # [B, 3, 3]
        cr = [np.cross(rows[:, 0], rows[:, 1]), np.cross(rows[:, 0], rows[:, 2]), np.cross(rows[:, 1], rows[:, 2])]
        nrm = np.stack([(c * c).sum(1) for c in cr], 1)
        v = np.stack(cr, 1)[np.arange(B), nrm.argmax(1)]
        with np.errstate(divide='ignore', invalid='ignore'):
            x, y = v[:, 0] / v[:, 2], v[:, 1] / v[:, 2]
            E = x[:, None] * ns[:, 0] + y[:, None] * ns[:, 1] + zr[:, None] * ns[:, 2] + ns[:, 3]
            E = E / np.linalg.norm(E, axis=1, keepdims=True)
        good = ok & ~np.isnan(z[:, r]) & np.isfinite(E).all(1)
        models[:, r] = np.where(good[:, None], E, 0.0)
        valid[:, r] = good
    return models, valid


def hypotheses(cam, hyps, seed):
    """Models of the given hypotheses on normalised rows -> (models [len(hyps) * 10, 3, 3], valid), slot layout as on
    the device (the k-th valid model of hypothesis i in slot i * 10 + k)."""
    idx, ok = V.draw_samples(seed, hyps, cam.shape[0], SAMPLE)
    models, valid = solve_e5(cam[idx])
    valid &= ok[:, None]
    B = len(hyps)
    order = np.argsort(~valid, axis=1, kind='stable')
    bi = np.arange(B)[:, None]
    vs = np.take_along_axis(valid, order, 1)
    models = np.where(vs[..., None], models[bi, order], 0.0)
    return models.reshape(B * SLOTS, 3, 3), vs.reshape(B * SLOTS)


def errors(models, cam):
    """Sampson error (no eps) of every (model, normalised row) pair in fp64."""
    return V.errors(0, models, cam)


def threshold(px_th, intr):
    """cv2.findEssentialMat's rule: the pixel threshold over the mean focal length (of view 2)."""
    return float(px_th) / ((float(intr[4]) + float(intr[5])) / 2.0)


def project_essential(M):
    U, _, Vt = np.linalg.svd(np.asarray(M, dtype=np.float64).reshape(3, 3))
    E = U @ np.diag([1.0, 1.0, 0.0]) @ Vt
    return E / np.linalg.norm(E)


def refit(cam, mask):
    """8-point fit on the rows under `mask`, projected onto the essential manifold, unit Frobenius norm."""
    A = V.f7_rows(cam[mask])
    _, W = np.linalg.eigh(A.T @ A)
    return project_essential(W[:, 0])


def find_essential(rows, intr, px_th, conf=0.999, max_iters=1000, seed=0, trace=None):
    """-> (E 3x3 or None, bool mask [n], inlier count), E relating normalised coordinates (x2^T E x1 = 0).  `trace`
    (a dict, optional) receives the winner's slot, its count before LO, its margin over the runner-up and the number
    of hypotheses drawn."""
    rows = np.asarray(rows, dtype=np.float64)
    n = rows.shape[0]
    if not np.isfinite(rows).all():
        raise ValueError('non-finite coordinate')
    if n < SAMPLE:
        return None, np.zeros(n, dtype=bool), 0
    cam = to_camera(rows, intr)
    th = threshold(px_th, intr)
    th2 = th * th
    best, best_count, best_slot, done, top = None, 0, -1, 0, [0, 0]
    for first in range(0, max_iters, ROUND):
        count = min(ROUND, max_iters - first)
        models, valid = hypotheses(cam, np.arange(first, first + count), seed)
        counts = np.where(valid, V.count_inliers(0, models, cam, th2), -1)
        c = int(counts.max())
        top = sorted(top + sorted(counts.tolist())[-2:])[-2:]
        if c > best_count:
            m = int(np.argmax(counts))
            best, best_count, best_slot = models[m], c, first * SLOTS + m
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
    cur, cur_mask = best, errors(best, cam)[0] < th2
    cur_count = int(cur_mask.sum())
    for _ in range(LO_ITERS):
        if cur_count < LO_MIN:
            break
        cand = refit(cam, cur_mask)
        cand_mask = errors(cand, cam)[0] < th2
        if int(cand_mask.sum()) <= cur_count:
            break
        cur, cur_mask, cur_count = cand, cand_mask, int(cand_mask.sum())
    return cur, cur_mask, cur_count


def decompose(E):
    """cv2.decomposeEssentialMat -> (R1, R2, t)."""
    U, _, Vt = np.linalg.svd(np.asarray(E, dtype=np.float64).reshape(3, 3))
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    return U @ W @ Vt, U @ W.T @ Vt, U[:, 2].copy()


def good_points(R, t, cam, dist_th=DIST_TH):
    """Linear triangulation against [I|0] and [R|t] (smallest eigenvector of the 4x4 normal matrix) and
    cv2.recoverPose's cheirality / distance test -> bool [n]."""
    x1, y1, x2, y2 = cam[:, 0], cam[:, 1], cam[:, 2], cam[:, 3]
    P0 = np.eye(3, 4)
    P1 = np.concatenate([R, t.reshape(3, 1)], 1)
    A = np.stack([x1[:, None] * P0[2] - P0[0], y1[:, None] * P0[2] - P0[1],
                  x2[:, None] * P1[2] - P1[0], y2[:, None] * P1[2] - P1[1]], 1)     # [n, 4, 4]
    _, W = np.linalg.eigh(np.transpose(A, (0, 2, 1)) @ A)
    Q = W[:, :, 0]
    with np.errstate(divide='ignore', invalid='ignore'):
        X = Q[:, :3] / Q[:, 3:4]
        z2 = X @ R[2] + t[2]
        return (Q[:, 2] * Q[:, 3] > 0) & (X[:, 2] < dist_th) & (z2 > 0) & (z2 < dist_th)


def recover_pose(E, rows, intr, mask=None, dist_th=DIST_TH):
    """cv2.recoverPose -> (n_good, R, t [3], good mask).  A zero E gives (0, zeros, zeros, empty mask)."""
    rows = np.asarray(rows, dtype=np.float64)
    n = rows.shape[0]
    E = np.asarray(E, dtype=np.float64).reshape(3, 3)
    if not (np.isfinite(E).all() and np.abs(E).max() > 0):
        return 0, np.zeros((3, 3)), np.zeros(3), np.zeros(n, dtype=bool)
    cam = to_camera(rows, intr)
    m = np.ones(n, dtype=bool) if mask is None else np.asarray(mask).astype(bool)
    R1, R2, t = decompose(E)
    cands = [(R1, t), (R2, t), (R1, -t), (R2, -t)]
    goods = [good_points(R, tt, cam, dist_th) & m for R, tt in cands]
    counts = [int(g.sum()) for g in goods]
    b = int(np.argmax(counts))                    # first maximum = OpenCV's order
    return counts[b], cands[b][0], cands[b][1], goods[b]
