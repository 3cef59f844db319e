"""numpy fp64 restatement of patch2pix_b200/csrc/verify.cu (p2p_find_model, p2p_sampson_distance), for tests only.

Same sample generator, Hartley normalisation, minimal solvers (full-pivoting Gauss-Jordan null space, the 7-point cubic
from its values at lambda = 0, 1, -1, 2, the 4-point DLT with its collinearity / orientation rejection), rounds of
1024 hypotheses with the same stopping bound, tie rule and local optimisation.  Differences from the device: scoring is
fp64 here (fp32 there), and the smallest eigenvector comes from numpy.linalg.eigh (Jacobi there).
"""
import numpy as np

ROUND = 1024
MAX_DRAWS = 64
LO_ITERS = 4
SAMPLE = {0: 7, 1: 4}
SLOTS = {0: 3, 1: 1}
LO_MIN = {0: 8, 1: 4}
_M64 = (1 << 64) - 1


def _mix64(z):
    z = z.astype(np.uint64)
    with np.errstate(over='ignore'):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def draw_index(seed, hyp, draw, n):
    """Index `draw` of hypothesis `hyp` (arrays broadcast) in [0, n)."""
    hyp = np.asarray(hyp, dtype=np.uint64)
    draw = np.asarray(draw, dtype=np.uint64)
    with np.errstate(over='ignore'):
        key = (np.uint64((int(seed) * 0xD1B54A32D192ED03) & _M64)
               + (hyp * np.uint64(MAX_DRAWS) + draw) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0x632BE59BD9B4E019))
    return (((_mix64(key) >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def draw_samples(seed, hyps, n, s):
    """[len(hyps), s] distinct indices per hypothesis (a repeat is re-drawn) and a validity flag (False after
    MAX_DRAWS draws)."""
    hyps = np.asarray(hyps, dtype=np.int64)
    B = hyps.shape[0]
    idx = np.zeros((B, s), dtype=np.int64)
    d = np.zeros(B, dtype=np.int64)
    ok = np.ones(B, dtype=bool)
    for k in range(s):
        todo = np.ones(B, dtype=bool)
        while True:
            todo &= ok
            if not todo.any():
                break
            ok &= ~(todo & (d >= MAX_DRAWS))
            todo &= ok
            v = draw_index(seed, hyps, d, n)
            idx[todo, k] = v[todo]
            d[todo] += 1
            dup = (idx[:, :k] == idx[:, k:k + 1]).any(1) if k else np.zeros(B, dtype=bool)
            todo &= dup
    return idx, ok


def normalisation(rows):
    """Hartley: per image, centroid to the origin and mean distance sqrt(2) -> (cx, cy, s) for images 1 and 2."""
    out = []
    for c in (0, 2):
        cx, cy = rows[:, c].mean(), rows[:, c + 1].mean()
        md = np.sqrt((rows[:, c] - cx) ** 2 + (rows[:, c + 1] - cy) ** 2).mean()
        out.append((cx, cy, np.sqrt(2.0) / md if md > 0 else 1.0))
    return out


def normalise(rows, T):
    (c1x, c1y, s1), (c2x, c2y, s2) = T
    return np.stack([(rows[..., 0] - c1x) * s1, (rows[..., 1] - c1y) * s1,
                     (rows[..., 2] - c2x) * s2, (rows[..., 3] - c2y) * s2], -1)


def null_space(A):
    """Batched full-pivoting Gauss-Jordan: A [B, R, 9] -> (ns [B, 9 - R, 9], ok [B])."""
    A = np.array(A, dtype=np.float64)
    B, R, _ = A.shape
    bi = np.arange(B)
    perm = np.tile(np.arange(9), (B, 1))
    amax0 = np.abs(A).reshape(B, -1).max(1)
    ok = amax0 > 0
    for k in range(R):
        sub = np.abs(A[:, k:, k:]).reshape(B, -1)
        flat = sub.argmax(1)
        best = sub[bi, flat]
        ok &= best > 1e-9 * amax0
        p, q = k + flat // (9 - k), k + flat % (9 - k)
        rk = A[bi, k].copy()
        A[bi, k] = A[bi, p]
        A[bi, p] = rk
        ck = A[bi, :, k].copy()
        A[bi, :, k] = A[bi, :, q]
        A[bi, :, q] = ck
        pk = perm[bi, k].copy()
        perm[bi, k] = perm[bi, q]
        perm[bi, q] = pk
        piv = np.where(ok, A[:, k, k], 1.0)
        A[:, k] /= piv[:, None]
        f = A[:, :, k].copy()
        f[:, k] = 0.0
        A -= f[:, :, None] * A[:, k:k + 1, :]
    ns = np.zeros((B, 9 - R, 9))
    for f in range(9 - R):
        ns[bi, f, perm[:, R + f]] = 1.0
        for i in range(R):
            ns[bi, f, perm[:, i]] = -A[:, i, R + f]
    return ns, ok


def cubic_roots(a3, a2, a1, a0):
    m = max(abs(a3), abs(a2), abs(a1), abs(a0))
    if not m > 0:
        return []
    if abs(a3) <= 1e-12 * m:
        if abs(a2) <= 1e-12 * m:
            return [] if abs(a1) <= 1e-12 * m else [-a0 / a1]
        disc = a1 * a1 - 4.0 * a2 * a0
        if disc < 0:
            return []
        qq = -0.5 * (a1 + np.copysign(np.sqrt(disc), a1))
        return [qq / a2] if qq == 0 else [qq / a2, a0 / qq]
    b, c, d = a2 / a3, a1 / a3, a0 / a3
    p = c - b * b / 3.0
    q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    shift = -b / 3.0
    disc = q * q / 4.0 + p * p * p / 27.0
    if disc > 0:
        sq = np.sqrt(disc)
        return [np.cbrt(-q / 2.0 + sq) + np.cbrt(-q / 2.0 - sq) + shift]
    if p >= 0:
        return [shift]
    rr = 2.0 * np.sqrt(-p / 3.0)
    phi = np.arccos(min(1.0, max(-1.0, 1.5 * q / p * np.sqrt(-3.0 / p)))) / 3.0
    return [rr * np.cos(phi - 2.0943951023931957 * k) + shift for k in range(3)]


def f7_rows(p):
    x1, y1, x2, y2 = p[..., 0], p[..., 1], p[..., 2], p[..., 3]
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones_like(x1)], -1)


def h4_rows(p):
    x, y, u, v = p[..., 0], p[..., 1], p[..., 2], p[..., 3]
    o, z = np.ones_like(x), np.zeros_like(x)
    r0 = np.stack([-x, -y, -o, z, z, z, u * x, u * y, u], -1)
    r1 = np.stack([z, z, z, -x, -y, -o, v * x, v * y, v], -1)
    return np.stack([r0, r1], -2).reshape(*x.shape[:-1], 2 * x.shape[-1], 9)


def _polish_sorted(coef, roots):
    """Two Newton steps per root of the cubic with coefficients coef = (a3, a2, a1, a0) [B] each, then ascending order
    (NaN = no root, last)."""
    a3, a2, a1, a0 = (c[:, None] for c in coef)
    r = roots.copy()
    for _ in range(2):
        f = ((a3 * r + a2) * r + a1) * r + a0
        df = (3.0 * a3 * r + 2.0 * a2) * r + a1
        with np.errstate(divide='ignore', invalid='ignore'):
            r = np.where(df != 0, r - f / np.where(df != 0, df, 1.0), r)
    return np.sort(r, 1)


def cubic_roots_batch(a3, a2, a1, a0):
    """Batched cubic_roots -> [B, 3] roots (NaN = none), polished and ascending."""
    B = a3.shape[0]
    out = np.full((B, 3), np.nan)
    m = np.maximum(np.maximum(np.abs(a3), np.abs(a2)), np.maximum(np.abs(a1), np.abs(a0)))
    drop = (m > 0) & (np.abs(a3) <= 1e-12 * m)
    for b in np.nonzero(drop)[0]:
        r = cubic_roots(a3[b], a2[b], a1[b], a0[b])
        out[b, :len(r)] = r
    full = (m > 0) & ~drop
    with np.errstate(divide='ignore', invalid='ignore'):
        b_, c_, d_ = a2 / a3, a1 / a3, a0 / a3
        p = c_ - b_ * b_ / 3.0
        q = 2.0 * b_ * b_ * b_ / 27.0 - b_ * c_ / 3.0 + d_
        shift = -b_ / 3.0
        disc = q * q / 4.0 + p * p * p / 27.0
        one = full & (disc > 0)
        sq = np.sqrt(np.where(one, disc, 0.0))
        out[one, 0] = (np.cbrt(-q / 2.0 + sq) + np.cbrt(-q / 2.0 - sq) + shift)[one]
        triple = full & ~(disc > 0) & (p >= 0)
        out[triple, 0] = shift[triple]
        three = full & ~(disc > 0) & ~(p >= 0)
        pp = np.where(three, p, -1.0)
        rr = 2.0 * np.sqrt(-pp / 3.0)
        phi = np.arccos(np.clip(1.5 * q / pp * np.sqrt(-3.0 / pp), -1.0, 1.0)) / 3.0
        for k in range(3):
            out[three, k] = (rr * np.cos(phi - 2.0943951023931957 * k) + shift)[three]
    return _polish_sorted((a3, a2, a1, a0), out)


def solve_f7(ns):
    """2-D null spaces [B, 2, 9] -> [B, 3, 9] normalised F (ascending lambda of det(l F1 + (1 - l) F2) = 0) and
    [B, 3] validity."""
    N1, N2 = ns[:, 0], ns[:, 1]
    D = N1 - N2
    v = [np.linalg.det((N2 + l * D).reshape(-1, 3, 3)) for l in (0.0, 1.0, -1.0, 2.0)]
    a0, a2, odd = v[0], 0.5 * (v[1] + v[2]) - v[0], 0.5 * (v[1] - v[2])
    a3 = (v[3] - v[0] - 4.0 * a2 - 2.0 * odd) / 6.0
    a1 = odd - a3
    r = cubic_roots_batch(a3, a2, a1, a0)
    ok = ~np.isnan(r)
    return N2[:, None, :] + np.where(ok, r, 0.0)[:, :, None] * D[:, None, :], ok


def h4_sample_ok(P):
    """Collinearity / orientation-consistency test of normalised 4-point samples [B, 4, 4] -> [B] bool."""
    ok = np.ones(P.shape[0], dtype=bool)
    signs = []
    for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
        o = [(P[:, b, i] - P[:, a, i]) * (P[:, c, i + 1] - P[:, a, i + 1])
             - (P[:, b, i + 1] - P[:, a, i + 1]) * (P[:, c, i] - P[:, a, i]) for i in (0, 2)]
        ok &= (np.abs(o[0]) > 1e-6) & (np.abs(o[1]) > 1e-6)
        signs.append((o[0] > 0) == (o[1] > 0))
    return ok & np.all(np.stack(signs) == signs[0], 0)


def denormalise(kind, mn, T):
    """Normalised models [..., 9] -> pixel models [..., 3, 3] and validity (F: T2^T Fn T1 at unit Frobenius norm;
    H: T2^-1 Hn T1 at H[2][2] = 1)."""
    (c1x, c1y, s1), (c2x, c2y, s2) = T
    T1 = np.array([[s1, 0, -s1 * c1x], [0, s1, -s1 * c1y], [0, 0, 1.0]])
    M = np.asarray(mn, dtype=np.float64).reshape(-1, 3, 3)
    with np.errstate(divide='ignore', invalid='ignore'):
        if kind == 0:
            T2 = np.array([[s2, 0, -s2 * c2x], [0, s2, -s2 * c2y], [0, 0, 1.0]])
            F = T2.T @ (M @ T1)
            nrm = np.sqrt((F * F).sum((1, 2)))
            ok = nrm > 0
            return F / np.where(ok, nrm, 1.0)[:, None, None], ok
        T2i = np.array([[1 / s2, 0, c2x], [0, 1 / s2, c2y], [0, 0, 1.0]])
        H = T2i @ (M @ T1)
        ok = np.abs(H[:, 2, 2]) > 1e-12 * np.abs(H).reshape(-1, 9).max(1)
        H = H / np.where(ok, H[:, 2, 2], 1.0)[:, None, None]
        H[:, 2, 2] = 1.0
        return H, ok


def hypotheses(kind, rows, T, hyps, seed):
    """Models of the given hypotheses -> (models [len(hyps) * slots, 3, 3], valid [len(hyps) * slots]), slot layout as
    on the device (the k-th valid model of hypothesis i in slot i * slots + k)."""
    s, sl = SAMPLE[kind], SLOTS[kind]
    idx, ok = draw_samples(seed, hyps, rows.shape[0], s)
    P = normalise(rows[idx], T)                                   # [B, s, 4]
    ns, ok2 = null_space(f7_rows(P) if kind == 0 else h4_rows(P))
    ok &= ok2
    B = len(hyps)
    if kind == 0:
        mn, okr = solve_f7(ns)                                   # [B, 3, 9]
        okr &= ok[:, None]
    else:
        mn, okr = ns[:, :1], (ok & h4_sample_ok(P))[:, None]
    M, okd = denormalise(kind, mn.reshape(-1, 9), T)
    okr = okr.reshape(-1) & okd
    M, okr = M.reshape(B, sl, 3, 3), okr.reshape(B, sl)
    # compact each hypothesis' valid models to its first slots, as the device does
    order = np.argsort(~okr, axis=1, kind='stable')
    bi = np.arange(B)[:, None]
    models = np.where(np.take_along_axis(okr, order, 1)[..., None, None], M[bi, order], 0.0)
    return models.reshape(B * sl, 3, 3), np.take_along_axis(okr, order, 1).reshape(B * sl)


def errors(kind, models, rows):
    """Per (model, row) error in fp64: F the Sampson error without eps, H the squared one-sided transfer error
    (inf where the third coordinate of H x1 is not above 1e-8)."""
    M = np.asarray(models, dtype=np.float64).reshape(-1, 9)
    x1, y1, x2, y2 = (rows[:, i][None, :] for i in range(4))
    m = [M[:, i][:, None] for i in range(9)]
    if kind == 0:
        l2x, l2y, l2z = m[0] * x1 + m[1] * y1 + m[2], m[3] * x1 + m[4] * y1 + m[5], m[6] * x1 + m[7] * y1 + m[8]
        l1x, l1y = m[0] * x2 + m[3] * y2 + m[6], m[1] * x2 + m[4] * y2 + m[7]
        dd = x2 * l2x + y2 * l2y + l2z
        with np.errstate(divide='ignore', invalid='ignore'):
            return dd * dd / (l1x * l1x + l1y * l1y + l2x * l2x + l2y * l2y)
    w = m[6] * x1 + m[7] * y1 + m[8]
    with np.errstate(divide='ignore', invalid='ignore'):
        u = (m[0] * x1 + m[1] * y1 + m[2]) / w - x2
        v = (m[3] * x1 + m[4] * y1 + m[5]) / w - y2
        return np.where(w > 1e-8, u * u + v * v, np.inf)


def count_inliers(kind, models, rows, th2, chunk=256):
    M = np.asarray(models).reshape(-1, 9)
    return np.concatenate([(errors(kind, M[i:i + chunk], rows) < th2).sum(1) for i in range(0, max(len(M), 1), chunk)])


def sampson_distance(rows, F, eps=1e-8):
    """utils/eval/measure.py:18-40."""
    p1 = np.concatenate([rows[:, 0:2], np.ones((rows.shape[0], 1))], 1)
    p2 = np.concatenate([rows[:, 2:4], np.ones((rows.shape[0], 1))], 1)
    F = np.asarray(F, dtype=np.float64).reshape(3, 3)
    l2 = F @ p1.T
    l1 = F.T @ p2.T
    dd = np.sum(l2.T * p2, 1)
    return dd ** 2 / (eps + l1[0] ** 2 + l1[1] ** 2 + l2[0] ** 2 + l2[1] ** 2)


def refit(kind, rows, mask, T):
    """Non-minimal fit on the rows under `mask` in normalised coordinates (F: 8-point + rank 2; H: DLT) -> pixel model
    or None."""
    P = normalise(rows[mask], T)
    A = f7_rows(P) if kind == 0 else h4_rows(P[None])[0]
    _, V = np.linalg.eigh(A.T @ A)
    h = V[:, 0]
    if kind == 0:
        Fn = h.reshape(3, 3)
        _, E = np.linalg.eigh(Fn.T @ Fn)
        e = E[:, 0]
        h = (Fn - np.outer(Fn @ e, e)).reshape(9)
    M, ok = denormalise(kind, h, T)
    return M[0] if ok[0] else None


def find_model(kind, rows, px_th, conf=0.999, max_iters=10000, seed=0, trace=None):
    """-> (model 3x3 or None, bool mask [n], inlier count).  `trace` (a dict, optional) receives the winner's
    hypothesis slot index, its count before LO, its margin over the runner-up model and the number of hypotheses
    drawn."""
    rows = np.asarray(rows, dtype=np.float64)
    n = rows.shape[0]
    if not np.isfinite(rows).all():
        raise ValueError('non-finite coordinate')
    s, sl = SAMPLE[kind], SLOTS[kind]
    if n < s:
        return None, np.zeros(n, dtype=bool), 0
    th2 = float(px_th) ** 2
    T = normalisation(rows)
    best, best_count, best_slot, done, top = None, 0, -1, 0, [0, 0]
    for first in range(0, max_iters, ROUND):
        count = min(ROUND, max_iters - first)
        models, valid = hypotheses(kind, rows, T, np.arange(first, first + count), seed)
        counts = np.where(valid, count_inliers(kind, models, rows, th2), -1)
        c = int(counts.max())
        top = sorted(top + sorted(counts.tolist())[-2:])[-2:]
        if c > best_count:
            m = int(np.argmax(counts))                    # first maximum = lowest (hypothesis, root) index
            best, best_count, best_slot = models[m], c, first * sl + m
        done = first + count
        needed = np.inf
        if best_count > 0:
            ws = (best_count / n) ** s
            needed = 0.0 if ws >= 1 else np.log(1.0 - conf) / np.log1p(-ws)
        if done >= max_iters or done >= needed:
            break
    if trace is not None:
        trace.update(slot=best_slot, ransac_count=best_count, margin=top[1] - top[0], hypotheses=done)
    if best is None:
        return None, np.zeros(n, dtype=bool), 0
    cur, cur_mask = best, errors(kind, best, rows)[0] < th2
    cur_count = int(cur_mask.sum())
    for _ in range(LO_ITERS):
        if cur_count < LO_MIN[kind]:
            break
        cand = refit(kind, rows, cur_mask, T)
        if cand is None:
            break
        cand_mask = errors(kind, cand, rows)[0] < th2
        if int(cand_mask.sum()) <= cur_count:
            break
        cur, cur_mask, cur_count = cand, cand_mask, int(cand_mask.sum())
    return cur, cur_mask, cur_count
