"""numpy fp64 restatement of model 2 of p2p_find_model (patch2pix_b200/csrc/degensac.cu: F RANSAC with the DEGENSAC
degeneracy check) and of p2p_test_degeneracy, for tests only.

Rounds, scoring, selection, stopping bound and LO are those of model 0 (oracle/verify_oracle.py).  In each round the
records -- the slots a sequential RANSAC would adopt, in slot order -- have their 7-point samples tested for
H-degeneracy until one is degenerate: for each triplet of TRIPLETS the homography induced by F and the three points
(Hartley & Zisserman, result 13.6) is built in normalised coordinates, and the sample is degenerate when at least
DEG_MIN of its 7 points lie within h_th = H_FACTOR * px_th of it (one-sided transfer error).  After the round's select,
that H is refitted on its inliers (DLT while the count grows) and one round of ROUND plane-and-parallax models
F = [e']x H is drawn from a second stream of the sample generator (rows within h_th of H re-drawn); a parallax model is
adopted when it has strictly more inliers.  Differences from the device: F scoring is fp64 here (fp32 there), and the
smallest eigenvectors come from numpy.linalg.eigh (Jacobi there).
"""
import numpy as np

from . import verify_oracle as V

ROUND = V.ROUND
H_FACTOR = 2.0
DEG_MIN = 5
TRIPLETS = ((0, 1, 2), (3, 4, 5), (0, 1, 6), (3, 4, 6), (2, 5, 6))
PARALLAX_KEY = 0x5851F42D4C957F2D          # the parallax stream draws with seed ^ PARALLAX_KEY


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def epipole2(F):
    """Unit e' with F^T e' = 0: the largest of the cross products of F's column pairs, or None when all vanish."""
    c = [F[:, 0], F[:, 1], F[:, 2]]
    cands = [np.cross(c[0], c[1]), np.cross(c[0], c[2]), np.cross(c[1], c[2])]
    nrm = [float(np.sqrt(x @ x)) for x in cands]
    k = int(np.argmax(nrm))                           # first of equal norms, as the device
    if not nrm[k] > 1e-10 * float((F * F).sum()):
        return None
    return cands[k] / nrm[k]


def induced_homography(F, p):
    """H = A - e' (M^-1 b)^T with A = [e']x F, M the rows x_i^T and b_i = (x'_i x A x_i)^T (x'_i x e') / |x'_i x e'|^2
    (Hartley & Zisserman, result 13.6) from three rows p [3, 4] (x, y, x', y') in the coordinates of F -> H or None
    (vanishing e', a point at the epipole, or collinear x_i)."""
    e = epipole2(F)
    if e is None:
        return None
    A = _skew(e) @ F
    M = np.stack([np.array([q[0], q[1], 1.0]) for q in p])
    b = np.zeros(3)
    for i, q in enumerate(p):
        x2 = np.array([q[2], q[3], 1.0])
        c = np.cross(x2, e)
        cc = float(c @ c)
        if not cc > 1e-12 * float(x2 @ x2):
            return None
        b[i] = float(np.cross(x2, A @ M[i]) @ c) / cc
    det = np.linalg.det(M)
    if not abs(det) > 1e-10 * np.prod(np.sqrt((M * M).sum(1))):
        return None
    return A - np.outer(e, np.linalg.solve(M, b))


def normalise_f(F, T):
    """Pixel F -> T2^-T F T1^-1, F in the Hartley-normalised coordinates of T."""
    (c1x, c1y, s1), (c2x, c2y, s2) = T
    T1i = np.array([[1 / s1, 0, c1x], [0, 1 / s1, c1y], [0, 0, 1.0]])
    T2it = np.array([[1 / s2, 0, 0], [0, 1 / s2, 0], [c2x, c2y, 1.0]])
    return T2it @ np.asarray(F, dtype=np.float64).reshape(3, 3) @ T1i


def degeneracy(F, rows7, T, h_th2):
    """H-degeneracy test of a 7-point sample rows7 [7, 4] (pixels) of the pixel F -> (first degenerate triplet or -1,
    its H in pixels at H[2][2] = 1 or None)."""
    Fn = normalise_f(F, T)
    P = V.normalise(rows7, T)
    for k, tri in enumerate(TRIPLETS):
        Hn = induced_homography(Fn, P[list(tri)])
        if Hn is None:
            continue
        H, ok = V.denormalise(1, Hn.reshape(9), T)
        if not ok[0]:
            continue
        if int((V.errors(1, H[0], rows7)[0] < h_th2).sum()) >= DEG_MIN:
            return k, H[0]
    return -1, None


def degeneracy_hypotheses(rows, T, hyps, seed, px_th):
    """Per slot of the given hypotheses (slot layout of verify_oracle.hypotheses): -2 no model, -1 not degenerate, else
    the first degenerate triplet; and its H (zeros otherwise)."""
    models, valid = V.hypotheses(0, rows, T, hyps, seed)
    idx, _ = V.draw_samples(seed, hyps, rows.shape[0], 7)
    h_th2 = (H_FACTOR * px_th) ** 2
    tri = np.full(len(models), -2, dtype=np.int64)
    Hs = np.zeros((len(models), 3, 3))
    for s in np.nonzero(valid)[0]:
        k, H = degeneracy(models[s], rows[idx[s // 3]], T, h_th2)
        tri[s] = k
        if H is not None:
            Hs[s] = H
    return tri, Hs


def plane_refit(rows, H, T, h_th2):
    """DLT refit of H on the rows within h_th, kept while the count grows (at most LO_ITERS refits)."""
    mask = V.errors(1, H, rows)[0] < h_th2
    count = int(mask.sum())
    for _ in range(V.LO_ITERS):
        if count < V.LO_MIN[1]:
            break
        cand = V.refit(1, rows, mask, T)
        if cand is None:
            break
        cmask = V.errors(1, cand, rows)[0] < h_th2
        if int(cmask.sum()) <= count:
            break
        H, mask, count = cand, cmask, int(cmask.sum())
    return H


def parallax_hypotheses(rows, H, hyps, seed, h_th2):
    """Plane-and-parallax models of the given hypotheses of the parallax stream -> (F [B, 3, 3] pixels at unit Frobenius
    norm, valid [B]).  Each draws two distinct rows that are not within h_th of H (a rejected draw is re-drawn, at most
    MAX_DRAWS draws), e' = (H x_a x x'_a) x (H x_b x x'_b) and F = [e']x H."""
    n = rows.shape[0]
    hyps = np.asarray(hyps, dtype=np.int64)
    B = len(hyps)
    hin = V.errors(1, H, rows)[0] < h_th2
    D = V.draw_index(int(seed) ^ PARALLAX_KEY, hyps[:, None], np.arange(V.MAX_DRAWS)[None, :], n)
    okd = ~hin[D]
    ia = np.argmax(okd, 1)
    a = D[np.arange(B), ia]
    okb = okd & (D != a[:, None]) & (np.arange(V.MAX_DRAWS)[None, :] > ia[:, None])
    ib = np.argmax(okb, 1)
    b = D[np.arange(B), ib]
    ok = okd.any(1) & okb.any(1)
    X1 = np.concatenate([rows[:, :2], np.ones((n, 1))], 1)
    X2 = np.concatenate([rows[:, 2:4], np.ones((n, 1))], 1)
    la = np.cross(X1[a] @ H.T, X2[a])
    lb = np.cross(X1[b] @ H.T, X2[b])
    e = np.cross(la, lb)
    ok &= np.sqrt((e * e).sum(1)) > 1e-12 * np.sqrt((la * la).sum(1) * (lb * lb).sum(1))
    F = np.stack([_skew(x) @ H for x in e])
    nrm = np.sqrt((F * F).sum((1, 2)))
    ok &= nrm > 0
    return F / np.where(ok, nrm, 1.0)[:, None, None], ok


def find_model(rows, px_th, conf=0.999, max_iters=10000, seed=0, trace=None):
    """Model 2 -> (F or None, bool mask [n], inlier count).  `trace` (a dict, optional) receives the winner's count
    before LO, its margin over the runner-up model, the number of hypotheses drawn and the number of parallax rounds."""
    rows = np.asarray(rows, dtype=np.float64)
    n = rows.shape[0]
    if not np.isfinite(rows).all():
        raise ValueError('non-finite coordinate')
    s, sl = 7, 3
    if n < s:
        return None, np.zeros(n, dtype=bool), 0
    th2 = float(px_th) ** 2
    h_th2 = (H_FACTOR * float(px_th)) ** 2
    T = V.normalisation(rows)
    best, best_count, done, top, events = None, 0, 0, [0, 0], 0
    for first in range(0, max_iters, ROUND):
        count = min(ROUND, max_iters - first)
        models, valid = V.hypotheses(0, rows, T, np.arange(first, first + count), seed)
        counts = np.where(valid, V.count_inliers(0, models, rows, th2), -1)
        top = sorted(top + sorted(counts.tolist())[-2:])[-2:]
        # the round's records, as sequential RANSAC would adopt them: slots beating the best so far, in slot order
        run = np.maximum.accumulate(np.concatenate([[best_count], counts]))[:-1]
        H = None
        for m in np.nonzero(counts > run)[0]:
            idx, _ = V.draw_samples(seed, [first + m // sl], n, s)
            k, H = degeneracy(models[m], rows[idx[0]], T, h_th2)
            if k >= 0:
                break
        c = int(counts.max())
        if c > best_count:
            best, best_count = models[int(np.argmax(counts))], c
        if H is not None:
            events += 1
            H = plane_refit(rows, H, T, h_th2)
            pm, pv = parallax_hypotheses(rows, H, np.arange(first, first + ROUND), seed, h_th2)
            pc = np.where(pv, V.count_inliers(0, pm, rows, th2), -1)
            top = sorted(top + sorted(pc.tolist())[-2:])[-2:]
            c2 = int(pc.max())
            if c2 > best_count:
                best, best_count = pm[int(np.argmax(pc))], c2
        done = first + count
        needed = np.inf
        if best_count > 0:
            ws = (best_count / n) ** s
            needed = 0.0 if ws >= 1 else np.log(1.0 - conf) / np.log1p(-ws)
        if done >= max_iters or done >= needed:
            break
    if trace is not None:
        trace.update(ransac_count=best_count, margin=top[1] - top[0], hypotheses=done, parallax_rounds=events)
    if best is None:
        return None, np.zeros(n, dtype=bool), 0
    cur, cur_mask = best, V.errors(0, best, rows)[0] < th2
    cur_count = int(cur_mask.sum())
    for _ in range(V.LO_ITERS):
        if cur_count < V.LO_MIN[0]:
            break
        cand = V.refit(0, rows, cur_mask, T)
        if cand is None:
            break
        cand_mask = V.errors(0, cand, rows)[0] < th2
        if int(cand_mask.sum()) <= cur_count:
            break
        cur, cur_mask, cur_count = cand, cand_mask, int(cand_mask.sum())
    return cur, cur_mask, cur_count
