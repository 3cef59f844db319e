"""numpy restatement of csrc/sfm.cu (protocol in patch2pix_b200/sfm.py).  Every expression is written in the kernels'
order of operations; sfm.cu is compiled without fused multiply-add, so keypoint means, undistorted coordinates and
query rows agree bit for bit, and the rest up to the order of a few additions."""
import math

import numpy as np

CELLS = 1 << 22
UNDISTORT_ITERS = 12
GN_STEPS = 5
MAX_POINTS = 8
SAMPLE = 32
MAX_TRACK = 1 << 16


def _cells(img, x, y, px):
    with np.errstate(invalid='ignore'):
        ok = np.isfinite(x) & np.isfinite(y) & (x >= 0) & (y >= 0)
        cx = np.floor(np.where(ok, x, 0.0) / px)
        cy = np.floor(np.where(ok, y, 0.0) / px)
    ok &= (cx < CELLS) & (cy < CELLS)
    key = (np.asarray(img, np.uint64) << np.uint64(44)) | (cy.astype(np.uint64) << np.uint64(22)) | \
        cx.astype(np.uint64)
    return np.where(ok, key, np.uint64(2 ** 64 - 1)), ok


def endpoints(matches, pair_img, both=True):
    """(image, x, y) of the endpoints in order: pair, match, side."""
    img, xs, ys = [], [], []
    for p, m in enumerate(matches):
        m = np.asarray(m, dtype=np.float64).reshape(-1, 4)
        sides = (0, 1) if both else (0,)
        im = np.stack([np.full(len(m), pair_img[p][s]) for s in sides], 1).reshape(-1)
        x = np.stack([m[:, 2 * s] for s in sides], 1).reshape(-1)
        y = np.stack([m[:, 2 * s + 1] for s in sides], 1).reshape(-1)
        img.append(im)
        xs.append(x)
        ys.append(y)
    cat = (lambda a: np.concatenate(a) if a else np.zeros(0))
    return cat(img).astype(np.int64), cat(xs), cat(ys)


def keypoints(img, x, y, px):
    """-> kp_xy [n, 2], kp_key [n] uint64, kp_of_ep [E] (-1 dropped), dropped count."""
    key, ok = _cells(img, x, y, px)
    idx = np.nonzero(ok)[0]
    order = idx[np.argsort(key[idx], kind='stable')]
    sk = key[order]
    head = np.ones(len(sk), bool)
    head[1:] = sk[1:] != sk[:-1]
    starts = np.nonzero(head)[0]
    lens = np.diff(np.append(starts, len(sk)))
    sx = np.zeros(len(starts))
    sy = np.zeros(len(starts))
    for r in range(int(lens.max()) if len(lens) else 0):     # each run summed in order
        m = lens > r
        sx[m] = sx[m] + x[order[starts[m] + r]]
        sy[m] = sy[m] + y[order[starts[m] + r]]
    kp_of_ep = np.full(len(x), -1, np.int64)
    kp_of_ep[order] = np.cumsum(head) - 1
    return np.stack([sx / lens, sy / lens], 1), sk[starts], kp_of_ep, int(len(x) - len(idx))


def undistort(c, xd, yd):
    x = (xd - c[3]) / c[1]
    y = (yd - c[4]) / c[2]
    k1, k2 = c[5], c[6]
    u, v = x.copy(), y.copy()
    for _ in range(UNDISTORT_ITERS):
        u2, v2, uv = u * u, v * v, u * v
        r2 = u2 + v2
        rad = k1 * r2 + k2 * r2 * r2
        dr = k1 + 2.0 * k2 * r2
        fu = u + u * rad - x
        fv = v + v * rad - y
        a = 1.0 + rad + 2.0 * u2 * dr
        b = 2.0 * uv * dr
        d = 1.0 + rad + 2.0 * v2 * dr
        det = a * d - b * b
        u, v = u - (d * fu - b * fv) / det, v - (a * fv - b * fu) / det
    return u, v


def distort_px(c, u, v):
    r2 = u * u + v * v
    rad = c[5] * r2 + c[6] * r2 * r2
    return c[1] * (u + u * rad) + c[3], c[2] * (v + v * rad) + c[4]


def undistort_keypoints(kp_xy, kp_key, img_cam, cams):
    out = np.zeros_like(kp_xy)
    cam = np.asarray(img_cam)[(kp_key >> np.uint64(44)).astype(np.int64)]
    for c in np.unique(cam):
        m = cam == c
        out[m, 0], out[m, 1] = undistort(cams[c], kp_xy[m, 0], kp_xy[m, 1])
    return out


def edges(kp_of_ep, counts, E, thr, kp_n):
    """Kept unique edges [(lo, hi)] (sorted) and the count of first-in-pair matches."""
    ka_all, kb_all = kp_of_ep[0::2], kp_of_ep[1::2]
    out, n_first, o = set(), 0, 0
    for p, n in enumerate(counts):
        ka, kb = ka_all[o:o + n], kb_all[o:o + n]
        o += n
        first_a = np.zeros(n, bool)
        first_b = np.zeros(n, bool)
        va, vb = np.nonzero(ka >= 0)[0], np.nonzero(kb >= 0)[0]
        first_a[va[np.unique(ka[va], return_index=True)[1]]] = True
        first_b[vb[np.unique(kb[vb], return_index=True)[1]]] = True
        e = E[p]
        for m in np.nonzero(first_a & first_b)[0]:
            n_first += 1
            a0, a1 = kp_n[ka[m]]
            b0, b1 = kp_n[kb[m]]
            e0 = e[0] * a0 + e[1] * a1 + e[2]
            e1 = e[3] * a0 + e[4] * a1 + e[5]
            e2 = e[6] * a0 + e[7] * a1 + e[8]
            f0 = e[0] * b0 + e[3] * b1 + e[6]
            f1 = e[1] * b0 + e[4] * b1 + e[7]
            num = b0 * e0 + b1 * e1 + e2
            s = num * num / (e0 * e0 + e1 * e1 + f0 * f0 + f1 * f1)
            if s <= thr[p] and ka[m] != kb[m]:
                out.add((min(ka[m], kb[m]), max(ka[m], kb[m])))
    return sorted(out), n_first


def components(n_kp, edge_list):
    """Labels: the smallest keypoint id of each component (union-find)."""
    parent = np.arange(n_kp)

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    for a, b in edge_list:
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    return np.array([find(i) for i in range(n_kp)], dtype=np.int64)


def tracks(labels):
    """-> obs_kp (keypoints sorted by (label, id)), [(start, len)] of the tracks, rejected count."""
    obs = np.argsort(labels, kind='stable')
    lab = labels[obs]
    head = np.ones(len(lab), bool)
    head[1:] = lab[1:] != lab[:-1]
    starts = np.nonzero(head)[0]
    lens = np.diff(np.append(starts, len(lab)))
    keep = (lens >= 2) & (lens <= MAX_TRACK)
    return obs, list(zip(starts[keep], lens[keep])), int(np.sum(lens > MAX_TRACK))


# ---- triangulation -----------------------------------------------------------------------------------------------------
def _solve3(m, b):
    c00 = m[4] * m[8] - m[5] * m[5]
    c01 = m[2] * m[5] - m[1] * m[8]
    c02 = m[1] * m[5] - m[2] * m[4]
    c11 = m[0] * m[8] - m[2] * m[2]
    c12 = m[1] * m[2] - m[0] * m[5]
    c22 = m[0] * m[4] - m[1] * m[1]
    det = m[0] * c00 + m[1] * c01 + m[2] * c02
    if not (det != 0.0) or not math.isfinite(det):
        return None
    x = [(c00 * b[0] + c01 * b[1] + c02 * b[2]) / det, (c01 * b[0] + c11 * b[1] + c12 * b[2]) / det,
         (c02 * b[0] + c12 * b[1] + c22 * b[2]) / det]
    return x if all(math.isfinite(v) for v in x) else None


def _dlt(r, x, y, m, v):
    for q in range(2):
        s = x if q == 0 else y
        a0, a1, a2 = s * r[6] - r[3 * q], s * r[7] - r[3 * q + 1], s * r[8] - r[3 * q + 2]
        b = r[9 + q] - s * r[11]
        m[0] += a0 * a0; m[1] += a0 * a1; m[2] += a0 * a2
        m[4] += a1 * a1; m[5] += a1 * a2; m[8] += a2 * a2
        v[0] += a0 * b; v[1] += a1 * b; v[2] += a2 * b


def _cos_angle(ra, rb, X):
    d0 = [X[c] - ra[12 + c] for c in range(3)]
    d1 = [X[c] - rb[12 + c] for c in range(3)]
    dot = d0[0] * d1[0] + d0[1] * d1[1] + d0[2] * d1[2]
    n0 = d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2]
    n1 = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]
    return dot / math.sqrt(n0 * n1)


class _Track:
    def __init__(self, obs, kp_xy, kp_n, kp_img, recs, img_cam, cams, th2, cos_min):
        self.obs, self.img = obs, kp_img[obs]
        self.xy, self.n = kp_xy[obs], kp_n[obs]
        self.recs, self.cams, self.img_cam, self.th2, self.cos_min = recs, cams, img_cam, th2, cos_min
        r = recs[self.img]
        self.R, self.t = r[:, :9], r[:, 9:12]
        self.c = cams[np.asarray(img_cam)[self.img]]

    def err2(self, X):
        R, t = self.R, self.t
        p0 = R[:, 0] * X[0] + R[:, 1] * X[1] + R[:, 2] * X[2] + t[:, 0]
        p1 = R[:, 3] * X[0] + R[:, 4] * X[1] + R[:, 5] * X[2] + t[:, 1]
        p2 = R[:, 6] * X[0] + R[:, 7] * X[1] + R[:, 8] * X[2] + t[:, 2]
        with np.errstate(divide='ignore', invalid='ignore'):
            u, v = p0 / p2, p1 / p2
            r2 = u * u + v * v
            rad = self.c[:, 5] * r2 + self.c[:, 6] * r2 * r2
            px = self.c[:, 1] * (u + u * rad) + self.c[:, 3]
            py = self.c[:, 2] * (v + v * rad) + self.c[:, 4]
            dx, dy = px - self.xy[:, 0], py - self.xy[:, 1]
            e = dx * dx + dy * dy
        return np.where(p2 > 0, e, -1.0)

    def inliers(self, X, rem):
        e = self.err2(X)
        return rem & (e >= 0) & (e <= self.th2), e

    def score(self, X, rem):
        inl, _ = self.inliers(X, rem)
        return len(np.unique(self.img[inl]))

    def two_view(self, i, j):
        m, v = [0.0] * 9, [0.0] * 3
        ri, rj = self.recs[self.img[i]], self.recs[self.img[j]]
        _dlt(ri, self.n[i, 0], self.n[i, 1], m, v)
        _dlt(rj, self.n[j, 0], self.n[j, 1], m, v)
        m[3], m[6], m[7] = m[1], m[2], m[5]
        X = _solve3(m, v)
        if X is None:
            return None, False
        for r in (ri, rj):
            if not (r[6] * X[0] + r[7] * X[1] + r[8] * X[2] + r[11] > 0.0):
                return X, False
        return X, _cos_angle(ri, rj, X) <= self.cos_min

    def refine(self, X, sel):
        X = list(X)
        for _ in range(GN_STEPS):
            m, g = [0.0] * 9, [0.0] * 3
            for o in np.nonzero(sel)[0]:
                r = self.recs[self.img[o]]
                p0 = r[0] * X[0] + r[1] * X[1] + r[2] * X[2] + r[9]
                p1 = r[3] * X[0] + r[4] * X[1] + r[5] * X[2] + r[10]
                p2 = r[6] * X[0] + r[7] * X[1] + r[8] * X[2] + r[11]
                if not (p2 > 0.0):
                    continue
                u, v = p0 / p2, p1 / p2
                ru, rv = u - self.n[o, 0], v - self.n[o, 1]
                J = [[(r[c] - u * r[6 + c]) / p2 for c in range(3)], [(r[3 + c] - v * r[6 + c]) / p2 for c in range(3)]]
                for q, rq in ((0, ru), (1, rv)):
                    m[0] += J[q][0] * J[q][0]; m[1] += J[q][0] * J[q][1]; m[2] += J[q][0] * J[q][2]
                    m[4] += J[q][1] * J[q][1]; m[5] += J[q][1] * J[q][2]; m[8] += J[q][2] * J[q][2]
                    g[0] -= J[q][0] * rq; g[1] -= J[q][1] * rq; g[2] -= J[q][2] * rq
            m[3], m[6], m[7] = m[1], m[2], m[5]
            d = _solve3(m, g)
            if d is None:
                break
            X = [X[c] + d[c] for c in range(3)]
        return X

    def run(self):
        """-> [(X, inlier observation indices, mean error)] of the accepted points in round order."""
        n = len(self.obs)
        slot = np.full(n, -2)
        out = []
        for _ in range(MAX_POINTS):
            rem = slot == -2
            idx = np.nonzero(rem)[0]
            if len(np.unique(self.img[idx])) < 2:
                break
            s = idx[:SAMPLE]
            best = None
            for i in range(len(s)):
                for j in range(i + 1, len(s)):
                    if self.img[s[i]] == self.img[s[j]]:
                        continue
                    X, ok = self.two_view(s[i], s[j])
                    if not ok:
                        continue
                    sc = self.score(X, rem)
                    if best is None or sc > best[0]:
                        best = (sc, s[i], s[j], X)
            if best is None:
                break
            score, oi, oj, X = best
            inl, e = self.inliers(X, rem)
            sel = np.zeros(n, bool)
            for im in np.unique(self.img[inl]):
                cand = np.nonzero(inl & (self.img == im))[0]
                sel[cand[np.argmin(e[cand])]] = True       # argmin: the first of equal errors
            Y = self.refine(X, sel)
            if self.score(Y, rem) >= score:
                X = Y
            inl, e = self.inliers(X, rem)
            reps = [np.nonzero(inl & (self.img == im))[0][0] for im in np.unique(self.img[inl])]
            wide = any(_cos_angle(self.recs[self.img[a]], self.recs[self.img[b]], X) <= self.cos_min
                       for ai, a in enumerate(reps) for b in reps[ai + 1:])
            accept = len(reps) >= 2 and wide
            slot[inl] = len(out) if accept else -1
            if accept:
                err = 0.0
                for o in np.nonzero(inl)[0]:
                    err = err + math.sqrt(e[o])
                out.append((np.array(X), np.nonzero(inl)[0], err / inl.sum()))
            for o in (oi, oj):
                if slot[o] == -2:
                    slot[o] = -1
        return out


def triangulate(obs_kp, track_list, kp_xy, kp_n, kp_key, recs, img_cam, cams, reproj_px=4.0, min_angle=1.5):
    """-> points [m, 3], point_len [m], point_err [m], kp_point [n_kp], points numbered by (track, round)."""
    kp_img = (kp_key >> np.uint64(44)).astype(np.int64)
    cos_min = math.cos(math.radians(min_angle))
    kp_point = np.full(len(kp_xy), -1, np.int64)
    pts, plen, perr = [], [], []
    for s, l in track_list:
        obs = obs_kp[s:s + l]
        for X, inl, err in _Track(obs, kp_xy, kp_n, kp_img, recs, img_cam, cams, reproj_px * reproj_px,
                                  cos_min).run():
            kp_point[obs[inl]] = len(pts)
            pts.append(X)
            plen.append(len(inl))
            perr.append(err)
    return np.array(pts).reshape(-1, 3), np.array(plen, np.int64), np.array(perr), kp_point


# ---- query rows ----------------------------------------------------------------------------------------------------------
def query_rows(q_matches, q_pair_img, q_cams, kp_xy, kp_key, kp_point, points, px):
    """q_matches: one [n, 4] per (query, db) pair; q_pair_img (query index, db image) -> rows [r, 5], offsets
    [Q + 1]."""
    Q = len(q_cams)
    img, x, y = endpoints(q_matches, q_pair_img, both=False)
    q_xy, q_key, q_of, _ = keypoints(img, x, y, px)
    q_n = undistort_keypoints(q_xy, q_key, np.arange(Q), np.asarray(q_cams))
    lookup = {int(k): i for i, k in enumerate(kp_key)}
    qm = [np.asarray(m, np.float64).reshape(-1, 4) for m in q_matches]
    dbx = np.concatenate([m[:, 2] for m in qm]) if qm else np.zeros(0)
    dby = np.concatenate([m[:, 3] for m in qm]) if qm else np.zeros(0)
    dbimg = np.concatenate([np.full(len(m), b) for m, (_, b) in zip(qm, q_pair_img)]) if qm else np.zeros(0, np.int64)
    keys, ok = _cells(dbimg, dbx, dby, px)
    found = set()
    for m in range(len(x)):
        if q_of[m] < 0 or not ok[m]:
            continue
        k = int(keys[m])
        cx, cy, im = k & (CELLS - 1), (k >> 22) & (CELLS - 1), k >> 44
        best, best_d = -1, 0.0
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                ny, nx = cy + dy, cx + dx
                if ny < 0 or nx < 0 or ny >= CELLS or nx >= CELLS:
                    continue
                kk = lookup.get((im << 44) | (ny << 22) | nx)
                if kk is None or kp_point[kk] < 0:
                    continue
                ex, ey = kp_xy[kk, 0] - dbx[m], kp_xy[kk, 1] - dby[m]
                d = ex * ex + ey * ey
                if d <= px * px and (best < 0 or d < best_d or (d == best_d and kk < best)):
                    best, best_d = kk, d
        if best >= 0:
            found.add((int(q_of[m]), int(kp_point[best])))
    rows, qs = [], []
    for qk, p in sorted(found):
        q = int(q_key[qk] >> np.uint64(44))
        c = q_cams[q]
        rows.append([c[1] * q_n[qk, 0] + c[3], c[2] * q_n[qk, 1] + c[4], *points[p]])
        qs.append(q)
    offsets = np.searchsorted(np.array(qs, np.int64), np.arange(Q + 1))
    return np.array(rows, dtype=np.float64).reshape(-1, 5), offsets


def triangulate_host(model_tables, pair_tables, matches, merge_px=4.0, reproj_px=4.0, min_angle=1.5):
    """The whole triangulation of sfm._triangulate in numpy.  model_tables = (cams, img_cam, recs), pair_tables =
    (pair_img, E, thr) as sfm builds them."""
    cams, img_cam, recs = model_tables
    pair_img, E, thr = pair_tables
    img, x, y = endpoints(matches, pair_img)
    kp_xy, kp_key, kp_of_ep, dropped = keypoints(img, x, y, merge_px)
    kp_n = undistort_keypoints(kp_xy, kp_key, img_cam, cams)
    counts = [len(np.asarray(m).reshape(-1, 4)) for m in matches]
    edge_list, _ = edges(kp_of_ep, counts, E, thr, kp_n)
    labels = components(len(kp_xy), edge_list)
    obs_kp, track_list, rejected = tracks(labels)
    pts, plen, perr, kp_point = triangulate(obs_kp, track_list, kp_xy, kp_n, kp_key, recs, img_cam, cams, reproj_px,
                                            min_angle)
    return dict(kp_xy=kp_xy, kp_key=kp_key, kp_of_ep=kp_of_ep, kp_n=kp_n, dropped=dropped, edges=edge_list,
                labels=labels, obs_kp=obs_kp, tracks=track_list, rejected=rejected, points=pts, point_len=plen,
                point_err=perr, kp_point=kp_point)
