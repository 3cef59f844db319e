"""The fp32 inlier decisions of the RANSAC kernels (csrc/verify_common.cuh `is_inlier`, csrc/abspose.cu
`Kind<4>::inlier`) against float64: a derived per-row width outside which the two must agree, and numpy emulations of
the fp32 arithmetic, for tests only.

The kernels decide `L < R` on fp32 values: F / E `dd*dd < th2*den`, H `u'*u' + v'*v' < th2*w*w` behind `w > 1e-8f`,
absolute pose `eu*eu + ev*ev < th2*z*z` behind `z > 0`.  With exact values L - R = D (e - th2) for the fp64 error e
(D = den, w^2, z^2 > 0), so the decisions can differ only when D |e - th2| <= |dL| + |dR|.  `decision_bound` bounds
|dL| and |dR| by a running error bound over the kernels' own operations in source order: every input cast, product and
sum rounds once (relative u = 2^-24); a contracted FMA rounds once where the separate product and sum round twice, so
the bound holds with or without contraction (DESIGN.md, "RANSAC inlier decisions in fp32").
"""
import numpy as np

U = 2.0 ** -24                  # fp32 unit roundoff
U64 = 2.0 ** -53
ETA = 2.0 ** -149               # absolute error of a rounding into the fp32 subnormal range
GATE_H = float(np.float32(1e-8))


class _R:
    """A quantity of the fp32 evaluation: its exact value v (fp64) and a bound e on |fp32 value - v|."""
    __slots__ = ('v', 'e')

    def __init__(self, v, e):
        self.v, self.e = v, e

    def __add__(self, o):
        v = self.v + o.v
        e = self.e + o.e
        return _R(v, e + U * (np.abs(v) + e) + ETA)

    def __sub__(self, o):
        v = self.v - o.v
        e = self.e + o.e
        return _R(v, e + U * (np.abs(v) + e) + ETA)

    def __mul__(self, o):
        v = self.v * o.v
        e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
        return _R(v, e + U * (np.abs(v) + e) + ETA)


def _cast(x, e64=0.0):
    """fp32 cast of a value computed in fp64 (e64: a bound on that fp64 value's own error)."""
    x = np.asarray(x, dtype=np.float64)
    return _R(x, e64 + U * (np.abs(x) + e64) + ETA)


def _width(L, R, D, gate=None):
    """|e - th2| beyond which sign(L~ - R~) = sign(L - R); inf where D <= 0 or the gate is undecided, 0 where the gate
    rejects for certain.  The factor and the last term cover the fp64 evaluation of e, of this bound and of the exact
    values themselves (relative 2^-50 of the fp32 terms at most)."""
    with np.errstate(divide='ignore', invalid='ignore'):
        w = (L.e + R.e) / D
        w = w * (1.0 + 2.0 ** -20) + 16 * U64 * (np.abs(L.v) + np.abs(R.v)) / D
    w = np.where(D > 0, w, np.inf)
    if gate is not None:
        sure_out, unsure = gate
        w = np.where(sure_out, 0.0, np.where(unsure, np.inf, w))
    return np.where(np.isnan(w), np.inf, w)


def _two_view(kind, model, rows, th2):
    m = [_cast(v) for v in np.asarray(model, dtype=np.float64).reshape(9)]
    x1, y1, x2, y2 = (_cast(rows[:, i]) for i in range(4))
    t = _cast(th2)
    if kind in (0, 3):
        l2x = m[0] * x1 + m[1] * y1 + m[2]
        l2y = m[3] * x1 + m[4] * y1 + m[5]
        l2z = m[6] * x1 + m[7] * y1 + m[8]
        l1x = m[0] * x2 + m[3] * y2 + m[6]
        l1y = m[1] * x2 + m[4] * y2 + m[7]
        dd = x2 * l2x + y2 * l2y + l2z
        den = l1x * l1x + l1y * l1y + l2x * l2x + l2y * l2y
        return _width(dd * dd, t * den, den.v)
    w = m[6] * x1 + m[7] * y1 + m[8]
    u = m[0] * x1 + m[1] * y1 + m[2] - x2 * w
    v = m[3] * x1 + m[4] * y1 + m[5] - y2 * w
    gate_slack = w.e + abs(GATE_H - 1e-8) + 4 * U64 * 1e-8
    sure_out = w.v < 1e-8 - gate_slack
    unsure = np.abs(w.v - 1e-8) <= gate_slack
    return _width(u * u + v * v, t * w * w, w.v * w.v, (sure_out, unsure))


def _abs_pose(model, rows, th2, intr, mean, mean_err):
    """Kind 4 on rows (u, v, X, Y, Z) and a pose (R row-major, t) in the frame centred on `mean`."""
    fx, fy, cx, cy = (float(v) for v in intr)
    M = np.asarray(model, dtype=np.float64).reshape(12)
    mean = np.asarray(mean, dtype=np.float64)
    R = M[:9].reshape(3, 3)
    # the pose's t went through t - R mean and back: 4 roundings of fp64 on those magnitudes, plus R times the
    # difference of the device's and this mean
    t_err = 4 * U64 * (np.abs(R) @ np.abs(mean) + 2 * np.abs(M[9:])) + np.abs(R) @ mean_err
    scale = (fx, fy, 1.0)
    p = []
    for i in range(3):
        for k in range(4):
            v = scale[i] * (M[3 * i + k] if k < 3 else M[9 + i])
            e = U64 * abs(v) + (scale[i] * t_err[i] if k == 3 else 0.0)
            p.append(_cast(v, e))
    X = [_cast(rows[:, 2 + i] - mean[i], U64 * np.abs(rows[:, 2 + i]) + mean_err[i]) for i in range(3)]
    du = _cast(rows[:, 0] - cx, U64 * np.abs(rows[:, 0] - cx))
    dv = _cast(rows[:, 1] - cy, U64 * np.abs(rows[:, 1] - cy))
    a = p[0] * X[0] + p[1] * X[1] + p[2] * X[2] + p[3]
    b = p[4] * X[0] + p[5] * X[1] + p[6] * X[2] + p[7]
    z = p[8] * X[0] + p[9] * X[1] + p[10] * X[2] + p[11]
    eu = a - du * z
    ev = b - dv * z
    t = _cast(th2)
    sure_out = z.v < -z.e
    unsure = np.abs(z.v) <= z.e
    return _width(eu * eu + ev * ev, t * z * z, z.v * z.v, (sure_out, unsure))


def mean_error(rows):
    """Bound on |device centroid - numpy centroid| of the world points rows[:, 2:5]: both are sums of n terms in some
    order divided by n, each within n u64 sum |X| / n of the exact mean."""
    X = np.abs(np.asarray(rows, dtype=np.float64)[:, 2:5])
    n = max(X.shape[0], 1)
    return 2.0 * (n + 2) * U64 * X.sum(0) / n


def decision_bound(kind, model, rows, th2, intr=None, mean=None):
    """-> [n] float64 widths: wherever |e64 - th2| > width, the kernel's fp32 inlier decision on row i equals fp64's
    e64 < th2.  kind 0 (F, pixel rows), 1 (H, pixel rows), 3 (E, rows in camera coordinates (p - c) / f, th2 from
    pose_oracle.threshold) or 4 (absolute pose: rows (u, v, X, Y, Z), the pose in the frame centred on `mean` (the
    world points' centroid), intr = (fx, fy, cx, cy))."""
    rows = np.asarray(rows, dtype=np.float64)
    if kind == 4:
        return _abs_pose(model, rows, th2, intr, mean, mean_error(rows))
    return _two_view(kind, model, rows, th2)


# ---- numpy emulation of the kernels' fp32 arithmetic ------------------------------------------------------------------
def _f32(x):
    return np.asarray(x, dtype=np.float32)


def _muladd(a, b, c, fma):
    """a * b + c: two roundings, or one (fma) as float32(float64(a) float64(b) + float64(c))."""
    if fma:
        return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    return a * b + c


def _lin3(m0, m1, m2, x, y, fma):
    """m0 x + m1 y + m2 in source order; contracted: fma(m1, y, m0 x) + m2."""
    return _muladd(m1, y, m0 * x, fma) + m2


def fp32_decision(kind, model, rows, th2, fma=False, intr=None, mean=None):
    """The kernel's inlier test emulated in fp32, operation by operation (fma: with the products contracted into the
    sums that consume them) -> (decision [n] bool, err [n]): err is (L~ - R~) / D - (e - th2), the fp32 error of
    e - th2 against fp64, which decision_bound bounds."""
    rows = np.asarray(rows, dtype=np.float64)
    with np.errstate(all='ignore'):
        if kind == 4:
            fx, fy, cx, cy = (float(v) for v in intr)
            M = np.asarray(model, dtype=np.float64).reshape(12)
            mean = np.asarray(mean, dtype=np.float64)
            s = (fx, fy, 1.0)
            p = [_f32(s[i] * (M[3 * i + k] if k < 3 else M[9 + i])) for i in range(3) for k in range(4)]
            X = [_f32(rows[:, 2 + i] - mean[i]) for i in range(3)]
            du, dv = _f32(rows[:, 0] - cx), _f32(rows[:, 1] - cy)
            t = np.float32(th2)

            def lin4(q):
                return _muladd(q[2], X[2], _muladd(q[1], X[1], q[0] * X[0], fma), fma) + q[3]
            a, b, z = lin4(p[0:4]), lin4(p[4:8]), lin4(p[8:12])
            eu = _muladd(-du, z, a, fma)
            ev = _muladd(-dv, z, b, fma)
            L = _muladd(ev, ev, eu * eu, fma)
            Rr = t * z * z
            dec = (z > 0) & (L < Rr)
            # exact values
            P = rows[:, 2:5] - mean
            R9 = M[:9].reshape(3, 3)
            P = P @ R9.T + M[9:]
            ze = P[:, 2]
            eue = fx * P[:, 0] - (rows[:, 0] - cx) * ze
            eve = fy * P[:, 1] - (rows[:, 1] - cy) * ze
            Le, Re, D = eue * eue + eve * eve, th2 * ze * ze, ze * ze
        else:
            m = [_f32(v) for v in np.asarray(model, dtype=np.float64).reshape(9)]
            x1, y1, x2, y2 = (_f32(rows[:, i]) for i in range(4))
            t = np.float32(th2)
            M = np.asarray(model, dtype=np.float64).reshape(9)
            X1, Y1, X2, Y2 = (rows[:, i] for i in range(4))
            if kind in (0, 3):
                l2x, l2y, l2z = (_lin3(m[3 * i], m[3 * i + 1], m[3 * i + 2], x1, y1, fma) for i in range(3))
                l1x = _lin3(m[0], m[3], m[6], x2, y2, fma)
                l1y = _lin3(m[1], m[4], m[7], x2, y2, fma)
                dd = _muladd(y2, l2y, x2 * l2x, fma) + l2z
                den = _muladd(l2y, l2y, _muladd(l2x, l2x, _muladd(l1y, l1y, l1x * l1x, fma), fma), fma)
                L, Rr = dd * dd, t * den
                dec = L < Rr
                e2x, e2y, e2z = (M[3 * i] * X1 + M[3 * i + 1] * Y1 + M[3 * i + 2] for i in range(3))
                e1x, e1y = M[0] * X2 + M[3] * Y2 + M[6], M[1] * X2 + M[4] * Y2 + M[7]
                ddd = X2 * e2x + Y2 * e2y + e2z
                D = e1x * e1x + e1y * e1y + e2x * e2x + e2y * e2y
                Le, Re = ddd * ddd, th2 * D
            else:
                w = _lin3(m[6], m[7], m[8], x1, y1, fma)
                u = _muladd(-x2, w, _lin3(m[0], m[1], m[2], x1, y1, fma), fma)
                v = _muladd(-y2, w, _lin3(m[3], m[4], m[5], x1, y1, fma), fma)
                L = _muladd(v, v, u * u, fma)
                Rr = t * w * w
                dec = (w > np.float32(1e-8)) & (L < Rr)
                we = M[6] * X1 + M[7] * Y1 + M[8]
                ue = M[0] * X1 + M[1] * Y1 + M[2] - X2 * we
                ve = M[3] * X1 + M[4] * Y1 + M[5] - Y2 * we
                Le, Re, D = ue * ue + ve * ve, th2 * we * we, we * we
        err = ((L.astype(np.float64) - Le) - (Rr.astype(np.float64) - Re)) / D
    return dec, err


def exact_error(kind, model, rows, th2, intr=None, mean=None):
    """fp64 e of every row under one model (verify_oracle.errors / abspose_oracle.errors, E on camera rows)."""
    from . import abspose_oracle as A
    from . import verify_oracle as V
    if kind == 4:
        return A.errors(model, np.asarray(rows, dtype=np.float64), intr, mean)[0]
    return V.errors(1 if kind == 1 else 0, model, np.asarray(rows, dtype=np.float64))[0]
