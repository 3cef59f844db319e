"""Relative pose on the GPU: essential-matrix RANSAC and pose recovery, plus the host helpers of the reference's pose
evaluation.

Drop-in for the reference's ``matches2relapose_cv`` (utils/eval/geometry.py:32-48: cv2.findEssentialMat + cv2.recoverPose)
and ``eval_matches_relapose`` (utils/eval/measure.py:102-113) on top of ``p2p_find_essential`` / ``p2p_recover_pose``
(include/p2p_b200.h).  The quaternion and pose helpers restate what the reference imports from transforms3d and
utils/eval/geometry.py, in numpy.

Conventions as patch2pix_b200.verify: numpy input gives numpy output through one device->host copy (E None when no
model was found); CUDA tensor input gives CUDA tensor output without a sync (E all zeros when no model was found, NaN
when a coordinate was not finite).  K1, K2 are 3x3 intrinsics in pixels (host arrays).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .verify import _rows

DIST_TH = 50.0            # cv2.recoverPose's default distanceThresh


def intrinsics(K1, K2):
    """(fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2) as a host double[8]."""
    K1 = np.asarray(K1, dtype=np.float64).reshape(3, 3)
    K2 = np.asarray(K2, dtype=np.float64).reshape(3, 3)
    return (C.c_double * 8)(K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2], K2[0, 0], K2[1, 1], K2[0, 2], K2[1, 2])


def out_size(n):
    """float64 elements of a pose buffer: E [0:9], int32 inlier count in 9, R|t [10:22], int32 good count in 22, the
    E-RANSAC mask from byte 184 and the pose mask after it."""
    return 23 + (2 * n + 7) // 8


def find_essential_into(handle, rows, row_stride, n, n_dev, intr, px_th, conf, max_iters, seed, out):
    """Enqueue p2p_find_essential on `rows` (a float64 device tensor, row r at offset r * row_stride) into a pose
    buffer `out` (see out_size).  `n_dev` is an optional pointer (ctypes) to a device double row count."""
    base = out.data_ptr()
    with torch.cuda.device(out.device):
        _lib.check(handle.lib.p2p_find_essential(handle.h, C.c_void_p(rows.data_ptr()), row_stride, n, n_dev, intr,
                                                 float(px_th), float(conf), int(max_iters), int(seed) & (2 ** 64 - 1),
                                                 C.c_void_p(base), C.c_void_p(base + 184), C.c_void_p(base + 72),
                                                 handle.stream()))


def recover_pose_into(handle, rows, row_stride, n, n_dev, intr, E_ptr, mask_ptr, out, dist_th=DIST_TH):
    """Enqueue p2p_recover_pose of the E at device address `E_ptr` on the rows under the device mask at `mask_ptr`
    (None: all rows) into the pose buffer `out`."""
    base = out.data_ptr()
    with torch.cuda.device(out.device):
        _lib.check(handle.lib.p2p_recover_pose(handle.h, C.c_void_p(rows.data_ptr()), row_stride, n, n_dev, intr,
                                               C.c_void_p(E_ptr), None if mask_ptr is None else C.c_void_p(mask_ptr),
                                               float(dist_th), C.c_void_p(base + 80), C.c_void_p(base + 184 + n),
                                               C.c_void_p(base + 176), handle.stream()))


def parse_host(host, n):
    """(E or None, E mask, n_good, R, t, pose mask) from the host copy of a pose buffer; raises on non-finite input."""
    count = int(host[9:10].view(np.int32)[0])
    if count < 0:
        raise ValueError('find_essential: a point coordinate is not finite')
    b = host.view(np.uint8)
    E = host[:9].reshape(3, 3).copy() if count > 0 else None
    n_good = int(host[22:23].view(np.int32)[0])
    return (E, b[184:184 + n].astype(bool), n_good, host[10:19].reshape(3, 3).copy(), host[19:22].reshape(3, 1).copy(),
            b[184 + n:184 + 2 * n].astype(bool))


def find_essential_matrix(pts1, pts2, K1, K2, px_th, conf=0.999, max_iters=1000, seed=0):
    """cv2.findEssentialMat(pts1, pts2, method=RANSAC) with two cameras -> (E, inlier mask).  E relates camera
    coordinates (x2^T E x1 = 0, unit Frobenius norm); a row is an inlier iff its Sampson error in camera coordinates
    is below (px_th / ((fx2 + fy2) / 2))^2."""
    rows, is_np = _rows(pts1, pts2)
    n = int(rows.shape[0])
    h = _lib.default_handle(rows.device)
    out = torch.empty(out_size(n), dtype=torch.float64, device=rows.device)
    find_essential_into(h, rows, 4, n, None, intrinsics(K1, K2), px_th, conf, max_iters, seed, out)
    if is_np:
        return parse_host(out.cpu().numpy(), n)[:2]
    return out[:9].view(3, 3), out.view(torch.uint8)[184:184 + n].bool()


def recover_pose(E, pts1, pts2, K1, K2, mask=None, dist_th=DIST_TH):
    """cv2.recoverPose(E, pts1, pts2, K, mask=mask) with two cameras -> (n_good, R, t [3, 1], good mask): the
    decomposition of E whose triangulated points lie in front of both cameras (x2 = R x1 + t, |t| = 1), and those
    points, a subset of `mask`.  A zero E gives zeros and an empty mask."""
    rows, is_np = _rows(pts1, pts2)
    n = int(rows.shape[0])
    dev = rows.device
    Ed = torch.as_tensor(np.asarray(E, dtype=np.float64) if not isinstance(E, torch.Tensor) else E,
                         dtype=torch.float64).reshape(9).to(dev).contiguous()
    md = None
    if mask is not None:
        md = torch.as_tensor(np.asarray(mask) if not isinstance(mask, torch.Tensor) else mask).reshape(-1)
        if md.shape[0] != n:
            raise ValueError(f'mask has {md.shape[0]} entries for {n} points')
        md = (md != 0).to(torch.uint8).to(dev).contiguous()
    out = torch.zeros(out_size(n), dtype=torch.float64, device=dev)
    h = _lib.default_handle(dev)
    recover_pose_into(h, rows, 4, n, None, intrinsics(K1, K2), Ed.data_ptr(), None if md is None else md.data_ptr(), out,
                      dist_th)
    if is_np:
        host = out.cpu().numpy()
        b = host.view(np.uint8)
        return (int(host[22:23].view(np.int32)[0]), host[10:19].reshape(3, 3).copy(), host[19:22].reshape(3, 1).copy(),
                b[184 + n:184 + 2 * n].astype(bool))
    return out[22:23].view(torch.int32)[0], out[10:19].view(3, 3), out[19:22].view(3, 1), \
        out.view(torch.uint8)[184 + n:184 + 2 * n].bool()


def reference_intrinsics(K1, K2):
    """The cameras of geometry.py:35-45 as a host double[8]: principal points K[:2, 2] and focal length K[0, 0] on both
    axes of each view.  The reference moves the principal points to the origin, rescales view 1 to view 2's focal
    length and passes K = diag(f2, f2, 1); in camera coordinates that is ((x - cx1) / f1, (y - cy1) / f1) and
    ((x - cx2) / f2, (y - cy2) / f2), with the threshold in view-2 pixels."""
    K1 = np.asarray(K1, dtype=np.float64).reshape(3, 3)
    K2 = np.asarray(K2, dtype=np.float64).reshape(3, 3)
    f1, f2 = K1[0, 0], K2[0, 0]
    return (C.c_double * 8)(f1, f1, K1[0, 2], K1[1, 2], f2, f2, K2[0, 2], K2[1, 2])


def matches2relapose_degensac(p1, p2, K1, K2, rthres=1):
    """utils/eval/geometry.py:50-71 on the GPU -> (E, inls, R, t): the rows rescaled as the reference does (p1 ->
    (p1 - pc1) * f2 / f1, p2 -> p2 - pc2, f = K[0, 0]), F RANSAC with the DEGENSAC check (model 2) at `rthres` px,
    E = K^T F K with K = diag(f2, f2, 1), the indices of F's inliers and the pose recovered from those rows (t [3, 1]).
    One device->host copy.  conf 0.999 and 10000 iterations are this project's F defaults; pydegensac's own defaults
    were not checked.  E is None and R, t are zero when no model was found."""
    from . import verify as V
    rows, _ = _rows(p1, p2)
    n = int(rows.shape[0])
    K1 = np.asarray(K1, dtype=np.float64).reshape(3, 3)
    K2 = np.asarray(K2, dtype=np.float64).reshape(3, 3)
    f1, f2 = float(K1[0, 0]), float(K2[0, 0])
    rows = torch.cat((((rows[:, 0:2] - torch.tensor(K1[:2, 2], device=rows.device)) * f2) / f1,
                      rows[:, 2:4] - torch.tensor(K2[:2, 2], device=rows.device)), 1).contiguous()
    h = _lib.default_handle(rows.device)
    intr = (C.c_double * 8)(f2, f2, 0.0, 0.0, f2, f2, 0.0, 0.0)
    buf = torch.zeros(out_size(n) + V.out_size(n), dtype=torch.float64, device=rows.device)
    out, fbuf = buf[:out_size(n)], buf[out_size(n):]        # pose buffer with E in [0:9], then the F-RANSAC buffer
    V.find_model_into(h, V.MODEL_F_DEGENSAC, rows, 4, n, None, rthres, 0.999, 10000, 0, fbuf)
    k = torch.tensor([f2, f2, 1.0], dtype=torch.float64, device=rows.device)
    out[:9] = ((fbuf[:9].view(3, 3) * k[:, None]) * k[None, :]).reshape(9)      # K^T F K, as fund2ess
    recover_pose_into(h, rows, 4, n, None, intr, out.data_ptr(), fbuf.data_ptr() + 80, out)
    host = buf.cpu().numpy()
    F, fmask = V.parse_host(host[out_size(n):], n)
    _, _, _, R, t, _ = parse_host(host[:out_size(n)], n)
    return (host[:9].reshape(3, 3).copy() if F is not None else None), np.where(fmask)[0], R, t


def matches2relapose(p1, p2, K1, K2, rthres=1):
    """utils/eval/geometry.py:32-48 on the GPU -> (E, inls, R, t): E-RANSAC (conf 0.999, 1000 iterations, as
    cv2.findEssentialMat's defaults) at `rthres` px, the indices of its inliers, and the pose recovered from those rows
    (t [3, 1]).  One device->host copy.  E is None and R, t are zero when no model was found."""
    rows, _ = _rows(p1, p2)
    n = int(rows.shape[0])
    h = _lib.default_handle(rows.device)
    intr = reference_intrinsics(K1, K2)
    out = torch.zeros(out_size(n), dtype=torch.float64, device=rows.device)
    find_essential_into(h, rows, 4, n, None, intr, rthres, 0.999, 1000, 0, out)
    recover_pose_into(h, rows, 4, n, None, intr, out.data_ptr(), out.data_ptr() + 184, out)
    E, emask, _, R, t, _ = parse_host(out.cpu().numpy(), n)
    return E, np.where(emask)[0], R, t


# ---- host helpers of the reference's pose evaluation (transforms3d conventions: quaternions w, x, y, z) -------------
def quat2mat(q):
    """Unit-normalised quaternion (w, x, y, z) -> 3x3 rotation (transforms3d.quaternions.quat2mat)."""
    w, x, y, z = (float(v) for v in q)
    nq = w * w + x * x + y * y + z * z
    if nq < np.finfo(np.float64).eps:
        return np.eye(3)
    s = 2.0 / nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def mat2quat(M):
    """3x3 rotation -> quaternion (w, x, y, z) with w >= 0 (transforms3d.quaternions.mat2quat: the eigenvector of the
    largest eigenvalue of Bar-Itzhack's symmetric 4x4 matrix)."""
    (Qxx, Qyx, Qzx), (Qxy, Qyy, Qzy), (Qxz, Qyz, Qzz) = np.asarray(M, dtype=np.float64).reshape(3, 3)
    Kq = np.array([[Qxx - Qyy - Qzz, 0, 0, 0],
                   [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0],
                   [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                   [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(Kq)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    return -q if q[0] < 0 else q


def skew(v):
    v = np.asarray(v, dtype=np.float64).reshape(3)
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def abs2relapose(c1, c2, q1, q2):
    """utils/eval/geometry.py:73-89: absolute camera positions c and orientations q (w, x, y, z) -> (t12, q12), the
    transformation from camera 1 to camera 2 coordinates."""
    r1, r2 = quat2mat(q1), quat2mat(q2)
    r12 = r2 @ r1.T
    return r2 @ (np.asarray(c1, dtype=np.float64) - np.asarray(c2, dtype=np.float64)), mat2quat(r12)


def pose2fund(K1, K2, R, t):
    """utils/eval/geometry.py:15: F of the relative pose (R, t) between cameras K1 and K2 (x2^T F x1 = 0)."""
    K1 = np.asarray(K1, dtype=np.float64)
    K2 = np.asarray(K2, dtype=np.float64)
    R = np.asarray(R, dtype=np.float64)
    return np.linalg.inv(K2).T @ R @ K1.T @ skew((K1 @ R.T).dot(np.asarray(t, dtype=np.float64).reshape(3)))


def cal_vec_angle_error(label, pred, eps=1e-14):
    """utils/eval/measure.py:73-84: angle in degrees between vectors (rows)."""
    label = np.atleast_2d(np.asarray(label, dtype=np.float64))
    pred = np.atleast_2d(np.asarray(pred, dtype=np.float64))
    v1 = pred / (np.linalg.norm(pred, axis=1, keepdims=True) + eps)
    v2 = label / (np.linalg.norm(label, axis=1, keepdims=True) + eps)
    d = np.clip(np.sum(v1 * v2, axis=1, keepdims=True), -1, 1)
    return np.degrees(np.arccos(d)).squeeze()


def cal_quat_angle_error(label, pred, eps=1e-14):
    """utils/eval/measure.py:86-96: rotation angle in degrees between quaternions (rows)."""
    label = np.atleast_2d(np.asarray(label, dtype=np.float64))
    pred = np.atleast_2d(np.asarray(pred, dtype=np.float64))
    q1 = pred / (np.linalg.norm(pred, axis=1, keepdims=True) + eps)
    q2 = label / (np.linalg.norm(label, axis=1, keepdims=True) + eps)
    d = np.clip(np.abs(np.sum(q1 * q2, axis=1, keepdims=True)), -1, 1)
    return (2 * np.degrees(np.arccos(d))).squeeze()


def eval_matches_relapose(matches, K1, K2, q_, t_, cv_thres=1.0):
    """utils/eval/measure.py:102-113 on the GPU: matches [n, 4] (x1, y1, x2, y2) -> (terr, qerr, inls), the angular
    errors in degrees of the recovered t and R against the ground truth t_ and q_ (w, x, y, z)."""
    matches = np.asarray(matches, dtype=np.float64)
    E, inls, R, t = matches2relapose(matches[:, :2], matches[:, 2:4], K1, K2, rthres=cv_thres)
    return cal_vec_angle_error(t.squeeze(), t_), cal_quat_angle_error(mat2quat(R), q_), inls


def first_essential_hypotheses(pts1, pts2, K1, K2, px_th, count, seed=0):
    """Test hook: the first `count` hypotheses of find_essential_matrix without selection -> (models [count*10, 9]
    float64 in camera coordinates, counts [count*10] int32, -1 where a slot holds no model)."""
    rows, _ = _rows(pts1, pts2)
    models = torch.empty(count * 10, 9, dtype=torch.float64, device=rows.device)
    counts = torch.empty(count * 10, dtype=torch.int32, device=rows.device)
    h = _lib.default_handle(rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_test_essential_hypotheses(h.h, _lib.ptr(rows), 4, int(rows.shape[0]), intrinsics(K1, K2),
                                                       float(px_th), int(seed) & (2 ** 64 - 1), count, _lib.ptr(models),
                                                       _lib.ptr(counts), h.stream()))
    return models.cpu().numpy(), counts.cpu().numpy()
