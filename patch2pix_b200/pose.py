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


# ---- many pairs per call (p2p_find_essential_batch, p2p_recover_pose_batch) ------------------------------------------
def _intr_rows(K1_list, K2_list, K, reference=False):
    """Validated [K, 8] intrinsics (as intrinsics() / reference_intrinsics()) of K pairs, on the host."""
    from .verify import _as_list
    K1_list, K2_list = _as_list(K1_list, 'K1_list'), _as_list(K2_list, 'K2_list')
    if len(K1_list) != K or len(K2_list) != K:
        raise ValueError(f'K1_list and K2_list must have one matrix per pair ({K}), got {len(K1_list)} and '
                         f'{len(K2_list)}')
    out = np.empty((K, 8), dtype=np.float64)
    for k in range(K):
        try:
            out[k] = (reference_intrinsics if reference else intrinsics)(K1_list[k], K2_list[k])
        except ValueError as e:
            raise ValueError(f'pair {k}: intrinsics must be 3x3: {e}') from None
        if not (np.all(np.isfinite(out[k])) and out[k, [0, 1, 4, 5]].min() > 0):
            raise ValueError(f'pair {k}: intrinsics must be finite with positive focal lengths')
    return out


def batch_out_size(K, N):
    """float64 elements of a pose batch buffer: E [0:9K], R|t [9K:21K], int32 inlier and good counts [2K] from element
    21K, then the row-aligned E-RANSAC mask and the row-aligned pose mask."""
    return 22 * K + (2 * N + 7) // 8


def _batch_ptrs(out, K, N):
    base = out.data_ptr()
    return dict(E=base, Rt=base + 72 * K, cnt=base + 168 * K, good=base + 172 * K, emask=base + 176 * K,
                pmask=base + 176 * K + N)


def find_essential_batch_into(handle, rows, row_stride, offsets, offsets_host, n_dev, intr_ptr, px_th, conf, max_iters,
                              seed, E_ptr, mask_ptr, counts_ptr):
    """Enqueue p2p_find_essential_batch (device addresses as verify.find_model_batch_into; intr_ptr: [K][8] doubles)."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_find_essential_batch(
            handle.h, C.c_void_p(rows.data_ptr()), row_stride, C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, C.c_void_p(intr_ptr), float(px_th), float(conf),
            int(max_iters), int(seed) & (2 ** 64 - 1), C.c_void_p(E_ptr), C.c_void_p(mask_ptr), C.c_void_p(counts_ptr),
            handle.stream()))


def find_essential_batch_th_into(handle, rows, row_stride, offsets, offsets_host, n_dev, intr_ptr, px_th_ptr, conf,
                                 max_iters, seed, E_ptr, mask_ptr, counts_ptr):
    """Enqueue p2p_find_essential_batch_th (as pose.find_essential_batch_into, px_th_ptr: DEVICE double [K])."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_find_essential_batch_th(
            handle.h, C.c_void_p(rows.data_ptr()), row_stride, C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, C.c_void_p(intr_ptr), C.c_void_p(px_th_ptr),
            float(conf), int(max_iters), int(seed) & (2 ** 64 - 1), C.c_void_p(E_ptr), C.c_void_p(mask_ptr),
            C.c_void_p(counts_ptr), handle.stream()))


def recover_pose_batch_into(handle, rows, row_stride, offsets, offsets_host, n_dev, intr_ptr, E_ptr, mask_in_ptr, Rt_ptr,
                            mask_ptr, good_ptr, dist_th=DIST_TH):
    """Enqueue p2p_recover_pose_batch (device addresses; mask_in_ptr None: all rows)."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_recover_pose_batch(
            handle.h, C.c_void_p(rows.data_ptr()), row_stride, C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, C.c_void_p(intr_ptr), C.c_void_p(E_ptr),
            None if mask_in_ptr is None else C.c_void_p(mask_in_ptr), float(dist_th), C.c_void_p(Rt_ptr),
            C.c_void_p(mask_ptr), C.c_void_p(good_ptr), handle.stream()))


def _parse_batch(host, offsets, K, N):
    """Per pair (E or None, E mask, n_good, R, t, pose mask) of a host pose batch buffer; raises on non-finite input."""
    cnt = host[21 * K:22 * K].view(np.int32)
    b = host[22 * K:].view(np.uint8)
    out = []
    for k in range(K):
        if cnt[k] < 0:
            raise ValueError(f'find_essential: a point coordinate is not finite (pair {k})')
        o0, o1 = offsets[k], offsets[k + 1]
        Rt = host[9 * K + 12 * k:9 * K + 12 * k + 12]
        out.append((host[9 * k:9 * k + 9].reshape(3, 3).copy() if cnt[k] > 0 else None, b[o0:o1].astype(bool),
                    int(cnt[K + k]), Rt[:9].reshape(3, 3).copy(), Rt[9:].reshape(3, 1).copy(),
                    b[N + o0:N + o1].astype(bool)))
    return out


def find_essential_matrices(pts1_list, pts2_list, K1_list, K2_list, px_th, conf=0.999, max_iters=1000, seed=0):
    """find_essential_matrix over a list of pairs in one batched call -> [(E, inlier mask)], element k equal to
    find_essential_matrix(pts1_list[k], pts2_list[k], K1_list[k], K2_list[k], px_th_k, ...), px_th_k = px_th, or
    px_th[k] when px_th is a sequence of one threshold per pair (p2p_find_essential_batch_th).  Numpy input crosses
    PCIe once each way and raises ValueError when a pair has a non-finite coordinate; CUDA tensor input gives CUDA
    tensor views without a sync."""
    from .verify import pair_lists, upload
    rows, offsets, is_np = pair_lists(pts1_list, pts2_list)
    K, N = offsets.size - 1, int(offsets[-1])
    intr = _intr_rows(K1_list, K2_list, K)
    per_pair = np.ndim(px_th) > 0
    if per_pair:
        px = np.asarray(px_th, dtype=np.float64).reshape(-1)
        if px.size != K or not (np.all(np.isfinite(px)) and np.all(px > 0)):
            raise ValueError(f'px_th must be one positive threshold, or {K} (one per pair), got {px.size} values')
    if K == 0:
        return []
    rows, offs, ex = upload(rows, offsets, is_np, np.concatenate((intr.reshape(-1), px)) if per_pair else intr)
    out = torch.zeros(batch_out_size(K, N), dtype=torch.float64, device=rows.device)
    p = _batch_ptrs(out, K, N)
    h = _lib.default_handle(rows.device)
    if per_pair:
        find_essential_batch_th_into(h, rows, 4, offs, offsets, None, ex.data_ptr(), ex.data_ptr() + 64 * K, conf,
                                     max_iters, seed, p['E'], p['emask'], p['cnt'])
    else:
        find_essential_batch_into(h, rows, 4, offs, offsets, None, ex.data_ptr(), px_th, conf, max_iters, seed, p['E'],
                                  p['emask'], p['cnt'])
    if is_np:
        return [r[:2] for r in _parse_batch(out.cpu().numpy(), offsets, K, N)]
    m = out[22 * K:].view(torch.uint8)
    return [(out[9 * k:9 * k + 9].view(3, 3), m[offsets[k]:offsets[k + 1]].bool()) for k in range(K)]


def recover_poses(E_list, pts1_list, pts2_list, K1_list, K2_list, mask_list=None, dist_th=DIST_TH):
    """recover_pose over a list of pairs in one batched call -> [(n_good, R, t [3, 1], good mask)], element k equal to
    recover_pose(E_list[k], pts1_list[k], pts2_list[k], K1_list[k], K2_list[k], mask_list[k], dist_th).  mask_list:
    None, or one mask (or None) per pair."""
    from .verify import _as_list, pair_lists, upload
    rows, offsets, is_np = pair_lists(pts1_list, pts2_list)
    K, N = offsets.size - 1, int(offsets[-1])
    E_list = _as_list(E_list, 'E_list')
    if len(E_list) != K:
        raise ValueError(f'E_list must have one matrix per pair ({K}), got {len(E_list)}')
    intr = _intr_rows(K1_list, K2_list, K)
    for k, E in enumerate(E_list):
        if (E.numel() if isinstance(E, torch.Tensor) else np.size(E)) != 9:
            raise ValueError(f'pair {k}: E must be 3x3')
    if mask_list is not None:
        mask_list = _as_list(mask_list, 'mask_list')
        if len(mask_list) != K:
            raise ValueError(f'mask_list must have one mask (or None) per pair ({K}), got {len(mask_list)}')
        for k, m in enumerate(mask_list):
            if m is not None and (m.numel() if isinstance(m, torch.Tensor) else np.size(m)) != offsets[k + 1] - offsets[k]:
                raise ValueError(f'pair {k}: mask has {np.size(m) if not isinstance(m, torch.Tensor) else m.numel()} '
                                 f'entries for {offsets[k + 1] - offsets[k]} points')
    if K == 0:
        return []
    if is_np:          # E and masks travel with the rows
        Es = np.stack([np.asarray(E, dtype=np.float64).reshape(9) for E in E_list])
        masks = None if mask_list is None else np.concatenate(
            [np.ones(offsets[k + 1] - offsets[k]) if m is None else (np.asarray(m).reshape(-1) != 0)
             for k, m in enumerate(mask_list)]).astype(np.float64)
        extra = np.concatenate((intr.reshape(-1), Es.reshape(-1)) + (() if masks is None else (masks,)))
        rows, offs, ex = upload(rows, offsets, is_np, extra)
        Ed = ex[8 * K:17 * K]
        md = None if masks is None else ex[17 * K:].to(torch.uint8)
    else:
        rows, offs, ex = upload(rows, offsets, is_np, intr)
        Ed = torch.stack([torch.as_tensor(E, dtype=torch.float64).reshape(9).to(rows.device) for E in E_list])
        md = None if mask_list is None else torch.cat(
            [torch.ones(int(offsets[k + 1] - offsets[k]), dtype=torch.uint8, device=rows.device) if m is None else
             (torch.as_tensor(m).reshape(-1) != 0).to(torch.uint8).to(rows.device) for k, m in enumerate(mask_list)])
    dev = rows.device
    out = torch.zeros(batch_out_size(K, N), dtype=torch.float64, device=dev)
    p = _batch_ptrs(out, K, N)
    recover_pose_batch_into(_lib.default_handle(dev), rows, 4, offs, offsets, None, ex.data_ptr(), Ed.data_ptr(),
                            None if md is None else md.data_ptr(), p['Rt'], p['pmask'], p['good'], dist_th)
    if is_np:
        return [r[2:] for r in _parse_batch(out.cpu().numpy(), offsets, K, N)]
    cnt = out[21 * K:22 * K].view(torch.int32)
    m = out[22 * K:].view(torch.uint8)
    return [(cnt[K + k], out[9 * K + 12 * k:9 * K + 12 * k + 9].view(3, 3),
             out[9 * K + 12 * k + 9:9 * K + 12 * k + 12].view(3, 1), m[N + offsets[k]:N + offsets[k + 1]].bool())
            for k in range(K)]


def _match_lists(matches_list):
    from .verify import _as_list
    ms = [np.asarray(m, dtype=np.float64) for m in _as_list(matches_list, 'matches_list')]
    for k, m in enumerate(ms):
        if m.ndim != 2 or m.shape[1] < 4:
            raise ValueError(f'pair {k}: matches must be [n, 4] (x1, y1, x2, y2), got {m.shape}')
    return [m[:, :2] for m in ms], [m[:, 2:4] for m in ms]


def matches2relapose_batch(matches_list, K1_list, K2_list, rthres=1):
    """matches2relapose over a list of pairs: one E-RANSAC launch chain and one pose-recovery chain for every pair ->
    [(E, inls, R, t)], element k equal to matches2relapose(m[:, :2], m[:, 2:4], K1_list[k], K2_list[k], rthres) for
    m = matches_list[k].  One host->device and one device->host copy."""
    from .verify import pair_lists, upload
    p1, p2 = _match_lists(matches_list)
    rows, offsets, _ = pair_lists(p1, p2)
    K, N = offsets.size - 1, int(offsets[-1])
    intr = _intr_rows(K1_list, K2_list, K, reference=True)
    if K == 0:
        return []
    rows, offs, intr_d = upload(rows, offsets, True, intr)
    h = _lib.default_handle(rows.device)
    out = torch.zeros(batch_out_size(K, N), dtype=torch.float64, device=rows.device)
    p = _batch_ptrs(out, K, N)
    find_essential_batch_into(h, rows, 4, offs, offsets, None, intr_d.data_ptr(), rthres, 0.999, 1000, 0, p['E'],
                              p['emask'], p['cnt'])
    recover_pose_batch_into(h, rows, 4, offs, offsets, None, intr_d.data_ptr(), p['E'], p['emask'], p['Rt'], p['pmask'],
                            p['good'])
    return [(E, np.where(em)[0], R, t) for E, em, _, R, t, _ in _parse_batch(out.cpu().numpy(), offsets, K, N)]


def matches2relapose_degensac_batch(matches_list, K1_list, K2_list, rthres=1):
    """matches2relapose_degensac over a list of pairs -> [(E, inls, R, t)], element k equal to
    matches2relapose_degensac(m[:, :2], m[:, 2:4], K1_list[k], K2_list[k], rthres) for m = matches_list[k]: the rows
    rescaled per pair as the reference does, one DEGENSAC launch chain and one pose-recovery chain for every pair.  One
    host->device and one device->host copy."""
    from . import verify as V
    p1, p2 = _match_lists(matches_list)
    rows, offsets, _ = V.pair_lists(p1, p2)
    K, N = offsets.size - 1, int(offsets[-1])
    ref = _intr_rows(K1_list, K2_list, K, reference=True)          # f1, f1, cx1, cy1, f2, f2, cx2, cy2
    if K == 0:
        return []
    f1, f2 = ref[:, 0], ref[:, 4]
    # per pair: rescale (pc1 x2, f2, 1 / f1, pc2 x2), intr (f2, f2, 0, 0) x2, k = (f2, f2, 1)
    z = np.zeros(K)
    per_pair = np.stack((ref[:, 2], ref[:, 3], f2, 1.0 / f1, ref[:, 6], ref[:, 7]), 1)
    intr = np.stack((f2, f2, z, z, f2, f2, z, z), 1)
    kk = np.stack((f2, f2, np.ones(K)), 1)
    rows, offs, ex = V.upload(rows, offsets, True, np.concatenate((per_pair.ravel(), intr.ravel(), kk.ravel())))
    dev = rows.device
    pp = ex[:6 * K].view(K, 6).repeat_interleave(torch.from_numpy(np.diff(offsets)).to(dev), dim=0)
    # as matches2relapose_degensac: ((p1 - pc1) * f2) / f1 (a division by a host scalar runs as a multiplication by
    # its reciprocal on the device), p2 - pc2
    rows = torch.cat((((rows[:, 0:2] - pp[:, 0:2]) * pp[:, 2:3]) * pp[:, 3:4], rows[:, 2:4] - pp[:, 4:6]), 1).contiguous()
    intr_d, k = ex[6 * K:14 * K], ex[14 * K:].view(K, 3)
    h = _lib.default_handle(dev)
    out = torch.zeros(batch_out_size(K, N) + V.batch_out_size(K, N), dtype=torch.float64, device=dev)
    fout = out[batch_out_size(K, N):]
    p, fb = _batch_ptrs(out, K, N), fout.data_ptr()
    V.find_model_batch_into(h, V.MODEL_F_DEGENSAC, rows, 4, offs, offsets, None, rthres, 0.999, 10000, 0, fb,
                            fb + 8 * (9 * K + (K + 1) // 2), fb + 72 * K)
    out[:9 * K] = ((fout[:9 * K].view(K, 3, 3) * k[:, :, None]) * k[:, None, :]).reshape(-1)      # K^T F K per pair
    recover_pose_batch_into(h, rows, 4, offs, offsets, None, intr_d.data_ptr(), p['E'],
                            fb + 8 * (9 * K + (K + 1) // 2), p['Rt'], p['pmask'], p['good'])
    host = out.cpu().numpy()
    fres = V.parse_batch_host(host[batch_out_size(K, N):], offsets)
    res = []
    for k, (F, fmask) in enumerate(fres):
        Rt = host[9 * K + 12 * k:9 * K + 12 * k + 12]
        res.append((host[9 * k:9 * k + 9].reshape(3, 3).copy() if F is not None else None, np.where(fmask)[0],
                    Rt[:9].reshape(3, 3).copy(), Rt[9:].reshape(3, 1).copy()))
    return res
