"""Visual localization on the GPU: absolute camera pose from 2D-3D matches (batched P3P RANSAC), and the InLoc
protocol of hloc's localize_inloc, with the matching, the lift of the matches to 3D and the RANSAC of many queries
on the device.

    python -m patch2pix_b200.localize --ckpt PATH --data_root DIR --pairs FILE --results OUT [--method patch2pix|nc]

find_absolute_pose / find_absolute_poses run p2p_find_absolute_pose_batch (include/p2p_b200.h): rows (u, v, X, Y, Z),
a pinhole camera per query, a pixel threshold; a row is an inlier iff its depth is positive and its reprojection error
is below the threshold.  The pose maps world to camera: x_cam = R X + t.

The InLoc protocol (hloc's pose_from_cluster, the localization of Patch2Pix's paper):

* The retrieval list has one 'query db' pair per line (paths relative to data_root), grouped by query in file order.
* Each query is matched against each of its retrieved database cutouts.  The matches' cutout pixels are lifted to 3D
  through the cutout's scan, data_root/<db>.mat (`XYZcut`, [H, W, 3], NaN holes): bilinear interpolation as
  grid_sample(align_corners=True), the nearest pixel where that is NaN, dropped where that is NaN too or outside the
  cutout (p2p_lift_scan).  The points are moved to world coordinates by the scan's alignment, the 4x4 P_after_GICP on
  lines 7-10 (counted from 0) of data_root/database/alignments/<floor>/transformations/<building>_trans_<scan>.txt, for
  a cutout database/cutouts/<floor>/<scan>/<image>; <building> is the first three characters of the image name.
* The 2D-3D matches of all of a query's cutouts are pooled, in retrieval order, and one pose is estimated at
  ransac_thres pixels (48 by default) with a SIMPLE_PINHOLE camera of focal length 4032 * 28 / 36 and the principal
  point at the image centre (hloc's model of InLoc's iPhone 7 queries).  Distortion and EXIF rotation are not handled.
* The results file has one line per query, 'name qw qx qy qz tx ty tz' (the query's file name, world -> camera,
  COLMAP's convention), the file InLoc's online benchmark takes.  A query whose matcher raised, or that got no model, is
  written with the identity pose so that every query is listed, and is returned in `failed` (this project's rule).

Reproducibility: matching, lifting and RANSAC of a chunk of queries run on one stream without a host sync; the poses
come back in one copy at the end.  The result does not depend on chunk_queries.
"""
import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib

INLOC_FOCAL = 4032.0 * 28.0 / 36.0
ENTRY_ABSPOSE = 3                  # p2p_batch_chunk_pairs entry of p2p_find_absolute_pose_batch


# ---- absolute pose ---------------------------------------------------------------------------------------------------
def _camera(K):
    """(fx, fy, cx, cy) of a 3x3 pinhole matrix or a 4-vector."""
    K = np.asarray(K, dtype=np.float64)
    if K.shape == (3, 3):
        if K[0, 1] != 0 or np.any(K[2] != (0, 0, 1)):
            raise ValueError('K must be a pinhole matrix [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]')
        v = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    elif K.shape == (4,):
        v = K.copy()
    else:
        raise ValueError(f'K must be 3x3 or (fx, fy, cx, cy), got shape {K.shape}')
    if not (np.all(np.isfinite(v)) and v[0] > 0 and v[1] > 0):
        raise ValueError('K must be finite with positive focal lengths')
    return v


def _query_rows(pts2d_list, pts3d_list):
    """Validated per-query rows [n, 5] (numpy float64, or CUDA tensors), host offsets [K+1], whether numpy."""
    for x, nm in ((pts2d_list, 'pts2d_list'), (pts3d_list, 'pts3d_list')):
        if isinstance(x, (np.ndarray, torch.Tensor)) or not hasattr(x, '__len__'):
            raise TypeError(f'{nm} must be a list of per-query arrays')
    if len(pts2d_list) != len(pts3d_list):
        raise ValueError(f'pts2d_list and pts3d_list must have the same length, got {len(pts2d_list)} and '
                         f'{len(pts3d_list)}')
    kinds = {isinstance(p, torch.Tensor) for p in list(pts2d_list) + list(pts3d_list)}
    if len(kinds) > 1:
        raise TypeError('the point lists must all be numpy arrays or all be tensors')
    is_np = not kinds or kinds == {False}
    rows = []
    for k, (a, b) in enumerate(zip(pts2d_list, pts3d_list)):
        if is_np:
            a = np.asarray(a, dtype=np.float64).reshape(-1, 2)
            b = np.asarray(b, dtype=np.float64).reshape(-1, 3)
            if a.shape[0] != b.shape[0]:
                raise ValueError(f'query {k}: {a.shape[0]} 2D points and {b.shape[0]} 3D points')
            rows.append(np.concatenate((a, b), 1))
        else:
            if a.device.type != 'cuda' or b.device != a.device or a.device != pts2d_list[0].device:
                raise ValueError('tensor input must be on one CUDA device')
            if a.dim() != 2 or a.shape[1] != 2 or b.dim() != 2 or b.shape[1] != 3 or a.shape[0] != b.shape[0]:
                raise ValueError(f'query {k}: pts2d must be [n, 2] and pts3d [n, 3], got {tuple(a.shape)} and '
                                 f'{tuple(b.shape)}')
            rows.append(torch.cat((a, b), 1).to(torch.float64))
    offsets = np.zeros(len(rows) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([int(r.shape[0]) for r in rows])
    if np.any(np.diff(offsets) > 1 << 26) or offsets[-1] >= 1 << 31:
        raise ValueError('a query has more than 2^26 rows or the batch has 2^31 rows or more')
    return rows, offsets, is_np


def find_absolute_pose_batch_into(handle, rows, row_stride, offsets, offsets_host, n_dev, intr_ptr, px_th, px_th_ptr,
                                  conf, max_iters, seed, Rt_ptr, mask_ptr, counts_ptr):
    """Enqueue p2p_find_absolute_pose_batch: `rows` a float64 device tensor, `offsets` an int64 device tensor [K+1]
    and `offsets_host` the same values in numpy; n_dev a ctypes device address or None; the other pointers are device
    addresses (intr [K][4], px_th_ptr [K] or None for the scalar px_th, Rt [K][12], row-aligned uint8 mask, int32
    counts [K])."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_find_absolute_pose_batch(
            handle.h, C.c_void_p(rows.data_ptr()), int(row_stride), C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, C.c_void_p(intr_ptr), float(px_th),
            None if px_th_ptr is None else C.c_void_p(px_th_ptr), float(conf), int(max_iters),
            int(seed) & (2 ** 64 - 1), C.c_void_p(Rt_ptr), C.c_void_p(mask_ptr), C.c_void_p(counts_ptr),
            handle.stream()))


def find_absolute_poses(pts2d_list, pts3d_list, K, px_th, conf=0.99999, max_iters=10000, seed=0):
    """Absolute pose of K queries in one batched call -> [(R, t, mask)], element k bit for bit the result of
    find_absolute_pose on query k.  K: one camera for every query or a list of one per query (3x3 pinhole matrices or
    (fx, fy, cx, cy)); px_th: one pixel threshold or one per query.

    Numpy input gives numpy output through one copy each way: R [3, 3] and t [3] float64 (None when there is no model:
    fewer than 4 rows or no pose found), a bool mask; a query with a non-finite value raises ValueError.  CUDA tensor
    input gives CUDA tensors without a sync: R and t are NaN without a model, the mask is all False."""
    rows, offsets, is_np = _query_rows(pts2d_list, pts3d_list)
    nq, N = offsets.size - 1, int(offsets[-1])
    if nq == 0:
        return []
    Ks = [K] * nq if np.shape(K) in ((3, 3), (4,)) else list(K)
    if len(Ks) != nq:
        raise ValueError(f'{len(Ks)} cameras for {nq} queries')
    intr = np.stack([_camera(k) for k in Ks])
    per_query = np.ndim(px_th) > 0
    th = np.asarray(px_th, dtype=np.float64).reshape(-1)
    if per_query and th.size != nq:
        raise ValueError(f'{th.size} thresholds for {nq} queries')
    if not (np.all(np.isfinite(th)) and np.all(th > 0)):
        raise ValueError('px_th must be positive and finite')
    dev = rows[0].device if not is_np else torch.device('cuda', torch.cuda.current_device())
    extra = np.concatenate([intr.reshape(-1), th if per_query else np.empty(0), offsets.view(np.float64)])
    if is_np:
        host = np.concatenate([np.concatenate(rows, 0).reshape(-1) if N else np.empty(0), extra])
        d = torch.from_numpy(host).to(dev)
        rd = d[:5 * N].view(N, 5) if N else torch.zeros(1, 5, dtype=torch.float64, device=dev)
        ex = d[5 * N:]
    else:
        rd = torch.cat(rows).contiguous() if N else torch.zeros(1, 5, dtype=torch.float64, device=dev)
        ex = torch.from_numpy(extra).to(dev)
    offs = ex[4 * nq + (nq if per_query else 0):].view(torch.int64)
    out = torch.empty(12 * nq + (nq + 1) // 2 + (N + 7) // 8 + 1, dtype=torch.float64, device=dev)
    base = out.data_ptr()
    cnt_ptr, mask_ptr = base + 96 * nq, base + 8 * (12 * nq + (nq + 1) // 2)
    find_absolute_pose_batch_into(_lib.default_handle(dev), rd, 5, offs, offsets, None, ex.data_ptr(),
                                  float(th[0]), ex.data_ptr() + 32 * nq if per_query else None, conf, max_iters, seed,
                                  base, mask_ptr, cnt_ptr)
    mask = out[12 * nq + (nq + 1) // 2:].view(torch.uint8)
    if not is_np:
        return [(out[12 * k:12 * k + 9].view(3, 3), out[12 * k + 9:12 * k + 12], mask[offsets[k]:offsets[k + 1]].bool())
                for k in range(nq)]
    host = out.cpu().numpy()
    counts = host[12 * nq:12 * nq + (nq + 1) // 2].view(np.int32)[:nq]
    masks = host[12 * nq + (nq + 1) // 2:].view(np.uint8)
    res = []
    for k in range(nq):
        if counts[k] < 0:
            raise ValueError(f'find_absolute_pose: a value is not finite (query {k})')
        m = masks[offsets[k]:offsets[k + 1]].astype(bool)
        if counts[k] == 0:
            res.append((None, None, m))
        else:
            res.append((host[12 * k:12 * k + 9].reshape(3, 3).copy(), host[12 * k + 9:12 * k + 12].copy(), m))
    return res


def find_absolute_pose(pts2d, pts3d, K, px_th, conf=0.99999, max_iters=10000, seed=0):
    """RANSAC absolute pose from [n, 2] pixels and [n, 3] world points -> (R, t, inlier mask), x_cam = R X + t; R and t
    are None when there is no model (numpy input; NaN for CUDA tensors).  K: 3x3 pinhole matrix or (fx, fy, cx, cy)."""
    return find_absolute_poses([pts2d], [pts3d], K, px_th, conf, max_iters, seed)[0]


def first_absolute_pose_hypotheses(pts2d, pts3d, K, px_th, count, seed=0):
    """Test hook: the first `count` hypotheses without selection -> (models [count * 4, 12] float64 in the centred
    frame, counts [count * 4] int32, -1 where a slot holds no pose)."""
    rows = torch.from_numpy(np.concatenate([np.asarray(pts2d, dtype=np.float64).reshape(-1, 2),
                                            np.asarray(pts3d, dtype=np.float64).reshape(-1, 3)], 1)).cuda()
    models = torch.empty(count * 4, 12, dtype=torch.float64, device=rows.device)
    counts = torch.empty(count * 4, dtype=torch.int32, device=rows.device)
    h = _lib.default_handle(rows.device)
    intr = (C.c_double * 4)(*_camera(K))
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_test_absolute_pose_hypotheses(h.h, _lib.ptr(rows), 5, int(rows.shape[0]), intr,
                                                           float(px_th), int(seed) & (2 ** 64 - 1), int(count),
                                                           _lib.ptr(models), _lib.ptr(counts), h.stream()))
    return models.cpu().numpy(), counts.cpu().numpy()


# ---- the scan lift -----------------------------------------------------------------------------------------------------
def lift_scan_into(handle, scan, align, matches, match_stride, n, n_dev, rows_out, row_stride, capacity, count_ptr):
    """Enqueue p2p_lift_scan: scan a CUDA float64 [H, W, 3] tensor, align a host 4x4, matches a CUDA float64 tensor
    (row r at r * match_stride, n rows, n_dev a ctypes device address or None), rows_out a CUDA float64 tensor,
    count_ptr the device address of the running count (a double)."""
    a = np.ascontiguousarray(align, dtype=np.float64).reshape(16)
    H, W = int(scan.shape[0]), int(scan.shape[1])
    with torch.cuda.device(scan.device):
        _lib.check(handle.lib.p2p_lift_scan(handle.h, C.c_void_p(scan.data_ptr()), H, W, (C.c_double * 16)(*a),
                                            C.c_void_p(matches.data_ptr()), int(match_stride), int(n), n_dev,
                                            C.c_void_p(rows_out.data_ptr()), int(row_stride), int(capacity),
                                            C.c_void_p(count_ptr), handle.stream()))


def lift_scans(items, device=None):
    """Lift several cutouts' matches into one row block, in order: items [(scan [H, W, 3], align 4x4, matches [N, 4])]
    (numpy or CUDA) -> numpy rows [m, 5] (xq, yq, X, Y, Z).  Synchronises (it reads the count back)."""
    dev = device or torch.device('cuda', torch.cuda.current_device())
    h = _lib.default_handle(dev)
    cap = sum(int(np.shape(m)[0]) for _, _, m in items)
    rows = torch.empty(max(cap, 1), 5, dtype=torch.float64, device=dev)
    count = torch.zeros(1, dtype=torch.float64, device=dev)
    keep = []
    for scan, align, m in items:
        s = torch.as_tensor(np.ascontiguousarray(scan, dtype=np.float64) if isinstance(scan, np.ndarray) else scan,
                            dtype=torch.float64, device=dev).contiguous()
        mt = torch.as_tensor(np.ascontiguousarray(m, dtype=np.float64) if isinstance(m, np.ndarray) else m,
                             dtype=torch.float64, device=dev).reshape(-1, 4).contiguous()
        keep.append((s, mt))
        lift_scan_into(h, s, align, mt, 4, int(mt.shape[0]), None, rows, 5, cap, count.data_ptr())
    m = int(count.item())
    return rows[:m].cpu().numpy()


# ---- InLoc files -------------------------------------------------------------------------------------------------------
def read_retrieval(path):
    """hloc's retrieval list ('query db' per line; blank lines skipped) -> [(query, [db, ...])] grouped by query in
    order of first appearance.  Raises ValueError naming the line on a line without exactly two fields."""
    order, groups = [], {}
    with open(path) as f:
        for ln, line in enumerate(f, 1):
            tok = line.split()
            if not tok:
                continue
            if len(tok) != 2:
                raise ValueError(f'{path}:{ln}: expected 2 fields (query db), got {len(tok)}')
            if tok[0] not in groups:
                groups[tok[0]] = []
                order.append(tok[0])
            groups[tok[0]].append(tok[1])
    return [(q, groups[q]) for q in order]


def read_scan(path):
    """A cutout's scan: `XYZcut` of its .mat file -> C-contiguous float64 [H, W, 3]."""
    from scipy.io import loadmat
    m = loadmat(path)
    if 'XYZcut' not in m:
        raise ValueError(f'{path}: no XYZcut variable')
    x = np.ascontiguousarray(m['XYZcut'], dtype=np.float64)
    if x.ndim != 3 or x.shape[2] != 3:
        raise ValueError(f'{path}: XYZcut must be [H, W, 3], got {x.shape}')
    return x


def alignment_path(data_root, db_name):
    """database/alignments/<floor>/transformations/<building>_trans_<scan>.txt of cutout .../<floor>/<scan>/<image>."""
    parts = db_name.replace('\\', '/').split('/')
    if len(parts) < 3:
        raise ValueError(f'{db_name}: a cutout path is .../<floor>/<scan>/<image>')
    floor, scan, image = parts[-3], parts[-2], parts[-1]
    return os.path.join(data_root, 'database', 'alignments', floor, 'transformations',
                        f'{image[:3]}_trans_{scan}.txt')


def read_alignment(path):
    """P_after_GICP: the 4x4 on lines 7-10 (counted from 0) of a scan's transformation file."""
    with open(path) as f:
        lines = f.readlines()
    try:
        A = np.array([[float(v) for v in lines[i].split()] for i in range(7, 11)], dtype=np.float64)
    except (IndexError, ValueError):
        raise ValueError(f'{path}: lines 7-10 must hold the 4x4 P_after_GICP') from None
    if A.shape != (4, 4) or not np.all(np.isfinite(A)):
        raise ValueError(f'{path}: lines 7-10 must hold a finite 4x4 matrix, got shape {A.shape}')
    return A


def rotmat_to_qvec(R):
    """Unit quaternion (w, x, y, z), w >= 0, of a rotation matrix."""
    R = np.asarray(R, dtype=np.float64)
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0:
        s = 2.0 * np.sqrt(tr + 1.0)
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = 2.0 * np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2])
        q = np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    elif R[1, 1] > R[2, 2]:
        s = 2.0 * np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2])
        q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
    else:
        s = 2.0 * np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1])
        q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])
    q /= np.linalg.norm(q)
    return -q if q[0] < 0 else q


def qvec_to_rotmat(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def write_results(path, poses):
    """poses: [(name, R, t)] -> 'name qw qx qy qz tx ty tz' per line (%.17g)."""
    with open(path, 'w') as f:
        for name, R, t in poses:
            v = np.concatenate([rotmat_to_qvec(R), np.asarray(t, dtype=np.float64).reshape(3)])
            f.write(' '.join([name] + ['%.17g' % x for x in v]) + '\n')


def read_results(path):
    """A results file -> {name: (R, t)}.  Raises ValueError naming the line on a malformed line."""
    out = {}
    with open(path) as f:
        for ln, line in enumerate(f, 1):
            tok = line.split()
            if not tok:
                continue
            if len(tok) != 8:
                raise ValueError(f'{path}:{ln}: expected 8 fields (name qw qx qy qz tx ty tz), got {len(tok)}')
            try:
                v = np.array([float(x) for x in tok[1:]])
            except ValueError as e:
                raise ValueError(f'{path}:{ln}: {e}') from None
            out[tok[0]] = (qvec_to_rotmat(v[:4]), v[4:])
    return out


def eval_localization(results, gt, thresholds=((0.25, 10), (0.5, 10), (1.0, 10))):
    """Share of ground-truth queries whose estimated camera centre lies within d metres of the true one and whose
    rotation lies within a degrees, for each (d, a) in thresholds.  results, gt: {name: (R, t)} or results files.  A
    query missing from results counts as a miss.  -> dict(recall={(d, a): share}, errors={name: (position error,
    rotation error in degrees)}); NaN recalls for an empty gt."""
    res = read_results(results) if isinstance(results, (str, os.PathLike)) else results
    gt = read_results(gt) if isinstance(gt, (str, os.PathLike)) else gt
    errs = {}
    for name, (Rg, tg) in gt.items():
        if name not in res:
            errs[name] = (np.inf, np.inf)
            continue
        R, t = (np.asarray(x, dtype=np.float64) for x in res[name])
        Rg, tg = np.asarray(Rg, dtype=np.float64), np.asarray(tg, dtype=np.float64)
        dp = float(np.linalg.norm(-R.T @ t.reshape(3) + Rg.T @ tg.reshape(3)))
        c = np.clip((np.trace(Rg.T @ R) - 1.0) / 2.0, -1.0, 1.0)
        errs[name] = (dp, float(np.degrees(np.arccos(c))))
    e = np.array(list(errs.values()), dtype=np.float64).reshape(-1, 2)
    recall = {(float(d), float(a)): (float(np.mean((e[:, 0] <= d) & (e[:, 1] <= a))) if len(e) else float('nan'))
              for d, a in thresholds}
    return dict(recall=recall, errors=errs)


# ---- the protocol ------------------------------------------------------------------------------------------------------
def _load_query(data_root, q, net):
    from PIL import Image
    im = Image.open(os.path.join(data_root, q))
    w, h = im.size
    return (w, h), (np.asarray(im.convert('RGB')) if net else None)


def _load_db(data_root, db, net):
    from PIL import Image
    scan = torch.from_numpy(read_scan(os.path.join(data_root, db + '.mat'))).pin_memory()
    align = read_alignment(alignment_path(data_root, db))
    img = np.asarray(Image.open(os.path.join(data_root, db)).convert('RGB')) if net else None
    return scan, align, img


class _Block:
    """One query's lifted rows: a device block grown by doubling (stream-ordered copies, no sync) and its running
    device count."""

    def __init__(self, dev):
        self.rows = torch.empty(64, 5, dtype=torch.float64, device=dev)
        self.count = torch.zeros(1, dtype=torch.float64, device=dev)
        self.cap = 0

    def reserve(self, extra):
        need = self.cap + extra
        if need > self.rows.shape[0]:
            grown = torch.empty(max(need, 2 * self.rows.shape[0]), 5, dtype=torch.float64, device=self.rows.device)
            grown[:self.cap].copy_(self.rows[:self.cap])
            self.rows = grown
        self.cap = need


def localize_inloc(matcher, data_root, pairs, results_path, ksize=2, eval_type='fine', io_thres=0.25, imsize=1024,
                   ransac_thres=48.0, chunk_queries=64, conf=0.99999, max_iters=10000, lprint_=print):
    """Localize the queries of an InLoc retrieval list and write the results file (protocol in the module docstring).

    `matcher` is a Patch2PixB200 (run as estimate_matches_from_files(net, query, db, ksize, 0.0, True, io_thres,
    eval_type, imsize) would run it, the query as image 1), or any callable (query_path, db_path) returning [N, 4]
    rows (xq, yq, xdb, ydb) in original-image pixels as numpy or a torch tensor (or a tuple whose first element is
    those).  `pairs` is a retrieval-list file or a list as read_retrieval returns it.

    -> dict(poses={query name: (R, t, n_inliers)}, failed=[(query, reason)], n_queries, time)."""
    from .model import Patch2PixB200
    if not (ransac_thres > 0 and np.isfinite(ransac_thres)):
        raise ValueError('ransac_thres must be positive')
    if int(chunk_queries) < 1:
        raise ValueError('chunk_queries must be at least 1')
    retrieval = read_retrieval(pairs) if isinstance(pairs, (str, os.PathLike)) else list(pairs)
    is_net = isinstance(matcher, Patch2PixB200)
    if is_net:
        matcher.eval()
        dev = matcher.device
    else:
        dev = torch.device('cuda', torch.cuda.current_device())
    lprint_(f'\n>>Localize InLoc: {len(retrieval)} queries, {sum(len(d) for _, d in retrieval)} pairs, '
            f'rthres={ransac_thres}')
    start = time.time()
    h = matcher._handle if is_net else _lib.default_handle(dev)
    nq = len(retrieval)
    table = torch.zeros(max(nq, 1), 13, dtype=torch.float64, device=dev)     # R|t [12], int32 count in element 12
    failed = {}
    jobs = [(i, db) for i, (_, dbs) in enumerate(retrieval) for db in dbs]
    chunk = []

    def flush(k0):
        K = len(chunk)
        if K == 0:
            return
        offsets = np.zeros(K + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([b.cap for b, _ in chunk])
        N = int(offsets[-1])
        rows = torch.cat([b.rows[:b.cap] for b, _ in chunk]) if N else torch.zeros(1, 5, dtype=torch.float64,
                                                                                   device=dev)
        n_t = torch.cat([b.count for b, _ in chunk])
        intr = np.stack([c for _, c in chunk]).reshape(-1)
        ex = torch.from_numpy(np.concatenate([intr, offsets.view(np.float64)])).pin_memory().to(dev, non_blocking=True)
        mask = torch.empty(N + 1, dtype=torch.uint8, device=dev)
        cnt = torch.empty(K, dtype=torch.int32, device=dev)
        rt = torch.empty(K, 12, dtype=torch.float64, device=dev)
        find_absolute_pose_batch_into(h, rows, 5, ex[4 * K:].view(torch.int64), offsets, C.c_void_p(n_t.data_ptr()),
                                      ex.data_ptr(), ransac_thres, None, conf, max_iters, 0, rt.data_ptr(),
                                      mask.data_ptr(), cnt.data_ptr())
        table[k0:k0 + K, :12].copy_(rt)
        table[k0:k0 + K, 12:13].view(torch.int32)[:, 0].copy_(cnt)
        chunk.clear()

    with ThreadPoolExecutor(max_workers=1) as pool:
        qfut = {0: pool.submit(_load_query, data_root, retrieval[0][0], is_net)} if nq else {}
        dfut = [pool.submit(_load_db, data_root, jobs[0][1], is_net)] if jobs else []
        j = 0
        k0 = 0
        for i, (q, dbs) in enumerate(retrieval):
            if i + 1 < nq:
                qfut[i + 1] = pool.submit(_load_query, data_root, retrieval[i + 1][0], is_net)
            block = _Block(dev)
            xq = scq = None
            try:
                (w, hgt), qimg = qfut.pop(i).result()
                cam = np.array([INLOC_FOCAL, INLOC_FOCAL, 0.5 * w, 0.5 * hgt])
                if is_net:
                    from .preprocess import preprocess_image
                    xq, scq = preprocess_image(qimg, ksize, matcher.upsample, imsize, dev, h)
            except Exception as e:
                failed[i] = f'{type(e).__name__}: {e}'
                cam = np.array([INLOC_FOCAL, INLOC_FOCAL, 0.5, 0.5])
            for _ in dbs:
                cur = dfut.pop(0)
                if j + 1 < len(jobs):
                    dfut.append(pool.submit(_load_db, data_root, jobs[j + 1][1], is_net))
                db = jobs[j][1]
                j += 1
                if i in failed:
                    continue
                try:
                    scan_h, align, dimg = cur.result()
                    if is_net:
                        from .eval_helper import match_device
                        from .preprocess import preprocess_image
                        xd, scd = preprocess_image(dimg, ksize, matcher.upsample, imsize, dev, h)
                        packed, n, _ = match_device(matcher, xq.unsqueeze(0), xd.unsqueeze(0), scq, scd, ksize, 0.0,
                                                    True, io_thres, eval_type, None)
                        mt, stride, n_dev = packed, 9, C.c_void_p(packed.data_ptr() + 72 * n)
                    else:
                        from .hpatches import _as_rows
                        mt = _as_rows(matcher(os.path.join(data_root, q), os.path.join(data_root, db)), dev)
                        n, stride, n_dev = int(mt.shape[0]), 4, None
                    if n:
                        scan = scan_h.to(dev, non_blocking=True)
                        block.reserve(n)
                        lift_scan_into(h, scan, align, mt, stride, n, n_dev, block.rows, 5, block.cap,
                                       block.count.data_ptr())
                except Exception as e:
                    failed[i] = f'{type(e).__name__}: {e}'
            if i in failed:
                block = _Block(dev)
            chunk.append((block, cam))
            if len(chunk) == int(chunk_queries):
                flush(k0)
                k0 = i + 1
        flush(k0)
    host = table.cpu().numpy()                       # the run's one copy of the poses
    runtime = time.time() - start
    poses, out = {}, []
    for i, (q, _) in enumerate(retrieval):
        cnt = int(host[i, 12:13].view(np.int32)[0])
        R, t = host[i, :9].reshape(3, 3).copy(), host[i, 9:12].copy()
        if i not in failed and cnt <= 0:
            failed[i] = 'no model'
        if i in failed:
            R, t = np.eye(3), np.zeros(3)
        name = os.path.basename(q)
        poses[name] = (R, t, cnt)
        out.append((name, R, t))
    write_results(results_path, out)
    lprint_(f'localized {nq - len(failed)} / {nq} queries, time={runtime:.2f}s -> {results_path}')
    return dict(poses=poses, failed=[(retrieval[i][0], failed[i]) for i in sorted(failed)], n_queries=nq,
                time=runtime)


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description='Localize InLoc queries with a Patch2Pix or NCNet checkpoint and write '
                                             'the results file of the InLoc benchmark.')
    ap.add_argument('--ckpt', required=True, help='checkpoint file (eval_helper.load_checkpoint)')
    ap.add_argument('--data_root', required=True, help='InLoc root: query/ and database/ (cutouts, alignments)')
    ap.add_argument('--pairs', required=True, help="hloc's retrieval list, 'query db' per line")
    ap.add_argument('--results', required=True, help='output: name qw qx qy qz tx ty tz per query')
    ap.add_argument('--method', default='patch2pix', choices=('patch2pix', 'nc'),
                    help="'patch2pix': fine matches; 'nc': the coarse NCNet matches of the checkpoint")
    ap.add_argument('--ksize', type=int, default=2)
    ap.add_argument('--io_thres', type=float, default=0.25)
    ap.add_argument('--imsize', type=int, default=1024)
    ap.add_argument('--ransac_thres', type=float, default=48.0)
    ap.add_argument('--chunk_queries', type=int, default=64)
    args = ap.parse_args(argv)
    if not os.path.isdir(args.data_root):
        ap.error(f'--data_root {args.data_root} is not a directory')
    if not os.path.isfile(args.pairs):
        ap.error(f'--pairs {args.pairs} is not a file')
    if not os.path.isfile(args.ckpt):
        ap.error(f'--ckpt {args.ckpt} is not a file')
    if not (args.ransac_thres > 0 and np.isfinite(args.ransac_thres)):
        ap.error('--ransac_thres must be positive')
    if args.chunk_queries < 1:
        ap.error('--chunk_queries must be at least 1')
    from .eval_helper import load_checkpoint
    net = load_checkpoint(args.ckpt, method=args.method)
    localize_inloc(net, args.data_root, args.pairs, args.results, ksize=args.ksize,
                   eval_type='coarse' if args.method == 'nc' else 'fine', io_thres=args.io_thres, imsize=args.imsize,
                   ransac_thres=args.ransac_thres, chunk_queries=args.chunk_queries)


if __name__ == '__main__':
    main()
