"""Relative-pose evaluation on MegaDepth-1500 / ScanNet-1500-style pair lists: pose AUC and epipolar precision, with the
RANSAC and the per-pair statistics of many pairs in one batched pass on the device.

    python -m patch2pix_b200.relpose --ckpt PATH --pairs FILE --data_root DIR [--method patch2pix|nc]

The protocol (the relative-pose evaluation of SuperGlue and LoFTR, by which detector-free matchers are ranked):

* Pairs come with intrinsics K0, K1 (3x3, pixels of the original images) and the ground-truth relative pose T_0to1
  (x1 = R x0 + t; t is not normalised).  Two pair-list formats are read:
  - SuperGlue's text format (ScanNet-1500, YFCC): one pair per line, ``name0 name1 rot0 rot1 K0 (9) K1 (9) T_0to1
    (16)``, images at data_root/name.  A non-zero rot (EXIF rotation) raises ValueError: it is not supported.
  - LoFTR's scene-info ``.npz`` (MegaDepth-1500): ``image_paths`` (relative to data_root), ``intrinsics`` [N, 3, 3],
    ``poses`` [N, 4, 4] world -> camera, ``pair_infos`` of ((i, j), overlap, ...); T_0to1 = poses[j] @ inv(poses[i]).
  A ground-truth t of zero norm raises ValueError, naming the pair.
* Matches are [N, 4] float64 rows (x0, y0, x1, y1) in original-image pixels.  E is estimated by the essential-matrix
  RANSAC of patch2pix_b200.pose at the camera-coordinate threshold ransac_thres / f_mean, f_mean = mean(K0[0, 0],
  K1[1, 1], K0[0, 0], K1[1, 1]) (conf 0.99999, 1000 iterations, seed 0), and the pose recovered from its inliers with
  distance threshold 1e9.  The engine returns one E, where cv2.findEssentialMat may return several, and its sampler and
  local optimisation differ from OpenCV's: the AUC differs from an OpenCV flow within RANSAC's randomness.
* R_err = arccos((tr(R_gt^T R) - 1) / 2), t_err = arccos(t_gt . t / (|t_gt| |t|)) folded to min(t_err, 180 - t_err)
  (E fixes t up to sign), in degrees; the pose error is max(R_err, t_err), +inf when RANSAC finds no model (fewer
  than 5 matches, among others) or the matcher raised (the pair is also listed as failed).
* AUC@t (t = 5, 10, 20 degrees by default) over every pair, failed ones included: errors sorted, recall (i + 1) / N,
  (0, 0) prepended, the curve cut at t (an error equal to t falls outside), trapezoid rule, divided by t.
* Precision at an epipolar threshold e (5e-4 by default): per pair, the share of its matches whose symmetric epipolar
  error in normalised coordinates under the ground-truth E = [t_gt]x R_gt is below e (0 for a pair without matches),
  averaged over pairs.  It does not depend on the estimator.  An empty pair list gives NaN for AUC and precision.

Every `chunk_pairs` pairs, the matches of the chunk are concatenated on the device and go through one
p2p_find_essential_batch_th, one p2p_recover_pose_batch and one p2p_relpose_errors_batch, which write the pairs'
records into a device table; the table comes back in one copy at the end of the run.  The host takes the arccos of the
cosines the device returns (the device's acos is not correctly rounded) and computes the statistics.
"""
import ctypes as C
import os
import time
from argparse import Namespace

import numpy as np
import torch

from . import _lib
from .eval_helper import PairRunner, check_thresholds, prefetch

DIST_TH = 1e9             # the protocol's recoverPose(..., 1e9, mask)

# A record is one float64 row of the device table: int32 E-RANSAC inlier count and int32 good-point count in element 0,
# the cosines of the rotation and translation-direction errors in 1 and 2, the int32 counts of p2p_relpose_errors_batch
# ([n_thr + 1]: rows under each epipolar threshold, then the rows considered) from element 3, then the estimated R|t
# [12].
_REC_COS = 1
_REC_COUNTS = 3


def _rec_rt(n_thr):
    return _REC_COUNTS + (n_thr + 2) // 2


def _rec_len(n_thr):
    return _rec_rt(n_thr) + 12


# ---- pair lists ------------------------------------------------------------------------------------------------------
def _pair(name0, name1, path0, path1, K0, K1, T, where):
    K0 = np.asarray(K0, dtype=np.float64).reshape(3, 3)
    K1 = np.asarray(K1, dtype=np.float64).reshape(3, 3)
    T = np.asarray(T, dtype=np.float64).reshape(4, 4)
    if not (np.all(np.isfinite(K0)) and np.all(np.isfinite(K1)) and np.all(np.isfinite(T))):
        raise ValueError(f'{where}: intrinsics and pose must be finite')
    if min(K0[0, 0], K0[1, 1], K1[0, 0], K1[1, 1]) <= 0:
        raise ValueError(f'{where}: focal lengths must be positive')
    if not np.linalg.norm(T[:3, 3]) > 0:
        raise ValueError(f'{where}: the ground-truth translation of {name0} -> {name1} has zero norm, so its direction '
                         f'error is undefined')
    return Namespace(name0=name0, name1=name1, path0=path0, path1=path1, K0=K0, K1=K1, T_0to1=T)


def read_pairs_txt(path, data_root):
    """SuperGlue's pair list (one pair per line: name0 name1 rot0 rot1 K0 (9) K1 (9) T_0to1 (16), whitespace-separated;
    blank lines skipped) -> [Namespace(name0, name1, path0, path1, K0, K1, T_0to1)], images at data_root/name.
    Raises ValueError naming the line on a malformed line, a non-zero rotation, or a zero ground-truth translation."""
    pairs = []
    with open(path) as f:
        for ln, line in enumerate(f, 1):
            tok = line.split()
            if not tok:
                continue
            where = f'{path}:{ln}'
            if len(tok) != 38:
                raise ValueError(f'{where}: expected 38 fields (name0 name1 rot0 rot1 K0 K1 T_0to1), got {len(tok)}')
            try:
                rot = (int(tok[2]), int(tok[3]))
                vals = np.array([float(v) for v in tok[4:]], dtype=np.float64)
            except ValueError as e:
                raise ValueError(f'{where}: {e}') from None
            if rot != (0, 0):
                raise ValueError(f'{where}: EXIF rotation {rot} is not supported (only 0 0)')
            pairs.append(_pair(tok[0], tok[1], os.path.join(data_root, tok[0]), os.path.join(data_root, tok[1]),
                               vals[:9], vals[9:18], vals[18:], where))
    return pairs


def read_pairs_npz(path, data_root):
    """LoFTR's scene-info file (image_paths, intrinsics [N, 3, 3], poses [N, 4, 4] world -> camera, pair_infos of
    ((i, j), overlap, ...)) -> pairs as read_pairs_txt, T_0to1 = poses[j] @ inv(poses[i]), images at
    data_root/image_paths[i].  Raises ValueError on a missing key or a zero ground-truth translation."""
    with np.load(path, allow_pickle=True) as z:
        missing = [k for k in ('image_paths', 'intrinsics', 'poses', 'pair_infos') if k not in z.files]
        if missing:
            raise ValueError(f'{path}: missing {missing} (a scene-info file has image_paths, intrinsics, poses and '
                             f'pair_infos)')
        paths, Ks, poses, infos = z['image_paths'], z['intrinsics'], z['poses'], z['pair_infos']
    pairs = []
    for p, info in enumerate(infos):
        try:
            i, j = (int(v) for v in info[0])
        except (TypeError, ValueError, IndexError):
            raise ValueError(f'{path}: pair_infos[{p}] is not ((i, j), overlap, ...)') from None
        n0, n1 = str(paths[i]), str(paths[j])
        T = np.asarray(poses[j], dtype=np.float64) @ np.linalg.inv(np.asarray(poses[i], dtype=np.float64))
        pairs.append(_pair(n0, n1, os.path.join(data_root, n0), os.path.join(data_root, n1), Ks[i], Ks[j], T,
                           f'{path}: pair_infos[{p}]'))
    return pairs


def read_pairs(pairs, data_root):
    """A pair-list file (.npz: read_pairs_npz, anything else: read_pairs_txt), or a list of pairs as they return."""
    if isinstance(pairs, (str, os.PathLike)):
        return (read_pairs_npz if str(pairs).endswith('.npz') else read_pairs_txt)(pairs, data_root)
    return list(pairs)


def pair_arrays(pairs, ransac_thres):
    """(intr [K, 8] as pose.intrinsics(K0, K1), T_0to1 as [K, 12] R|t, px_th [K]) of the pairs: px_th_k = ransac_thres *
    ((fx1 + fy1) / 2) / f_mean_k, the pixel threshold at which the engine's camera-coordinate threshold px_th /
    ((fx1 + fy1) / 2) is the protocol's ransac_thres / f_mean_k."""
    K = len(pairs)
    intr, Rt, px = np.empty((K, 8)), np.empty((K, 12)), np.empty(K)
    for k, p in enumerate(pairs):
        intr[k] = (p.K0[0, 0], p.K0[1, 1], p.K0[0, 2], p.K0[1, 2], p.K1[0, 0], p.K1[1, 1], p.K1[0, 2], p.K1[1, 2])
        Rt[k, :9] = p.T_0to1[:3, :3].reshape(9)
        Rt[k, 9:] = p.T_0to1[:3, 3]
        f_mean = np.mean([p.K0[0, 0], p.K1[1, 1], p.K0[0, 0], p.K1[1, 1]])
        px[k] = ransac_thres * ((p.K1[0, 0] + p.K1[1, 1]) / 2.0) / f_mean
    return intr, Rt, px


# ---- device entry points -------------------------------------------------------------------------------------------
def relpose_errors_batch_into(handle, rows, row_stride, offsets, offsets_host, n_dev, intr_ptr, Rt_gt_ptr, Rt_est_ptr,
                              n_inliers_ptr, thresholds, out_ptr, out_stride):
    """Enqueue p2p_relpose_errors_batch (device addresses; thresholds a host array; out_stride in doubles)."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    t = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(-1)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_relpose_errors_batch(
            handle.h, C.c_void_p(rows.data_ptr()), row_stride, C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, C.c_void_p(intr_ptr), C.c_void_p(Rt_gt_ptr),
            C.c_void_p(Rt_est_ptr), C.c_void_p(n_inliers_ptr), (C.c_double * len(t))(*t), len(t), C.c_void_p(out_ptr),
            int(out_stride), handle.stream()))


def relpose_errors(rows_list, intr, Rt_gt, Rt_est, n_inliers, thresholds=(5e-4,)):
    """p2p_relpose_errors_batch on K pairs: rows_list [K] of CUDA [n_k, >= 4] rows (x0, y0, x1, y1 in columns 0..3),
    intr [K, 8], Rt_gt / Rt_est [K, 12], n_inliers [K] (host arrays or CUDA tensors) -> (cosines float64 CUDA [K, 2]
    (rotation, translation direction; NaN where n_inliers <= 0), counts int32 CUDA [K, len(thresholds) + 1]).  No host
    sync."""
    t = check_thresholds(thresholds)
    K = len(rows_list)
    if K == 0:
        raise ValueError('relpose_errors needs at least one pair')
    dev = rows_list[0].device
    rows = torch.cat([r[:, :4].to(torch.float64) for r in rows_list]).contiguous()
    offsets = np.zeros(K + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([int(r.shape[0]) for r in rows_list])
    intr_d, gt_d, est_d = (torch.as_tensor(x, dtype=torch.float64).to(dev).reshape(K, w).contiguous()
                           for x, w in ((intr, 8), (Rt_gt, 12), (Rt_est, 12)))
    cnt_d = torch.as_tensor(n_inliers).to(device=dev, dtype=torch.int32).reshape(K).contiguous()
    L = 2 + (t.size + 2) // 2
    out = torch.zeros(K, L, dtype=torch.float64, device=dev)
    relpose_errors_batch_into(_lib.default_handle(dev), rows, 4, torch.from_numpy(offsets).to(dev), offsets, None,
                              intr_d.data_ptr(), gt_d.data_ptr(), est_d.data_ptr(), cnt_d.data_ptr(), t,
                              out.data_ptr(), L)
    return out[:, :2], out[:, 2:].contiguous().view(torch.int32)[:, :t.size + 1]


# ---- evaluation -------------------------------------------------------------------------------------------------------
class _Table:
    """The device record table and the chunk being gathered: per pair its rows ([n, stride] CUDA float64) and, for
    Patch2Pix rows, the device kept-row count."""

    def __init__(self, dev, pairs, ransac_thres, conf, max_iters, epi, chunk_pairs):
        self.dev, self.epi, self.conf, self.max_iters, self.chunk = dev, epi, conf, max_iters, chunk_pairs
        self.L = _rec_len(epi.size)
        self.table = torch.zeros(len(pairs), self.L, dtype=torch.float64, device=dev)
        intr, Rt, px = pair_arrays(pairs, ransac_thres)
        gt = torch.from_numpy(np.concatenate((intr.reshape(-1), Rt.reshape(-1), px))).to(dev)
        K = len(pairs)
        self.intr, self.Rt_gt, self.px = gt[:8 * K], gt[8 * K:20 * K], gt[20 * K:]
        self.h = _lib.default_handle(dev)
        self.k0, self.items = 0, []

    def add(self, rows, n_dev=None):
        self.items.append((rows, n_dev))
        if len(self.items) == self.chunk:
            self.flush()

    def flush(self):
        K, k0 = len(self.items), self.k0
        if K == 0:
            return
        stride = int(self.items[0][0].shape[1])
        rows = torch.cat([r for r, _ in self.items]).contiguous()
        if rows.shape[0] == 0:
            rows = torch.zeros(1, stride, dtype=torch.float64, device=self.dev)     # a valid pointer for the launches
        n_t = torch.cat([n for _, n in self.items]) if self.items[0][1] is not None else None
        n_dev = None if n_t is None else C.c_void_p(n_t.data_ptr())       # n_t stays referenced until the launches
        offsets = np.zeros(K + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([int(r.shape[0]) for r, _ in self.items])
        offs = torch.from_numpy(offsets).pin_memory().to(self.dev, non_blocking=True)
        N = int(offsets[-1])
        from . import pose as P
        buf = torch.zeros(P.batch_out_size(K, N), dtype=torch.float64, device=self.dev)
        p = P._batch_ptrs(buf, K, N)
        intr = self.intr.data_ptr() + 64 * k0
        P.find_essential_batch_th_into(self.h, rows, stride, offs, offsets, n_dev, intr, self.px.data_ptr() + 8 * k0,
                                       self.conf, self.max_iters, 0, p['E'], p['emask'], p['cnt'])
        P.recover_pose_batch_into(self.h, rows, stride, offs, offsets, n_dev, intr, p['E'], p['emask'], p['Rt'],
                                  p['pmask'], p['good'], DIST_TH)
        rec = self.table[k0:k0 + K]
        relpose_errors_batch_into(self.h, rows, stride, offs, offsets, n_dev, intr, self.Rt_gt.data_ptr() + 96 * k0,
                                  p['Rt'], p['cnt'], self.epi, rec.data_ptr() + 8 * _REC_COS, self.L)
        rt0 = _rec_rt(self.epi.size)
        rec[:, 0:1].view(torch.int32).copy_(buf[21 * K:22 * K].view(torch.int32).view(2, K).t())
        rec[:, rt0:rt0 + 12].copy_(buf[9 * K:21 * K].view(K, 12))
        self.k0, self.items = k0 + K, []


def parse_record(row, pair, n_thr, failed=False):
    """One pair's Namespace(name0, name1, N, n_inliers, n_good, cos_R, cos_t, R_err, t_err, err, counts, R, t,
    match_failed) from its host table row.  Errors in degrees; +inf without a model or when the matcher raised."""
    ints = row[0:1].view(np.int32)
    cnt = row[_REC_COUNTS:].view(np.int32)[:n_thr + 1].copy()
    rt0 = _rec_rt(n_thr)
    cr, ct = float(row[_REC_COS]), float(row[_REC_COS + 1])
    r_err = t_err = np.inf
    if not failed and np.isfinite(cr) and np.isfinite(ct):
        r_err = float(np.degrees(np.arccos(cr)))
        t_err = float(np.degrees(np.arccos(ct)))
        t_err = min(t_err, 180.0 - t_err)
    return Namespace(name0=pair.name0, name1=pair.name1, N=int(cnt[-1]), n_inliers=int(ints[0]), n_good=int(ints[1]),
                     cos_R=cr, cos_t=ct, R_err=r_err, t_err=t_err, err=max(r_err, t_err), counts=cnt,
                     R=row[rt0:rt0 + 9].reshape(3, 3).copy(), t=row[rt0 + 9:rt0 + 12].copy(), match_failed=failed)


def pose_auc(errors, thresholds):
    """{t: AUC of the pose-error recall curve up to t, divided by t} (module docstring); NaN for an empty list."""
    errors = np.sort(np.asarray(errors, dtype=np.float64).reshape(-1))
    if errors.size == 0:
        return {t: float('nan') for t in thresholds}
    recall = np.r_[0.0, (np.arange(errors.size) + 1) / errors.size]
    errors = np.r_[0.0, errors]
    out = {}
    for t in thresholds:
        last = int(np.searchsorted(errors, t))
        out[t] = float(np.trapezoid(np.r_[recall[:last], recall[last - 1]], x=np.r_[errors[:last], t]) / t)
    return out


def precision(records, thresholds):
    """{e: mean over pairs of correct(e) / N (0 for N = 0)}; NaN for an empty list."""
    if not records:
        return {e: float('nan') for e in thresholds}
    c = np.stack([r.counts for r in records]).astype(np.float64)
    n = c[:, -1:]
    p = np.where(n > 0, c[:, :-1] / np.where(n > 0, n, 1.0), 0.0)
    return {e: float(p[:, j].mean()) for j, e in enumerate(thresholds)}


def eval_relpose(matcher, pairs, data_root, ksize=2, eval_type='fine', io_thres=0.25, ncn_thres=0.0, imsize=1024,
                 ransac_thres=0.5, conf=0.99999, max_iters=1000, epi_thresholds=(5e-4,), auc_thresholds=(5, 10, 20),
                 chunk_pairs=512, lprint_=print):
    """Pose AUC and epipolar precision of `matcher` on a pair list (protocol in the module docstring).

    `matcher` is a Patch2PixB200 (run as estimate_matches_from_files(..., ksize, ncn_thres, True, io_thres, eval_type,
    imsize) would run it), or any callable (im0_path, im1_path) returning [N, 4] rows as numpy or a torch tensor, or a
    tuple whose first element is those rows.  `pairs` is a pair-list file (read_pairs) or a list of pairs as
    read_pairs returns them; image paths are relative to `data_root`.

    -> dict(auc={t: AUC@t}, prec={e: precision@e}, n_matches: mean matches per pair, failed: [(index, name0, name1,
    error text)] of the pairs whose matcher raised, records: one Namespace per pair (parse_record), n_pairs, time)."""
    epi = check_thresholds(epi_thresholds, 'epi_thresholds')
    auc_t = [float(t) for t in check_thresholds(auc_thresholds, 'auc_thresholds')]
    if not (ransac_thres > 0 and np.isfinite(ransac_thres)):
        raise ValueError('ransac_thres must be positive')
    if not (int(chunk_pairs) >= 1):
        raise ValueError('chunk_pairs must be at least 1')
    pairs = read_pairs(pairs, data_root)
    run = PairRunner(matcher, ksize, eval_type, io_thres, ncn_thres, imsize)
    lprint_(f'\n>>Eval relative pose: {len(pairs)} pairs, '
            + (f'eval_type={eval_type} ksize={ksize} io={io_thres} nc={ncn_thres} im={imsize} ' if run.is_net else '')
            + f'rthres={ransac_thres} conf={conf}')
    start = time.time()
    tab = _Table(run.dev, pairs, ransac_thres, conf, max_iters, epi, int(chunk_pairs))
    failed = {}
    # a failed pair adds no rows; Patch2Pix rows are the packed [n, 9] rows with their device count
    empty = torch.zeros(0, 9 if run.is_net else 4, dtype=torch.float64, device=run.dev)
    zero = torch.zeros(1, dtype=torch.float64, device=run.dev) if run.is_net else None
    for i, ims in prefetch(pairs, lambda p: run.decode([p.path0, p.path1])):
        try:
            if isinstance(ims, Exception):
                raise ims
            if run.is_net:
                packed, n = run.match(run.prepare(ims[0]), run.prepare(ims[1]))
                item = packed[:n * 9].view(n, 9), packed[n * 9:n * 9 + 1]
            else:
                item = run.call(pairs[i].path0, pairs[i].path1), None
        except Exception as e:
            failed[i] = f'{type(e).__name__}: {e}'
            item = empty, zero
        tab.add(*item)
    tab.flush()
    host = tab.table.cpu().numpy()                    # the run's one copy of the records
    runtime = time.time() - start
    records = [parse_record(host[i], p, epi.size, i in failed) for i, p in enumerate(pairs)]
    auc = pose_auc([r.err for r in records], auc_t)
    prec = precision(records, epi.tolist())
    n_matches = float(np.mean([r.N for r in records])) if records else float('nan')
    lprint_('AUC@{}deg {} prec@{} {} matches={:.1f} no_model={} failed={} time={:.2f}s'.format(
        auc_t, ' '.join(f'{auc[t]:.4f}' for t in auc_t), epi.tolist(), ' '.join(f'{v:.4f}' for v in prec.values()),
        n_matches, sum(1 for r in records if not np.isfinite(r.err)), len(failed), runtime))
    return dict(auc=auc, prec=prec, n_matches=n_matches,
                failed=[(i, pairs[i].name0, pairs[i].name1, failed[i]) for i in sorted(failed)], records=records,
                n_pairs=len(pairs), time=runtime)


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description='Relative-pose AUC and epipolar precision of a Patch2Pix or NCNet '
                                             'checkpoint on a MegaDepth-1500 / ScanNet-1500-style pair list.')
    ap.add_argument('--ckpt', required=True, help='checkpoint file (eval_helper.load_checkpoint)')
    ap.add_argument('--pairs', required=True, help="pair list: SuperGlue's text format, or LoFTR's scene-info .npz")
    ap.add_argument('--data_root', required=True, help='directory the image names of the pair list are relative to')
    ap.add_argument('--method', default='patch2pix', choices=('patch2pix', 'nc'),
                    help="'patch2pix': fine matches; 'nc': the coarse NCNet matches of the checkpoint")
    ap.add_argument('--ksize', type=int, default=2)
    ap.add_argument('--io_thres', type=float, default=0.25)
    ap.add_argument('--ncn_thres', type=float, default=0.0)
    ap.add_argument('--imsize', type=int, default=1024)
    ap.add_argument('--ransac_thres', type=float, default=0.5)
    ap.add_argument('--chunk_pairs', type=int, default=512)
    args = ap.parse_args(argv)
    from .eval_helper import load_checkpoint
    net = load_checkpoint(args.ckpt, method=args.method)
    eval_relpose(net, args.pairs, args.data_root, ksize=args.ksize,
                 eval_type='coarse' if args.method == 'nc' else 'fine', io_thres=args.io_thres,
                 ncn_thres=args.ncn_thres, imsize=args.imsize, ransac_thres=args.ransac_thres,
                 chunk_pairs=args.chunk_pairs)


if __name__ == '__main__':
    main()
