"""HPatches-sequences evaluation: mean matching accuracy (MMA) and homography accuracy, per-pair statistics on the device.

    python -m patch2pix_b200.hpatches --ckpt PATH --data_root hpatches-sequences-release [--method patch2pix|nc]

The protocol (D2-Net's HPatches-sequences protocol for MMA, the usual corner-error protocol for homographies):

* Sequences are the subdirectories of `data_root` in sorted order, each with 1.ppm .. 6.ppm and H_1_2 .. H_1_6
  (3x3, np.loadtxt).  A name starting with ``i_`` is an illumination sequence, ``v_`` a viewpoint one; any other name,
  or a missing file, raises with the path.  `exclude` defaults to D2-Net's eight high-resolution sequences, which
  leaves the 108-sequence split (52 i / 56 v); ``exclude=()`` keeps all of them.
* Each sequence gives the 5 pairs (1, k), k = 2..6.  Matches are [N, 4] float64 rows (x1, y1, x2, y2) in
  original-image pixels.
* A row's reprojection error is d = |pi(H_gt [x1, y1, 1]^T) - (x2, y2)| in fp64; it is correct at threshold t iff
  d <= t (NaN and inf never are).  The pair's MMA at t is correct(t) / N, 0 at every t when N = 0 (the pair still
  counts).  A split's MMA is the mean over its pairs (i, v, and all); an empty split gives NaN.
* The homography is the H RANSAC of patch2pix_b200.verify (one-sided transfer error < ransac_thres, conf 0.999,
  10000 iterations, seed 0; ransac_thres defaults to the 2 px of findHomography(..., 2.0)).  The corner error is the
  mean over the corners (0, 0), (w-1, 0), (0, h-1), (w-1, h-1) of 1.ppm at its original size of
  |pi(H_gt c) - pi(H_pred c)|, +inf when RANSAC found no model (inlier count <= 0: fewer than 4 rows, or a
  non-finite coordinate), a corner projects with w = 0, or the result is not finite.  A split's homography accuracy
  at t is its share of pairs with corner error <= t (t = 1, 3, 5, 10 px by default).
* A pair whose matcher raises is recorded as failed: MMA 0 and corner error +inf.

Per pair, the matcher, the RANSAC and ``p2p_homography_errors`` are enqueued on the device; the pair's record is copied
device to device into a table that comes back in one copy at the end of the run.
"""
import ctypes as C
import os
import time
from argparse import Namespace

import numpy as np
import torch

from . import _lib
from . import verify as V
from .eval_helper import PairRunner, as_rows, check_thresholds, prefetch

D2NET_EXCLUDED = ('i_contruction', 'i_crownnight', 'i_dc', 'i_pencils', 'i_whitebuilding', 'v_artisans',
                  'v_astronautis', 'v_talent')

# A record is one float64 row of the device table: the kept-match count N, the find_model buffer up to its int32
# inlier count (H [9], count in the low half of element 10), the corner error, then the int32 counts [n_thr + 1] of
# p2p_homography_errors (correct rows per threshold, then the rows considered).
_REC_H = 1
_REC_CORNER = 11
_REC_COUNTS = 12


def _rec_len(n_thr):
    return _REC_COUNTS + (n_thr + 2) // 2


def read_hpatches(data_root, exclude=D2NET_EXCLUDED):
    """The sequences of an hpatches-sequences-release directory -> [Namespace(name, split ('i' or 'v'), paths
    [1.ppm .. 6.ppm], H_gt [5 x (3, 3) float64, H_1_2 .. H_1_6], size (width, height) of 1.ppm)] in sorted name order,
    without the names in `exclude`.  Raises ValueError on a subdirectory whose name starts with neither i_ nor v_ and
    FileNotFoundError on a missing file, naming the path."""
    from PIL import Image
    if not os.path.isdir(data_root):
        raise FileNotFoundError(f'{data_root}: not a directory')
    exclude = set(exclude)
    seqs = []
    for name in sorted(os.listdir(data_root)):
        d = os.path.join(data_root, name)
        if not os.path.isdir(d) or name in exclude:
            continue
        if name.startswith('i_'):
            split = 'i'
        elif name.startswith('v_'):
            split = 'v'
        else:
            raise ValueError(f'{d}: an HPatches sequence name starts with i_ (illumination) or v_ (viewpoint)')
        paths = [os.path.join(d, f'{k}.ppm') for k in range(1, 7)]
        h_paths = [os.path.join(d, f'H_1_{k}') for k in range(2, 7)]
        for p in paths + h_paths:
            if not os.path.isfile(p):
                raise FileNotFoundError(f'{p}: missing from the HPatches sequence {name}')
        H_gt = []
        for p in h_paths:
            H = np.loadtxt(p, dtype=np.float64)
            if H.shape != (3, 3):
                raise ValueError(f'{p}: expected a 3x3 matrix, got shape {H.shape}')
            H_gt.append(H)
        with Image.open(paths[0]) as im:
            size = im.size
        seqs.append(Namespace(name=name, split=split, paths=paths, H_gt=H_gt, size=size))
    return seqs


def homography_errors_into(handle, rows, row_stride, n, n_dev, H_gt, H_pred_ptr, width, height, thresholds,
                           counts_ptr, corner_ptr):
    """Enqueue p2p_homography_errors on `rows` (a float64 device tensor, row r at offset r * row_stride) with H_gt and
    the thresholds from the host; `n_dev`, `H_pred_ptr`, `counts_ptr` and `corner_ptr` are device addresses (ctypes;
    n_dev may be None) of the row count, the find_model buffer, the int32 [n_thr + 1] counts and the double corner
    error."""
    H = np.ascontiguousarray(H_gt, dtype=np.float64).reshape(9)
    t = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(-1)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_homography_errors(handle.h, C.c_void_p(rows.data_ptr()), row_stride, n, n_dev,
                                                    (C.c_double * 9)(*H), H_pred_ptr, int(width), int(height),
                                                    (C.c_double * len(t))(*t), len(t), counts_ptr, corner_ptr,
                                                    handle.stream()))


def homography_errors(rows, H_gt, H_pred_buf, width, height, thresholds=range(1, 11), n_dev=None):
    """HPatches statistics of CUDA float64 rows [n, stride] (x1, y1, x2, y2 in columns 0..3) against H_gt, and the
    corner error of the model in `H_pred_buf` (a CUDA float64 find_model_into buffer: H at [0:9], int32 inlier count in
    element 9) on an image of width x height (include/p2p_b200.h, p2p_homography_errors) -> (counts int32 CUDA
    [len(thresholds) + 1]: rows with error <= t per threshold, then the rows considered; corner_err float64 CUDA [1]).
    `n_dev`: optional CUDA float64 scalar, use min(n, n_dev) rows.  No host sync."""
    if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype == torch.float64 and rows.dim() == 2):
        raise ValueError('rows must be a CUDA float64 tensor [n, stride]')
    if not (isinstance(H_pred_buf, torch.Tensor) and H_pred_buf.is_cuda and H_pred_buf.dtype == torch.float64
            and H_pred_buf.is_contiguous() and H_pred_buf.numel() >= 10 and H_pred_buf.device == rows.device):
        raise ValueError('H_pred_buf must be a contiguous CUDA float64 find_model buffer of at least 10 elements on '
                         'the device of rows')
    t = check_thresholds(thresholds)
    rows = rows.contiguous()
    n, stride = int(rows.shape[0]), int(rows.shape[1])
    counts = torch.empty(t.size + 1, dtype=torch.int32, device=rows.device)
    corner = torch.empty(1, dtype=torch.float64, device=rows.device)
    homography_errors_into(_lib.default_handle(rows.device), rows, stride, n,
                           None if n_dev is None else C.c_void_p(n_dev.data_ptr()), H_gt,
                           C.c_void_p(H_pred_buf.data_ptr()), width, height, t, C.c_void_p(counts.data_ptr()),
                           C.c_void_p(corner.data_ptr()))
    return counts, corner


def _record_into(h, rec, rows, row_stride, n, n_dev, seq, k, buf, thresholds):
    """The pair's statistics into its table row `rec`: p2p_homography_errors on the rows, then the count and the
    find_model buffer (`buf`: N followed by that buffer) copied device to device."""
    homography_errors_into(h, rows, row_stride, n, n_dev, seq.H_gt[k - 2], C.c_void_p(buf.data_ptr() + 8),
                           seq.size[0], seq.size[1], thresholds, C.c_void_p(rec.data_ptr() + _REC_COUNTS * 8),
                           C.c_void_p(rec.data_ptr() + _REC_CORNER * 8))
    rec[:_REC_CORNER].copy_(buf[:_REC_CORNER])


def parse_record(row, seq, k, n_thr, failed=False):
    """One pair's Namespace(seq, k, N, n_inliers, corner_err, counts, match_failed) from its host table row; counts is
    int32 [n_thr + 1] (correct rows per threshold, then N).  A failed pair has N 0, n_inliers 0, corner error inf."""
    if failed:
        return Namespace(seq=seq, k=k, N=0, n_inliers=0, corner_err=np.inf,
                         counts=np.zeros(n_thr + 1, dtype=np.int32), match_failed=True)
    return Namespace(seq=seq, k=k, N=int(row[0]), n_inliers=int(row[_REC_H + 9:_REC_H + 10].view(np.int32)[0]),
                     corner_err=float(row[_REC_CORNER]),
                     counts=row[_REC_COUNTS:].view(np.int32)[:n_thr + 1].copy(), match_failed=False)


def summarize(records, h_thresholds):
    """({'all', 'i', 'v'} -> mean per-pair MMA per threshold, {'all', 'i', 'v'} -> share of pairs with corner error
    <= t per h_threshold), numpy arrays; an empty split gives NaN."""
    n_thr = len(records[0].counts) - 1 if records else 0
    mma, h_acc = {}, {}
    for split in ('all', 'i', 'v'):
        sel = [r for r in records if split == 'all' or r.seq.startswith(split + '_')]
        if not sel:
            mma[split] = np.full(n_thr, np.nan)
            h_acc[split] = np.full(len(h_thresholds), np.nan)
            continue
        pm = [np.zeros(n_thr) if r.counts[-1] == 0 else r.counts[:-1].astype(np.float64) / r.counts[-1] for r in sel]
        mma[split] = np.mean(pm, axis=0)
        ce = np.array([r.corner_err for r in sel])
        h_acc[split] = np.array([np.mean(ce <= t) for t in h_thresholds])
    return mma, h_acc


def eval_hpatches(matcher, data_root, ksize=2, eval_type='fine', io_thres=0.25, ncn_thres=0.0, imsize=1024,
                  ransac_thres=2.0, thresholds=range(1, 11), h_thresholds=(1, 3, 5, 10), exclude=D2NET_EXCLUDED,
                  lprint_=print):
    """MMA and homography accuracy of `matcher` on the HPatches sequences under `data_root` (protocol in the module
    docstring), printing a header, an MMA line, a homography-accuracy line and a matches / inlier-ratio / time line
    through lprint_.

    `matcher` is a Patch2PixB200 (run as estimate_matches_from_files(..., ksize, ncn_thres, True, io_thres, eval_type,
    imsize, verify=('H', ransac_thres)) would run it), or any callable (im1_path, im2_path) returning [N, 4] rows as
    numpy or a torch tensor, or a tuple whose first element is those rows (the reference's estimate_matches).

    -> dict(mma={'all', 'i', 'v'} -> float64 [len(thresholds)], h_acc={'all', 'i', 'v'} -> float64
    [len(h_thresholds)], n_pairs, h_failed (pairs without a finite corner error), records: one Namespace per pair
    (seq, k, N, n_inliers, corner_err, counts, match_failed), thresholds, h_thresholds, time)."""
    thr = check_thresholds(thresholds)
    h_thr = check_thresholds(h_thresholds, 'h_thresholds')
    if not (ransac_thres > 0 and np.isfinite(ransac_thres)):
        raise ValueError('ransac_thres must be positive')
    seqs = read_hpatches(data_root, exclude)
    pairs = [(seq, k) for seq in seqs for k in range(2, 7)]
    run = PairRunner(matcher, ksize, eval_type, io_thres, ncn_thres, imsize)
    n_i = sum(s.split == 'i' for s in seqs)
    lprint_(f'\n>>Eval on HPatches: {len(seqs)} sequences ({n_i} i / {len(seqs) - n_i} v), {len(pairs)} pairs, '
            + (f'eval_type={eval_type} ksize={ksize} io={io_thres} nc={ncn_thres} im={imsize} ' if run.is_net else '')
            + f'rthres={ransac_thres}')
    start = time.time()
    table = torch.zeros(len(pairs), _rec_len(thr.size), dtype=torch.float64, device=run.dev)
    failed = {}
    x1 = None

    def load(pair):             # image 1 is decoded, and prepared, once per sequence
        seq, k = pair
        return run.decode(seq.paths[:1] + [seq.paths[k - 1]] if k == 2 else [seq.paths[k - 1]])
    for i, ims in prefetch(pairs, load):
        seq, k = pairs[i]
        if k == 2:
            x1 = None
        try:
            if isinstance(ims, Exception):
                raise ims
            if run.is_net:          # the packed rows, their device count and the RANSAC buffer, read in place
                if k == 2:
                    x1 = run.prepare(ims[0])
                if x1 is None:
                    raise RuntimeError(f'{seq.paths[0]} could not be loaded')
                rows, n = run.match(x1, run.prepare(ims[-1]), ('H', ransac_thres))
                stride, n_dev, buf = 9, C.c_void_p(rows.data_ptr() + n * 9 * 8), rows[n * 9:]
            else:
                rows = matcher(seq.paths[0], seq.paths[k - 1])
        except Exception as e:
            failed[i] = f'{type(e).__name__}: {e}'
            continue
        if not run.is_net:          # rows of the wrong shape raise rather than fail the pair
            rows = as_rows(rows, run.dev)
            n, stride, n_dev = int(rows.shape[0]), 4, None
            buf = torch.empty(1 + V.out_size(n), dtype=torch.float64, device=run.dev)
            buf[0].fill_(float(n))
            V.find_model_into(run.h, V.MODEL_H, rows, 4, n, None, ransac_thres, 0.999, 10000, 0, buf[1:])
        _record_into(run.h, table[i], rows, stride, n, n_dev, seq, k, buf, thr)
    host = table.cpu().numpy()                        # the run's one copy of the records
    runtime = time.time() - start
    records = [parse_record(host[i], seq.name, k, thr.size, i in failed) for i, (seq, k) in enumerate(pairs)]
    mma, h_acc = summarize(records, h_thr)
    h_failed = sum(1 for r in records if not np.isfinite(r.corner_err))

    def fmt(a):
        return '[' + ' '.join(f'{v:.3f}' for v in a) + ']'
    lprint_('MMA@{}px all={} i={} v={}'.format(list(thr.tolist()), fmt(mma['all']), fmt(mma['i']), fmt(mma['v'])))
    lprint_('Hacc@{}px all={} i={} v={} failed={} (matcher errors {})'.format(
        list(h_thr.tolist()), fmt(h_acc['all']), fmt(h_acc['i']), fmt(h_acc['v']), h_failed, len(failed)))
    matched = [r for r in records if r.N > 0]
    lprint_('Matches mean={:.1f} inlier_ratio={:.3f} time={:.2f}s'.format(
        np.mean([r.N for r in records]) if records else float('nan'),
        np.mean([max(r.n_inliers, 0) / r.N for r in matched]) if matched else float('nan'), runtime))
    return dict(mma=mma, h_acc=h_acc, n_pairs=len(pairs), h_failed=h_failed, records=records,
                thresholds=thr, h_thresholds=h_thr, time=runtime)


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description='MMA and homography accuracy of a Patch2Pix or NCNet checkpoint on the '
                                             'HPatches sequences (hpatches-sequences-release).')
    ap.add_argument('--ckpt', required=True, help='checkpoint file (eval_helper.load_checkpoint)')
    ap.add_argument('--data_root', required=True, help='directory of the HPatches sequences')
    ap.add_argument('--method', default='patch2pix', choices=('patch2pix', 'nc'),
                    help="'patch2pix': fine matches; 'nc': the coarse NCNet matches of the checkpoint")
    ap.add_argument('--ksize', type=int, default=2)
    ap.add_argument('--io_thres', type=float, default=0.25)
    ap.add_argument('--ncn_thres', type=float, default=0.9)
    ap.add_argument('--imsize', type=int, default=1024)
    ap.add_argument('--ransac_thres', type=float, default=2.0)
    ap.add_argument('--all', action='store_true', help="evaluate every sequence (exclude=()), not D2-Net's 108")
    args = ap.parse_args(argv)
    from .eval_helper import load_checkpoint
    net = load_checkpoint(args.ckpt, method=args.method)
    eval_hpatches(net, args.data_root, ksize=args.ksize, eval_type='coarse' if args.method == 'nc' else 'fine',
                  io_thres=args.io_thres, ncn_thres=args.ncn_thres, imsize=args.imsize,
                  ransac_thres=args.ransac_thres, exclude=() if args.all else D2NET_EXCLUDED)


if __name__ == '__main__':
    main()
