"""Match verification on the GPU: RANSAC for a fundamental matrix (optionally with the DEGENSAC plane-degeneracy check)
or a homography, and the Sampson distance.

Drop-in for the reference's consumers of the match list -- ``pydegensac.findFundamentalMatrix(p1, p2, 1.0)`` and
``findHomography(p1, p2, 2.0)`` in examples/visualize_matches.ipynb, ``sampson_distance`` of utils/eval/measure.py:18-40
-- on top of ``p2p_find_model`` / ``p2p_sampson_distance`` (include/p2p_b200.h).

Numpy input gives numpy output through one device->host copy: a (3, 3) float64 model, or None when no model was found,
and a bool mask.  CUDA tensor input gives CUDA tensor output without a sync: the model is all zeros when no model was
found and NaN when a coordinate was not finite.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

MODEL_F, MODEL_H, MODEL_F_DEGENSAC = 0, 1, 2


def _rows(pts1, pts2):
    """[n, 4] float64 rows (x1, y1, x2, y2) on the device, and whether the input was numpy."""
    if isinstance(pts1, torch.Tensor) != isinstance(pts2, torch.Tensor):
        raise TypeError('pts1 and pts2 must both be numpy arrays or both be tensors')
    if isinstance(pts1, torch.Tensor):
        if pts1.device.type != 'cuda' or pts2.device != pts1.device:
            raise ValueError('tensor input must be on one CUDA device')
        if pts1.dim() != 2 or pts1.shape[1] != 2 or pts2.shape != pts1.shape:
            raise ValueError(f'pts1 and pts2 must both be [n, 2], got {tuple(pts1.shape)} and {tuple(pts2.shape)}')
        return torch.cat((pts1, pts2), 1).to(torch.float64).contiguous(), False
    p1 = np.asarray(pts1, dtype=np.float64).reshape(-1, 2)
    p2 = np.asarray(pts2, dtype=np.float64).reshape(-1, 2)
    if p1.shape != p2.shape:
        raise ValueError(f'pts1 and pts2 must have the same number of points, got {p1.shape[0]} and {p2.shape[0]}')
    dev = torch.device('cuda', torch.cuda.current_device())
    return torch.from_numpy(np.ascontiguousarray(np.concatenate((p1, p2), 1))).to(dev), True


def find_model_into(handle, model, rows, row_stride, n, n_dev, px_th, conf, max_iters, seed, out):
    """Enqueue p2p_find_model on `rows` (a float64 device tensor, row r at offset r * row_stride) writing into `out`, a
    float64 device tensor of at least 10 + ceil(n / 8) elements: model at [0:9], the int32 inlier count in element 9,
    the uint8 mask from byte 80 on.  `n_dev` is an optional pointer (ctypes) to a device double row count."""
    base = out.data_ptr()
    with torch.cuda.device(out.device):
        _lib.check(handle.lib.p2p_find_model(handle.h, model, C.c_void_p(rows.data_ptr()), row_stride, n, n_dev,
                                             float(px_th), float(conf), int(max_iters), int(seed) & (2 ** 64 - 1),
                                             C.c_void_p(base), C.c_void_p(base + 80),
                                             C.c_void_p(base + 72), handle.stream()))


def out_size(n):
    return 10 + (n + 7) // 8


def parse_host(host, n):
    """(model or None, bool mask) from the host copy of a find_model_into buffer; raises on non-finite input."""
    count = int(host[9:10].view(np.int32)[0])
    if count < 0:
        raise ValueError('find_model: a point coordinate is not finite')
    mask = host.view(np.uint8)[80:80 + n].astype(bool)
    return (host[:9].reshape(3, 3).copy() if count > 0 else None), mask


def _find(model, pts1, pts2, px_th, conf, max_iters, seed):
    rows, is_np = _rows(pts1, pts2)
    n = int(rows.shape[0])
    h = _lib.default_handle(rows.device)
    out = torch.empty(out_size(n), dtype=torch.float64, device=rows.device)
    find_model_into(h, model, rows, 4, n, None, px_th, conf, max_iters, seed, out)
    if is_np:
        return parse_host(out.cpu().numpy(), n)
    mask = out.view(torch.uint8)[80:80 + n].bool()
    return out[:9].view(3, 3), mask


def find_fundamental_matrix(pts1, pts2, px_th, conf=0.999, max_iters=10000, seed=0, degeneracy_check=False):
    """RANSAC fundamental matrix (x2^T F x1 = 0, unit Frobenius norm) from [n, 2] point lists -> (F, inlier mask).
    A row is an inlier iff its Sampson error (measure.py:36-39 without eps) is below px_th^2.

    degeneracy_check=True adds DEGENSAC's plane-degeneracy test (pydegensac.findFundamentalMatrix): when the samples
    that win a round have 5 of their 7 points on one plane, a plane-and-parallax round recovers the off-plane
    geometry that plain RANSAC loses on scenes dominated by one plane (include/p2p_b200.h, model 2)."""
    return _find(MODEL_F_DEGENSAC if degeneracy_check else MODEL_F, pts1, pts2, px_th, conf, max_iters, seed)


def find_homography(pts1, pts2, px_th, conf=0.999, max_iters=10000, seed=0):
    """RANSAC homography (x2 ~ H x1, H[2][2] = 1) from [n, 2] point lists -> (H, inlier mask).
    A row is an inlier iff its one-sided transfer error |pi(H x1) - x2| is below px_th."""
    return _find(MODEL_H, pts1, pts2, px_th, conf, max_iters, seed)


def sampson_distance(pts1, pts2, F):
    """utils/eval/measure.py:18-40 (eps = 1e-8) in fp64 on the GPU -> per-row distances (numpy or CUDA tensor)."""
    rows, is_np = _rows(pts1, pts2)
    n = int(rows.shape[0])
    Fd = torch.as_tensor(np.asarray(F, dtype=np.float64) if not isinstance(F, torch.Tensor) else F,
                         dtype=torch.float64).reshape(9).to(rows.device).contiguous()
    out = torch.empty(n, dtype=torch.float64, device=rows.device)
    h = _lib.default_handle(rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_sampson_distance(h.h, _lib.ptr(rows), 4, n, _lib.ptr(Fd), _lib.ptr(out), h.stream()))
    return out.cpu().numpy() if is_np else out


def epipolar_histograms_into(handle, rows, row_stride, n, n_dev, coarse_col, F, mask_ptr, edges, counts_ptr):
    """Enqueue p2p_epipolar_histograms on `rows` (a float64 device tensor, row r at offset r * row_stride) with F and
    the edges from the host; `n_dev`, `mask_ptr` and `counts_ptr` are device addresses (ctypes, None for the first
    two) of the row count, the uint8 mask and the int32 [3][len(edges)] output."""
    F = np.asarray(F, dtype=np.float64).reshape(9)
    edges = np.asarray(edges, dtype=np.float64).reshape(-1)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_epipolar_histograms(handle.h, C.c_void_p(rows.data_ptr()), row_stride, n, n_dev,
                                                      int(coarse_col), (C.c_double * 9)(*F), mask_ptr,
                                                      (C.c_double * len(edges))(*edges), len(edges), counts_ptr,
                                                      handle.stream()))


def epipolar_histograms(rows, F, edges, coarse_col=-1, mask=None, n_dev=None):
    """Sampson-distance histograms of CUDA float64 rows [n, stride] against F (include/p2p_b200.h,
    p2p_epipolar_histograms) -> int32 CUDA tensor [3, len(edges)]: coarse (columns coarse_col..+3, zeros with -1),
    refined (columns 0..3), refined under `mask` (CUDA bool/uint8 [n], or None); each ends with its row count.
    `n_dev`: optional CUDA float64 scalar, use min(n, n_dev) rows.  No host sync."""
    if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype == torch.float64 and rows.dim() == 2):
        raise ValueError('rows must be a CUDA float64 tensor [n, stride]')
    rows = rows.contiguous()
    n, stride = int(rows.shape[0]), int(rows.shape[1])
    counts = torch.empty(3, len(edges), dtype=torch.int32, device=rows.device)
    md = None
    if mask is not None:
        md = (mask.reshape(-1) != 0).to(torch.uint8).contiguous()
        if md.shape[0] != n:
            raise ValueError(f'mask has {md.shape[0]} entries for {n} rows')
    epipolar_histograms_into(_lib.default_handle(rows.device), rows, stride, n,
                             None if n_dev is None else C.c_void_p(n_dev.data_ptr()), coarse_col, F,
                             None if md is None else C.c_void_p(md.data_ptr()), edges, C.c_void_p(counts.data_ptr()))
    return counts


def first_hypotheses(model, pts1, pts2, px_th, count, seed=0):
    """Test hook: the first `count` hypotheses of find_model without selection -> (models [count*slots, 9] float64,
    counts [count*slots] int32, -1 where a slot holds no model); slots = 3 for F, 1 for H."""
    rows, _ = _rows(pts1, pts2)
    slots = 3 if model == MODEL_F else 1
    models = torch.empty(count * slots, 9, dtype=torch.float64, device=rows.device)
    counts = torch.empty(count * slots, dtype=torch.int32, device=rows.device)
    h = _lib.default_handle(rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_test_hypotheses(h.h, model, _lib.ptr(rows), 4, int(rows.shape[0]), float(px_th),
                                             int(seed) & (2 ** 64 - 1), count, _lib.ptr(models), _lib.ptr(counts),
                                             h.stream()))
    return models.cpu().numpy(), counts.cpu().numpy()


def first_degeneracy(pts1, pts2, px_th, count, seed=0):
    """Test hook: DEGENSAC's degeneracy test on every root of the first `count` F hypotheses -> (triplet [count*3]
    int32: -2 no model, -1 not degenerate, else the first degenerate triplet; H [count*3, 9] float64 in pixels)."""
    rows, _ = _rows(pts1, pts2)
    tri = torch.empty(count * 3, dtype=torch.int32, device=rows.device)
    H = torch.empty(count * 3, 9, dtype=torch.float64, device=rows.device)
    h = _lib.default_handle(rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_test_degeneracy(h.h, _lib.ptr(rows), 4, int(rows.shape[0]), float(px_th),
                                             int(seed) & (2 ** 64 - 1), count, _lib.ptr(tri), _lib.ptr(H), h.stream()))
    return tri.cpu().numpy(), H.cpu().numpy()
