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


# ---- many pairs per call (p2p_find_model_batch) ----------------------------------------------------------------------
def _as_list(x, name):
    if isinstance(x, (np.ndarray, torch.Tensor)) or not hasattr(x, '__len__'):
        raise TypeError(f'{name} must be a list of per-pair arrays')
    return list(x)


def pair_lists(pts1_list, pts2_list):
    """Validate a batch of point-list pairs before any device work -> (per-pair [n, 4] rows (numpy float64 arrays, or
    CUDA tensors of the caller's dtype), offsets int64 [K+1] on the host, whether the input was numpy)."""
    pts1_list, pts2_list = _as_list(pts1_list, 'pts1_list'), _as_list(pts2_list, 'pts2_list')
    if len(pts1_list) != len(pts2_list):
        raise ValueError(f'pts1_list and pts2_list must have the same length, got {len(pts1_list)} and '
                         f'{len(pts2_list)}')
    kinds = {isinstance(p, torch.Tensor) for p in pts1_list + pts2_list}
    if len(kinds) > 1:
        raise TypeError('the point lists must all be numpy arrays or all be tensors')
    is_np = not kinds or kinds == {False}
    rows = []
    for k, (p1, p2) in enumerate(zip(pts1_list, pts2_list)):
        if is_np:
            a = np.asarray(p1, dtype=np.float64).reshape(-1, 2)
            b = np.asarray(p2, dtype=np.float64).reshape(-1, 2)
            if a.shape != b.shape:
                raise ValueError(f'pair {k}: pts1 and pts2 must have the same number of points, got {a.shape[0]} and '
                                 f'{b.shape[0]}')
            rows.append(np.concatenate((a, b), 1))
        else:
            if p1.device.type != 'cuda' or p2.device != p1.device or p1.device != pts1_list[0].device:
                raise ValueError('tensor input must be on one CUDA device')
            if p1.dim() != 2 or p1.shape[1] != 2 or p2.shape != p1.shape:
                raise ValueError(f'pair {k}: pts1 and pts2 must both be [n, 2], got {tuple(p1.shape)} and '
                                 f'{tuple(p2.shape)}')
            rows.append((p1, p2))
    offsets = np.zeros(len(rows) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([r.shape[0] if is_np else r[0].shape[0] for r in rows])
    if np.any(np.diff(offsets) > 1 << 26) or offsets[-1] >= 1 << 31:
        raise ValueError('a pair has more than 2^26 rows or the batch has 2^31 rows or more')
    return rows, offsets, is_np


def upload(rows, offsets, is_np, extra=None, device=None):
    """(rows [N, 4] float64, offsets int64 [K+1], extra float64 [...] or None) on the device.  Numpy input crosses PCIe
    in one copy; tensor input is concatenated on its device (the offsets and `extra`, host arrays, are copied)."""
    extra = None if extra is None else np.ascontiguousarray(extra, dtype=np.float64).reshape(-1)
    n_ex = 0 if extra is None else extra.size
    N, K1 = int(offsets[-1]), offsets.size
    if is_np:
        dev = device or torch.device('cuda', torch.cuda.current_device())
        host = np.empty(4 * N + K1 + n_ex, dtype=np.float64)
        if N:
            host[:4 * N] = np.concatenate(rows, 0).reshape(-1)
        host[4 * N:4 * N + K1] = offsets.view(np.float64)
        if n_ex:
            host[4 * N + K1:] = extra
        d = torch.from_numpy(host).to(dev)
        return (d[:4 * N].view(N, 4), d[4 * N:4 * N + K1].view(torch.int64),
                None if extra is None else d[4 * N + K1:])
    dev = rows[0][0].device
    r = torch.cat([torch.cat(p, 1).to(torch.float64) for p in rows]).contiguous()
    tail = np.concatenate((offsets.view(np.float64), extra if n_ex else np.empty(0)))
    d = torch.from_numpy(tail).to(dev)
    return r, d[:K1].view(torch.int64), None if extra is None else d[K1:]


def find_model_batch_into(handle, model, rows, row_stride, offsets, offsets_host, n_dev, px_th, conf, max_iters, seed,
                          models_ptr, mask_ptr, counts_ptr):
    """Enqueue p2p_find_model_batch: `rows` a float64 device tensor, `offsets` an int64 device tensor [K+1] and
    `offsets_host` the same values in numpy; the outputs are device addresses (models [K][9] float64, row-aligned uint8
    mask, int32 counts [K]); `n_dev` an optional device address of K doubles."""
    oh = np.ascontiguousarray(offsets_host, dtype=np.int64)
    with torch.cuda.device(rows.device):
        _lib.check(handle.lib.p2p_find_model_batch(
            handle.h, model, C.c_void_p(rows.data_ptr()), row_stride, C.c_void_p(offsets.data_ptr()),
            oh.ctypes.data_as(C.POINTER(C.c_int64)), oh.size - 1, n_dev, float(px_th), float(conf), int(max_iters),
            int(seed) & (2 ** 64 - 1), C.c_void_p(models_ptr), C.c_void_p(mask_ptr), C.c_void_p(counts_ptr),
            handle.stream()))


def batch_out_size(K, N):
    """float64 elements of a batch buffer: models [0:9K], int32 counts from element 9K, the uint8 mask after them."""
    return 9 * K + (K + 1) // 2 + (N + 7) // 8


def parse_batch_host(host, offsets, what='find_model'):
    """[(model or None, bool mask)] from the host copy of a batch buffer; raises on a pair with non-finite input."""
    K = offsets.size - 1
    counts = host[9 * K:9 * K + (K + 1) // 2].view(np.int32)[:K]
    masks = host[9 * K + (K + 1) // 2:].view(np.uint8)
    out = []
    for k in range(K):
        if counts[k] < 0:
            raise ValueError(f'{what}: a point coordinate is not finite (pair {k})')
        out.append((host[9 * k:9 * k + 9].reshape(3, 3).copy() if counts[k] > 0 else None,
                    masks[offsets[k]:offsets[k + 1]].astype(bool)))
    return out


def _find_batch(model, pts1_list, pts2_list, px_th, conf, max_iters, seed):
    rows, offsets, is_np = pair_lists(pts1_list, pts2_list)
    K, N = offsets.size - 1, int(offsets[-1])
    if K == 0:
        return []
    rows, offs, _ = upload(rows, offsets, is_np)
    out = torch.empty(batch_out_size(K, N), dtype=torch.float64, device=rows.device)
    base = out.data_ptr()
    find_model_batch_into(_lib.default_handle(rows.device), model, rows, 4, offs, offsets, None, px_th, conf, max_iters,
                          seed, base, base + 8 * (9 * K + (K + 1) // 2), base + 72 * K)
    if is_np:
        return parse_batch_host(out.cpu().numpy(), offsets)
    mask = out[9 * K + (K + 1) // 2:].view(torch.uint8)
    return [(out[9 * k:9 * k + 9].view(3, 3), mask[offsets[k]:offsets[k + 1]].bool()) for k in range(K)]


def find_fundamental_matrices(pts1_list, pts2_list, px_th, conf=0.999, max_iters=10000, seed=0, degeneracy_check=False):
    """find_fundamental_matrix over a list of pairs in one batched call -> [(F, inlier mask)], element k equal to
    find_fundamental_matrix(pts1_list[k], pts2_list[k], ...).  Numpy input crosses PCIe once each way and raises
    ValueError when a pair has a non-finite coordinate; CUDA tensor input gives CUDA tensor views without a sync."""
    return _find_batch(MODEL_F_DEGENSAC if degeneracy_check else MODEL_F, pts1_list, pts2_list, px_th, conf, max_iters,
                       seed)


def find_homographies(pts1_list, pts2_list, px_th, conf=0.999, max_iters=10000, seed=0):
    """find_homography over a list of pairs in one batched call -> [(H, inlier mask)] (as find_fundamental_matrices)."""
    return _find_batch(MODEL_H, pts1_list, pts2_list, px_th, conf, max_iters, seed)


def batch_chunk_pairs(entry, device=None):
    """Pairs per launch of a batched entry point (0 find_model, 1 find_essential, 2 recover_pose)."""
    h = _lib.default_handle(device or torch.device('cuda', torch.cuda.current_device()))
    v = C.c_int()
    _lib.check(h.lib.p2p_batch_chunk_pairs(h.h, int(entry), C.byref(v)))
    return v.value
