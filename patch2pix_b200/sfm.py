"""Aachen Day-Night localization: triangulate a detector-free matcher's database matches against the model's known
poses on the GPU, then localize each query from its matches to the triangulated keypoints (hloc's protocol, with
COLMAP's point_triangulator replaced by the kernels of csrc/sfm.cu).

    python -m patch2pix_b200.sfm --ckpt PATH --images DIR --model DIR --db_pairs FILE --query_pairs FILE \\
        --queries FILE [FILE ...] --results OUT [--sfm_out DIR] [--method patch2pix|nc]

Triangulation (triangulate_from_matches; every stage deterministic, ids from sorted keys):

1. Keypoints.  Each image's keypoints are the endpoints of its database-pair matches snapped to cells of merge_px
   pixels, cell (floor(x / merge_px), floor(y / merge_px)); a keypoint is the mean of its cell's endpoints, summed in
   pair order then match order; ids in order of (image, cell_y, cell_x).  Endpoints that are not finite, negative or
   in a cell index of 2^22 or more are dropped and counted.
2. Edges and tracks.  A match is an edge if it is the first match of its pair, in match order, for its keypoint in
   image A and also for its keypoint in image B, and its Sampson error in undistorted normalised coordinates under the
   model's E = [t]x R is at most (epi_px / f_mean)^2, f_mean the mean focal length of the two cameras.  Tracks are the
   connected components of the edges (labelled by their smallest keypoint id); one of more than 2^16 observations is
   rejected and counted.
3. Triangulation, per track, observations in keypoint-id order, in rounds (at most 8, each making at most one point):
   every pair i < j of different images among the first 32 remaining observations is a hypothesis, the linear
   two-view point of the normalised rays (least squares on the 4 DLT rows); it is valid iff both depths are positive
   and the triangulation angle is at least min_angle.  Its score is the number of distinct images with an inlier (depth
   > 0, reprojection error in original, distorted pixels <= reproj_px); the highest score wins, ties to the lowest
   (i, j).  Five Gauss-Newton steps (normalised-plane residuals) refine it over one inlier per image (the smallest
   error, ties to the lower observation); the refined point is kept if its score does not drop.  The point is accepted
   with inliers in at least 2 images whose largest pairwise triangulation angle is at least min_angle.  Its inliers,
   and the two hypothesis observations, are removed whether or not it is accepted.  Rounds stop when fewer than 2
   images remain or no hypothesis is valid.
4. Query rows (localize_from_matches).  A query's match endpoints are merged into query keypoints as in 1.  Each
   database endpoint takes the nearest keypoint of its image within merge_px, among the 3x3 cells around its own, that
   has a point (ties to the lower id).  Rows are the distinct (query keypoint, point) pairs in that order, the query
   keypoint undistorted to the pinhole with the same f, cx, cy; p2p_find_absolute_pose_batch localizes them at
   ransac_thres undistorted pixels (hloc's 12 px; pycolmap measures its threshold in distorted pixels).

The file layouts follow hloc's published Aachen pipeline: pair lists 'name0 name1' per line, queries with intrinsics
'name MODEL w h params...', the results file of localize.write_results.  They have not been checked against released
files.
"""
import ctypes as C
import math
import os
import struct
import time
from argparse import Namespace

import numpy as np
import torch

from . import _lib
from .evaluation import qvec2rotmat, read_cameras_binary, read_images_binary
from .eval_helper import PairRunner, as_rows, prefetch
from .localize import AbsPoseTable, read_retrieval

AACHEN_THRESHOLDS = ((0.25, 2), (0.5, 5), (5, 10))
CAMERA_CODES = {'SIMPLE_PINHOLE': 0, 'PINHOLE': 1, 'SIMPLE_RADIAL': 2, 'RADIAL': 3}
MAX_IMAGES = 1 << 20


# ---- cameras and poses --------------------------------------------------------------------------------------------------
def camera_record(model, params, name='camera'):
    """(model, fx, fy, cx, cy, k1, k2, 0) of a SIMPLE_PINHOLE / PINHOLE / SIMPLE_RADIAL / RADIAL camera."""
    p = [float(v) for v in params]
    n = {'SIMPLE_PINHOLE': 3, 'PINHOLE': 4, 'SIMPLE_RADIAL': 4, 'RADIAL': 5}.get(model)
    if n is None:
        raise ValueError(f'{name}: camera model {model} is not supported (SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, '
                         f'RADIAL)')
    if len(p) != n:
        raise ValueError(f'{name}: {model} takes {n} parameters, got {len(p)}')
    if model == 'PINHOLE':
        fx, fy, cx, cy = p
        k = (0.0, 0.0)
    else:
        fx = fy = p[0]
        cx, cy = p[1], p[2]
        k = (tuple(p[3:]) + (0.0, 0.0))[:2]
    rec = np.array([CAMERA_CODES[model], fx, fy, cx, cy, k[0], k[1], 0.0])
    if not (np.all(np.isfinite(rec)) and fx > 0 and fy > 0):
        raise ValueError(f'{name}: camera parameters must be finite with positive focal lengths')
    return rec


def image_record(qvec, tvec):
    """R row-major, t, centre -R^T t of a world -> camera pose."""
    R = qvec2rotmat(np.asarray(qvec, dtype=np.float64) / np.linalg.norm(qvec))
    t = np.asarray(tvec, dtype=np.float64).reshape(3)
    return np.concatenate([R.reshape(-1), t, -R.T @ t])


def pair_geometry(rec_a, rec_b, cam_a, cam_b, epi_px):
    """E (row-major, x_b^T E x_a = 0 in normalised coordinates) and the Sampson threshold (epi_px / f_mean)^2."""
    Ra, ta = rec_a[:9].reshape(3, 3), rec_a[9:12]
    Rb, tb = rec_b[:9].reshape(3, 3), rec_b[9:12]
    R = Rb @ Ra.T
    t = tb - R @ ta
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    f_mean = 0.5 * (0.5 * (cam_a[1] + cam_a[2]) + 0.5 * (cam_b[1] + cam_b[2]))
    return (tx @ R).reshape(-1), (epi_px / f_mean) ** 2


# ---- files ----------------------------------------------------------------------------------------------------------------
def read_pairs(path):
    """hloc's pair list ('name0 name1' per line; blank lines skipped) -> [(name0, name1)].  Raises ValueError naming the
    line on a line without exactly two fields."""
    out = []
    with open(path) as f:
        for ln, line in enumerate(f, 1):
            tok = line.split()
            if not tok:
                continue
            if len(tok) != 2:
                raise ValueError(f'{path}:{ln}: expected 2 fields (name0 name1), got {len(tok)}')
            out.append((tok[0], tok[1]))
    return out


def read_queries_with_intrinsics(path):
    """'name MODEL width height params...' per line -> {name: Namespace(model, width, height, params)} in file order.
    Raises ValueError naming the line on a malformed line or an unsupported model."""
    out = {}
    with open(path) as f:
        for ln, line in enumerate(f, 1):
            tok = line.split()
            if not tok:
                continue
            try:
                if len(tok) < 5:
                    raise ValueError(f'expected name MODEL width height params..., got {len(tok)} fields')
                q = Namespace(model=tok[1], width=int(tok[2]), height=int(tok[3]),
                              params=np.array([float(v) for v in tok[4:]]))
                camera_record(q.model, q.params, tok[0])
            except ValueError as e:
                raise ValueError(f'{path}:{ln}: {e}') from None
            out[tok[0]] = q
    return out


# ---- the model ------------------------------------------------------------------------------------------------------------
class SfmModel:
    """A triangulated model: the known cameras and images, keypoints (kp_xy [n, 2], kp_img [n] image index into
    `images`, kp_key [n] uint64 cell keys, kp_point [n] point index or -1) and points (points [m, 3], point_len [m],
    point_err [m] mean reprojection error in pixels), with the run's stats."""

    def __init__(self, cameras, images, merge_px, kp_xy, kp_key, kp_point, points, point_len, point_err, stats):
        self.cameras, self.images, self.merge_px = cameras, images, float(merge_px)
        self.kp_xy, self.kp_key, self.kp_point = kp_xy, kp_key, kp_point
        self.kp_img = (kp_key >> np.uint64(44)).astype(np.int64)
        self.points, self.point_len, self.point_err, self.stats = points, point_len, point_err, stats
        self.index = {im.name: i for i, im in enumerate(images)}
        self._dev = {}

    def device_arrays(self, dev):
        """(kp_key, kp_xy, kp_point, points) on `dev`, uploaded once."""
        if dev not in self._dev:
            n = max(len(self.kp_key), 1)
            key = torch.zeros(n, dtype=torch.int64)
            key[:len(self.kp_key)] = torch.from_numpy(self.kp_key.view(np.int64))
            xy = torch.zeros(n, 2, dtype=torch.float64)
            xy[:len(self.kp_xy)] = torch.from_numpy(self.kp_xy)
            kp = torch.full((n,), -1, dtype=torch.int32)
            kp[:len(self.kp_point)] = torch.from_numpy(self.kp_point.astype(np.int32))
            pts = torch.zeros(max(len(self.points), 1), 3, dtype=torch.float64)
            pts[:len(self.points)] = torch.from_numpy(self.points)
            self._dev[dev] = tuple(t.to(dev) for t in (key, xy, kp, pts))
        return self._dev[dev]

    def write(self, model_dir):
        """cameras.bin, images.bin (each image's keypoints in id order with their point3D ids, -1 without one) and
        points3D.bin (point id = index; error = mean reprojection error; track = (image id, point2D index))."""
        os.makedirs(model_dir, exist_ok=True)
        with open(os.path.join(model_dir, 'cameras.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(self.cameras)))
            for cam in self.cameras.values():
                code = {'SIMPLE_PINHOLE': 0, 'PINHOLE': 1, 'SIMPLE_RADIAL': 2, 'RADIAL': 3}[cam.model]
                f.write(struct.pack('<iiQQ', cam.id, code, cam.width, cam.height) +
                        struct.pack(f'<{len(cam.params)}d', *cam.params))
        first = np.searchsorted(self.kp_img, np.arange(len(self.images) + 1))
        track = [[] for _ in range(len(self.points))]
        with open(os.path.join(model_dir, 'images.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(self.images)))
            for i, im in enumerate(self.images):
                a, b = first[i], first[i + 1]
                pts = np.zeros(b - a, dtype=[('xy', '<f8', (2,)), ('id', '<i8')])
                pts['xy'] = self.kp_xy[a:b]
                pts['id'] = self.kp_point[a:b]
                for k in np.nonzero(self.kp_point[a:b] >= 0)[0]:
                    track[self.kp_point[a + k]].append((im.id, int(k)))
                f.write(struct.pack('<i7di', im.id, *im.qvec, *im.tvec, im.camera_id) + im.name.encode('utf-8') +
                        b'\x00' + struct.pack('<Q', b - a) + pts.tobytes())
        with open(os.path.join(model_dir, 'points3D.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(self.points)))
            for p in range(len(self.points)):
                f.write(struct.pack('<Q3d3Bd', p, *self.points[p], 128, 128, 128, float(self.point_err[p])) +
                        struct.pack('<Q', len(track[p])) + np.asarray(track[p], dtype='<i4').reshape(-1).tobytes())


def read_points3D_binary(path):
    """points3D.bin -> {point3D_id: Namespace(id, xyz, error, track [(image_id, point2D_idx)])}, in file order."""
    from .evaluation import _Reader
    r = _Reader(path)
    out = {}
    for _ in range(r.take('<Q')[0]):
        pid, x, y, z, _, _, _, err, n = r.take('<Q3d3BdQ')
        tr = r.take(f'<{2 * n}i') if n else ()
        out[pid] = Namespace(id=pid, xyz=np.array([x, y, z]), error=err,
                             track=list(zip(tr[0::2], tr[1::2])))
    return out


def load_sfm_model(model_dir, merge_px=4.0):
    """The SfmModel that SfmModel.write wrote to model_dir.  Keypoint cell keys are recomputed with merge_px."""
    cameras = read_cameras_binary(os.path.join(model_dir, 'cameras.bin'))
    images = list(read_images_binary(os.path.join(model_dir, 'images.bin'), points2D=True).values())
    pts3d = read_points3D_binary(os.path.join(model_dir, 'points3D.bin'))
    ids = sorted(pts3d)
    if ids != list(range(len(ids))):
        raise ValueError(f'{model_dir}: point3D ids must be 0 .. n-1')
    xy = np.concatenate([im.xys for im in images]) if images else np.zeros((0, 2))
    kp_point = np.concatenate([im.point3D_ids for im in images]) if images else np.zeros(0, np.int64)
    img = np.concatenate([np.full(len(im.xys), i, np.uint64) for i, im in enumerate(images)]) if images else \
        np.zeros(0, np.uint64)
    key = (img << np.uint64(44)) | (np.floor(xy[:, 1] / merge_px).astype(np.uint64) << np.uint64(22)) | \
        np.floor(xy[:, 0] / merge_px).astype(np.uint64)
    points = np.array([pts3d[i].xyz for i in ids]).reshape(-1, 3)
    plen = np.array([len(pts3d[i].track) for i in ids], dtype=np.int64)
    perr = np.array([pts3d[i].error for i in ids], dtype=np.float64)
    return SfmModel(cameras, images, merge_px, xy, key, kp_point.astype(np.int64), points, plen, perr,
                    _stats(len(xy), None, None, points, plen, perr))


def _stats(n_kp, n_edges, n_tracks, points, plen, perr, **extra):
    return dict(n_keypoints=int(n_kp), n_edges=n_edges, n_tracks=n_tracks, n_points=int(len(points)),
                mean_track_length=float(np.mean(plen)) if len(plen) else float('nan'),
                mean_reproj_error=float(np.mean(perr)) if len(perr) else float('nan'), **extra)


# ---- triangulation ----------------------------------------------------------------------------------------------------------
def _model_tables(model_dir):
    cameras = read_cameras_binary(os.path.join(model_dir, 'cameras.bin'))
    images = list(read_images_binary(os.path.join(model_dir, 'images.bin')).values())
    if len(images) >= MAX_IMAGES:
        raise ValueError(f'{model_dir}: at most {MAX_IMAGES - 1} images')
    cam_index = {cid: i for i, cid in enumerate(cameras)}
    cams = np.stack([camera_record(c.model, c.params, f'camera {c.id}') for c in cameras.values()]) if cameras else \
        np.zeros((0, 8))
    for im in images:
        if im.camera_id not in cam_index:
            raise ValueError(f'{model_dir}: image {im.name} has no camera {im.camera_id}')
    img_cam = np.array([cam_index[im.camera_id] for im in images], dtype=np.int32)
    recs = np.stack([image_record(im.qvec, im.tvec) for im in images]) if images else np.zeros((0, 15))
    return cameras, images, cams, img_cam, recs


def _pair_tables(images, cams, img_cam, recs, pairs, epi_px):
    index = {im.name: i for i, im in enumerate(images)}
    pair_img = np.zeros((max(len(pairs), 1), 2), dtype=np.int32)
    E = np.zeros((max(len(pairs), 1), 9))
    thr = np.zeros(max(len(pairs), 1))
    for p, (a, b) in enumerate(pairs):
        for nm in (a, b):
            if nm not in index:
                raise ValueError(f'pair {p} ({a} {b}): {nm} is not an image of the model')
        ia, ib = index[a], index[b]
        if ia == ib:
            raise ValueError(f'pair {p} ({a} {b}) matches an image with itself')
        pair_img[p] = ia, ib
        E[p], thr[p] = pair_geometry(recs[ia], recs[ib], cams[img_cam[ia]], cams[img_cam[ib]], epi_px)
    return pair_img, E, thr


def _check(pos_args):
    for name, v in pos_args:
        if not (v > 0 and math.isfinite(v)):
            raise ValueError(f'{name} must be positive and finite')


def _triangulate(dev, cameras, images, cams, img_cam, recs, pair_img, E, thr, m4, offsets, merge_px, reproj_px,
                 min_angle):
    """The device stages on a compact match block m4 [M, 4] with host offsets [P + 1] -> SfmModel."""
    h = _lib.default_handle(dev)
    lib, st = h.lib, h.stream()
    M, P = int(offsets[-1]), len(offsets) - 1
    cap = max(2 * M, 1)
    if M == 0:
        m4 = torch.zeros(1, 4, dtype=torch.float64, device=dev)
    host = np.concatenate([offsets.astype(np.int64).view(np.float64), pair_img.reshape(-1).view(np.float64)
                           if pair_img.size % 2 == 0 else np.empty(0), E.reshape(-1), thr,
                           cams.reshape(-1), recs.reshape(-1)])
    ex = torch.from_numpy(host).to(dev)
    o = 0
    off_d = ex[o:o + P + 1].view(torch.int64)
    o += P + 1
    pimg_d = ex[o:o + P].view(torch.int32)
    o += P
    E_d = ex[o:o + 9 * P]
    o += 9 * P
    thr_d = ex[o:o + P]
    o += P
    cams_d = ex[o:o + cams.size]
    o += cams.size
    recs_d = ex[o:o + recs.size]
    img_cam_d = torch.from_numpy(np.concatenate([img_cam, [0]]).astype(np.int32)).to(dev)
    kp_xy = torch.empty(cap, 2, dtype=torch.float64, device=dev)
    kp_key = torch.empty(cap, dtype=torch.int64, device=dev)
    kp_of_ep = torch.empty(cap, dtype=torch.int32, device=dev)
    cnt = torch.zeros(8, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.p2p_sfm_keypoints(h.h, _lib.ptr(m4), M, _lib.ptr(off_d), P, _lib.ptr(pimg_d), 1, float(merge_px),
                                         _lib.ptr(kp_xy), _lib.ptr(kp_key), _lib.ptr(kp_of_ep), _lib.ptr(cnt), st))
        kp_n = torch.empty_like(kp_xy)
        _lib.check(lib.p2p_sfm_undistort(h.h, _lib.ptr(kp_xy), _lib.ptr(kp_key), 2 * M, _lib.ptr(cnt),
                                         _lib.ptr(img_cam_d), _lib.ptr(cams_d), _lib.ptr(kp_n), st))
        c0 = cnt[:2].cpu().numpy()                     # the keypoint stage's sync
        n_kp, dropped = int(c0[0]), int(c0[1])
        nk = max(n_kp, 1)
        labels, obs_kp, tstart, tlen = (torch.empty(nk, dtype=torch.int32, device=dev) for _ in range(4))
        ct = np.zeros(6, dtype=np.int64)
        _lib.check(lib.p2p_sfm_tracks(h.h, _lib.ptr(kp_of_ep), M, _lib.ptr(off_d), P, _lib.ptr(E_d), _lib.ptr(thr_d),
                                      _lib.ptr(kp_n), n_kp, _lib.ptr(labels), _lib.ptr(obs_kp), _lib.ptr(tstart),
                                      _lib.ptr(tlen), _lib.ptr(cnt), ct.ctypes.data_as(C.POINTER(C.c_int64)), st))
        n_tracks = int(ct[1])
        slots = max(8 * n_tracks, 1)
        pts = torch.empty(slots, 3, dtype=torch.float64, device=dev)
        plen = torch.empty(slots, dtype=torch.int32, device=dev)
        perr = torch.empty(slots, dtype=torch.float64, device=dev)
        kp_point = torch.empty(nk, dtype=torch.int32, device=dev)
        _lib.check(lib.p2p_sfm_triangulate(h.h, _lib.ptr(obs_kp), _lib.ptr(tstart), _lib.ptr(tlen), n_tracks, n_kp,
                                           _lib.ptr(kp_xy), _lib.ptr(kp_n), _lib.ptr(kp_key), _lib.ptr(recs_d),
                                           _lib.ptr(img_cam_d), _lib.ptr(cams_d), float(reproj_px),
                                           math.cos(math.radians(min_angle)), _lib.ptr(pts), _lib.ptr(plen),
                                           _lib.ptr(perr), _lib.ptr(kp_point), _lib.ptr(cnt), st))
        n_pts = int(cnt[0].item())                      # the triangulation stage's sync
    points = pts[:n_pts].cpu().numpy()
    point_len = plen[:n_pts].cpu().numpy().astype(np.int64)
    point_err = perr[:n_pts].cpu().numpy()
    stats = _stats(n_kp, int(ct[0]), n_tracks, points, point_len, point_err, n_observations=int(ct[2]),
                   n_dropped_endpoints=dropped, n_rejected_components=int(ct[3]), n_matches=M)
    return SfmModel(cameras, images, merge_px, kp_xy[:n_kp].cpu().numpy(),
                    kp_key[:n_kp].cpu().numpy().view(np.uint64), kp_point[:n_kp].cpu().numpy().astype(np.int64),
                    points, point_len, point_err, stats)


def _geometry_args(merge_px, epi_px, reproj_px, min_angle):
    _check([('merge_px', merge_px), ('epi_px', epi_px), ('reproj_px', reproj_px)])
    if not (0 <= min_angle < 180):
        raise ValueError('min_angle must lie in [0, 180) degrees')


def triangulate_from_matches(model_dir, pairs, matches, merge_px=4.0, epi_px=4.0, reproj_px=4.0, min_angle=1.5,
                             device=None):
    """Triangulate the matches of database pairs against the poses of the COLMAP model in model_dir (the protocol in
    the module docstring).  pairs: [(name0, name1)] or a pair-list file; matches: one [N, 4] (x0, y0, x1, y1) numpy
    array or CUDA tensor per pair, in original-image pixels.  -> SfmModel."""
    _geometry_args(merge_px, epi_px, reproj_px, min_angle)
    pairs = read_pairs(pairs) if isinstance(pairs, (str, os.PathLike)) else list(pairs)
    if len(matches) != len(pairs):
        raise ValueError(f'{len(matches)} match arrays for {len(pairs)} pairs')
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    cameras, images, cams, img_cam, recs = _model_tables(model_dir)
    pair_img, E, thr = _pair_tables(images, cams, img_cam, recs, pairs, epi_px)
    rows = [as_rows(m, dev) for m in matches]
    offsets = np.zeros(max(len(rows), 1) + 1, dtype=np.int64)
    offsets[1:len(rows) + 1] = np.cumsum([int(r.shape[0]) for r in rows])
    offsets[len(rows) + 1:] = offsets[len(rows)]
    m4 = torch.cat(rows) if rows else torch.zeros(0, 4, dtype=torch.float64, device=dev)
    return _triangulate(dev, cameras, images, cams, img_cam, recs, pair_img, E, thr, m4, offsets, merge_px,
                        reproj_px, min_angle)


# ---- matching drivers -------------------------------------------------------------------------------------------------------
def _each(run, images_dir, pairs):
    """Yields (index, result or the exception raised) for the pairs (name0, name1) in order, decodes one pair ahead; a
    result is (rows [cap, 4] device tensor, the device kept-row count or None, cap)."""
    for i, ims in prefetch(pairs, lambda p: run.decode([os.path.join(images_dir, n) for n in p])):
        try:
            if isinstance(ims, Exception):
                raise ims
            if run.is_net:
                packed, n = run.match(run.prepare(ims[0]), run.prepare(ims[1]))
                r = packed[:9 * n].view(n, 9)[:, :4], packed[9 * n:9 * n + 1], n
            else:
                rows = run.call(*(os.path.join(images_dir, n) for n in pairs[i]))
                r = rows, None, int(rows.shape[0])
        except Exception as e:
            r = e
        yield i, r


def _collect(results, dev):
    """[(rows, n_dev, n) or None] -> compact device block [M, 4] and host offsets, with one host sync for the device
    counts."""
    caps = [r[2] if r is not None else 0 for r in results]
    devc = [r[1] for r in results if r is not None and r[1] is not None]
    counts = np.array(caps, dtype=np.int64)
    if devc:
        dv = torch.cat(devc).cpu().numpy()
        j = 0
        for i, r in enumerate(results):
            if r is not None and r[1] is not None:
                v = dv[j]
                j += 1
                counts[i] = int(v) if 0 <= v < caps[i] else caps[i]
    rows = [r[0][:counts[i]] for i, r in enumerate(results) if r is not None]
    offsets = np.zeros(max(len(results), 1) + 1, dtype=np.int64)
    offsets[1:len(results) + 1] = np.cumsum(counts)
    offsets[len(results) + 1:] = offsets[len(results)]
    m4 = torch.cat(rows).contiguous() if rows else torch.zeros(0, 4, dtype=torch.float64, device=dev)
    return m4.to(torch.float64), offsets


def _device_rows(r):
    """A pair result of _each as rows without a host sync: rows from the device count on are NaN, which every stage
    drops."""
    rows, n_dev, n = r
    if n_dev is None:
        return rows
    keep = torch.arange(n, device=rows.device, dtype=torch.float64) < n_dev
    return torch.where(keep[:, None], rows, torch.full_like(rows, float('nan')))


def triangulate_db(matcher, images_dir, model_dir, db_pairs, chunk_pairs=512, merge_px=4.0, epi_px=4.0,
                   reproj_px=4.0, min_angle=1.5, ksize=2, eval_type='fine', io_thres=0.25, imsize=1024,
                   lprint_=print):
    """Match the database pairs (a pair-list file or [(name0, name1)]) with `matcher`, a Patch2PixB200 or a callable
    (path0, path1) -> [N, 4], and triangulate them (triangulate_from_matches).  Match counts stay on the device until
    all pairs are matched; every chunk_pairs pairs the chunk's rows are gathered into one block.  A pair whose matcher
    raises is dropped and listed in the model's failed_pairs.  -> SfmModel."""
    _geometry_args(merge_px, epi_px, reproj_px, min_angle)
    if int(chunk_pairs) < 1:
        raise ValueError('chunk_pairs must be at least 1')
    pairs = read_pairs(db_pairs) if isinstance(db_pairs, (str, os.PathLike)) else list(db_pairs)
    cameras, images, cams, img_cam, recs = _model_tables(model_dir)
    pair_img, E, thr = _pair_tables(images, cams, img_cam, recs, pairs, epi_px)
    run = PairRunner(matcher, ksize, eval_type, io_thres, 0.0, imsize)
    lprint_(f'\n>>Triangulate: {len(images)} images, {len(pairs)} database pairs')
    start = time.time()
    results, failed, chunk = [], [], []

    def flush():
        if not chunk:
            return
        blocks = [r[0] for r in chunk if r is not None]
        block = torch.cat(blocks) if blocks else None
        o = 0
        for r in chunk:
            if r is None:
                results.append(None)
                continue
            results.append((block[o:o + r[2]], r[1], r[2]))
            o += r[2]
        chunk.clear()
    for i, r in _each(run, images_dir, pairs):
        if isinstance(r, Exception):
            failed.append((pairs[i], f'{type(r).__name__}: {r}'))
            r = None
        chunk.append(r)
        if len(chunk) == int(chunk_pairs):
            flush()
    flush()
    m4, offsets = _collect(results, run.dev)
    model = _triangulate(run.dev, cameras, images, cams, img_cam, recs, pair_img, E, thr, m4, offsets, merge_px,
                         reproj_px, min_angle)
    model.failed_pairs = failed
    lprint_(f'triangulated {model.stats["n_points"]} points from {model.stats["n_tracks"]} tracks, '
            f'{len(failed)} failed pairs, time={time.time() - start:.2f}s')
    return model


# ---- localization -----------------------------------------------------------------------------------------------------------
def _query_list(queries, query_pairs):
    qs = read_queries_with_intrinsics(queries) if isinstance(queries, (str, os.PathLike)) else dict(queries)
    ret = read_retrieval(query_pairs) if isinstance(query_pairs, (str, os.PathLike)) else list(query_pairs)
    for q, _ in ret:
        if q not in qs:
            raise ValueError(f'query {q} has no intrinsics')
    return qs, ret


def _localize(dev, sfm, qs, ret, per_query, results_path, ransac_thres, chunk_queries, conf, max_iters, failed):
    """per_query(i) -> ([(db index, rows [n, 4] device tensor)], or an exception).  Writes the results file."""
    h = _lib.default_handle(dev)
    lib, st = h.lib, h.stream()
    kp_key, kp_xy, kp_point, pts = sfm.device_arrays(dev)
    n_kp = len(sfm.kp_key)
    nq = len(ret)
    table = AbsPoseTable(nq, dev)
    for k0 in range(0, nq, int(chunk_queries)):
        K = min(int(chunk_queries), nq - k0)
        items, pimg, cams = [], [], []
        for k in range(K):
            q = ret[k0 + k][0]
            cam = camera_record(qs[q].model, qs[q].params, q)
            cams.append(cam)
            got = per_query(k0 + k)
            if isinstance(got, Exception):
                failed[k0 + k] = f'{type(got).__name__}: {got}'
                continue
            for d, rows in got:
                items.append(rows)
                pimg.append((k, d))
        offsets = np.zeros(max(len(items), 1) + 1, dtype=np.int64)
        offsets[1:len(items) + 1] = np.cumsum([int(r.shape[0]) for r in items])
        offsets[len(items) + 1:] = offsets[len(items)]
        M = int(offsets[-1])
        m4 = torch.cat(items).contiguous() if M else torch.zeros(1, 4, dtype=torch.float64, device=dev)
        cams = np.stack(cams)
        intr = cams[:, 1:5]
        pim = np.array(pimg if pimg else [(0, 0)], dtype=np.int32)
        ex = torch.from_numpy(np.concatenate([offsets.view(np.float64), cams.reshape(-1), intr.reshape(-1)])).to(dev)
        P = len(offsets) - 1
        off_d = ex[:P + 1].view(torch.int64)
        cams_d = ex[P + 1:P + 1 + 8 * K]
        intr_d = ex[P + 1 + 8 * K:]
        pim_d = torch.from_numpy(pim.reshape(-1)).to(dev)
        qcam_d = torch.arange(K, dtype=torch.int32, device=dev)
        cap = max(M, 1)
        q_xy = torch.empty(cap, 2, dtype=torch.float64, device=dev)
        q_key = torch.empty(cap, dtype=torch.int64, device=dev)
        q_of = torch.empty(cap, dtype=torch.int32, device=dev)
        q_n = torch.empty(cap, 2, dtype=torch.float64, device=dev)
        cnt = torch.zeros(2, dtype=torch.int64, device=dev)
        rows = torch.empty(cap, 5, dtype=torch.float64, device=dev)
        q_off = torch.empty(K + 1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.p2p_sfm_keypoints(h.h, _lib.ptr(m4), M, _lib.ptr(off_d), P, _lib.ptr(pim_d), 0,
                                             float(sfm.merge_px), _lib.ptr(q_xy), _lib.ptr(q_key), _lib.ptr(q_of),
                                             _lib.ptr(cnt), st))
            _lib.check(lib.p2p_sfm_undistort(h.h, _lib.ptr(q_xy), _lib.ptr(q_key), M, _lib.ptr(cnt), _lib.ptr(qcam_d),
                                             _lib.ptr(cams_d), _lib.ptr(q_n), st))
            _lib.check(lib.p2p_sfm_query_rows(h.h, _lib.ptr(m4), M, _lib.ptr(off_d), P, _lib.ptr(pim_d), K,
                                              float(sfm.merge_px), _lib.ptr(q_of), _lib.ptr(q_key), _lib.ptr(q_n),
                                              _lib.ptr(intr_d), _lib.ptr(kp_key), _lib.ptr(kp_xy), _lib.ptr(kp_point),
                                              n_kp, _lib.ptr(pts), _lib.ptr(rows), _lib.ptr(q_off), st))
        off_h = q_off.cpu().numpy()                     # the chunk's one sync: the row offsets RANSAC is planned by
        table.solve(k0, h, rows, q_off, off_h, None, intr_d.data_ptr(), ransac_thres, conf, max_iters)
    return table.finish([q for q, _ in ret], failed, results_path)


def _loc_args(ransac_thres, chunk_queries):
    _check([('ransac_thres', ransac_thres)])
    if int(chunk_queries) < 1:
        raise ValueError('chunk_queries must be at least 1')


def localize_from_matches(sfm, queries, query_pairs, matches, results_path, ransac_thres=12.0, chunk_queries=64,
                          conf=0.99999, max_iters=10000, device=None):
    """Localize queries from given matches (step 4 of the module docstring).  queries: a queries-with-intrinsics file or
    {name: Namespace(model, width, height, params)}; query_pairs: a retrieval list or [(query, [db, ...])]; matches:
    one [N, 4] (xq, yq, xdb, ydb) array or CUDA tensor per (query, db) pair, in retrieval order.  A query with no
    model is written with the identity pose and listed in `failed`.
    -> dict(poses={name: (R, t, n_inliers)}, failed, n_queries, time)."""
    _loc_args(ransac_thres, chunk_queries)
    qs, ret = _query_list(queries, query_pairs)
    flat = [(i, d) for i, (_, dbs) in enumerate(ret) for d in dbs]
    if len(matches) != len(flat):
        raise ValueError(f'{len(matches)} match arrays for {len(flat)} query pairs')
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    by_q = [[] for _ in ret]
    for (i, d), m in zip(flat, matches):
        if d not in sfm.index:
            raise ValueError(f'query pair ({ret[i][0]} {d}): {d} is not an image of the model')
        by_q[i].append((sfm.index[d], as_rows(m, dev)))
    start = time.time()
    failed = {}
    poses = _localize(dev, sfm, qs, ret, lambda i: by_q[i], results_path, ransac_thres, chunk_queries, conf,
                      max_iters, failed)
    return dict(poses=poses, failed=[(ret[i][0], failed[i]) for i in sorted(failed)], n_queries=len(ret),
                time=time.time() - start)


def localize_sfm(matcher, sfm, images_dir, queries, query_pairs, results_path, ransac_thres=12.0, chunk_queries=64,
                 conf=0.99999, max_iters=10000, ksize=2, eval_type='fine', io_thres=0.25, imsize=1024,
                 lprint_=print):
    """Match each query against its retrieved database images (the query as image 0) with `matcher` and localize it
    against `sfm` (localize_from_matches).  A query whose matcher raises on any of its pairs gets the identity pose and
    an entry in `failed`; the other queries are unaffected.  -> dict(poses, failed, n_queries, time)."""
    _loc_args(ransac_thres, chunk_queries)
    qs, ret = _query_list(queries, query_pairs)
    for q, dbs in ret:
        for d in dbs:
            if d not in sfm.index:
                raise ValueError(f'query pair ({q} {d}): {d} is not an image of the model')
    run = PairRunner(matcher, ksize, eval_type, io_thres, 0.0, imsize)
    lprint_(f'\n>>Localize: {len(ret)} queries, {sum(len(d) for _, d in ret)} pairs, rthres={ransac_thres}')
    start = time.time()
    flat = [(q, d) for q, dbs in ret for d in dbs]
    owner = [i for i, (_, dbs) in enumerate(ret) for _ in dbs]
    gen = _each(run, images_dir, flat)

    def per_query(i):
        got, err = [], None
        for _ in ret[i][1]:
            k, r = next(gen)
            if isinstance(r, Exception):
                err = err or r
            elif err is None:
                got.append((sfm.index[flat[k][1]], _device_rows(r)))
        return got if err is None else err
    failed = {}
    poses = _localize(run.dev, sfm, qs, ret, per_query, results_path, ransac_thres, chunk_queries, conf, max_iters,
                      failed)
    runtime = time.time() - start
    nq = len(ret)
    lprint_(f'localized {nq - len(failed)} / {nq} queries, time={runtime:.2f}s -> {results_path}')
    return dict(poses=poses, failed=[(ret[i][0], failed[i]) for i in sorted(failed)], n_queries=nq, time=runtime)


def localize_aachen(matcher, images_dir, model_dir, db_pairs, query_pairs, queries, results_path, sfm_out=None,
                    chunk_pairs=512, chunk_queries=64, merge_px=4.0, epi_px=4.0, reproj_px=4.0, min_angle=1.5,
                    ransac_thres=12.0, ksize=2, eval_type='fine', io_thres=0.25, imsize=1024, lprint_=print):
    """triangulate_db, then localize_sfm: hloc's Aachen pipeline on the GPU.  sfm_out: also write the triangulated
    model there.  -> dict(poses, failed, failed_pairs, n_queries, time, stats, sfm)."""
    start = time.time()
    sfm = triangulate_db(matcher, images_dir, model_dir, db_pairs, chunk_pairs, merge_px, epi_px, reproj_px,
                         min_angle, ksize, eval_type, io_thres, imsize, lprint_)
    if sfm_out:
        sfm.write(sfm_out)
    res = localize_sfm(matcher, sfm, images_dir, queries, query_pairs, results_path, ransac_thres, chunk_queries,
                       ksize=ksize, eval_type=eval_type, io_thres=io_thres, imsize=imsize, lprint_=lprint_)
    res.update(failed_pairs=sfm.failed_pairs, stats=sfm.stats, sfm=sfm, time=time.time() - start)
    return res


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description='Localize Aachen Day-Night queries with a Patch2Pix or NCNet checkpoint: '
                                             'triangulate the database matches against the model, then localize.')
    ap.add_argument('--ckpt', required=True, help='checkpoint file (eval_helper.load_checkpoint)')
    ap.add_argument('--images', required=True, help='image directory (names in the pair lists are relative to it)')
    ap.add_argument('--model', required=True, help='COLMAP model of the database: cameras.bin, images.bin')
    ap.add_argument('--db_pairs', required=True, help="database pairs, 'name0 name1' per line")
    ap.add_argument('--query_pairs', required=True, help="retrieval list, 'query db' per line")
    ap.add_argument('--queries', required=True, nargs='+', help="queries with intrinsics, 'name MODEL w h params...'")
    ap.add_argument('--results', required=True, help='output: name qw qx qy qz tx ty tz per query')
    ap.add_argument('--sfm_out', default=None, help='also write the triangulated model to this directory')
    ap.add_argument('--method', default='patch2pix', choices=('patch2pix', 'nc'),
                    help="'patch2pix': fine matches; 'nc': the coarse NCNet matches of the checkpoint")
    ap.add_argument('--ksize', type=int, default=2)
    ap.add_argument('--io_thres', type=float, default=0.25)
    ap.add_argument('--imsize', type=int, default=1024)
    ap.add_argument('--merge_px', type=float, default=4.0)
    ap.add_argument('--ransac_thres', type=float, default=12.0)
    ap.add_argument('--chunk_pairs', type=int, default=512)
    ap.add_argument('--chunk_queries', type=int, default=64)
    args = ap.parse_args(argv)
    if not os.path.isdir(args.images):
        ap.error(f'--images {args.images} is not a directory')
    if not os.path.isdir(args.model):
        ap.error(f'--model {args.model} is not a directory')
    for flag, path in (('--db_pairs', args.db_pairs), ('--query_pairs', args.query_pairs), ('--ckpt', args.ckpt)):
        if not os.path.isfile(path):
            ap.error(f'{flag} {path} is not a file')
    for path in args.queries:
        if not os.path.isfile(path):
            ap.error(f'--queries {path} is not a file')
    for flag, v in (('--merge_px', args.merge_px), ('--ransac_thres', args.ransac_thres)):
        if not (v > 0 and np.isfinite(v)):
            ap.error(f'{flag} must be positive')
    if args.chunk_pairs < 1 or args.chunk_queries < 1:
        ap.error('--chunk_pairs and --chunk_queries must be at least 1')
    queries = {}
    for path in args.queries:
        queries.update(read_queries_with_intrinsics(path))
    from .eval_helper import load_checkpoint
    net = load_checkpoint(args.ckpt, method=args.method)
    localize_aachen(net, args.images, args.model, args.db_pairs, args.query_pairs, queries, args.results,
                    sfm_out=args.sfm_out, chunk_pairs=args.chunk_pairs, chunk_queries=args.chunk_queries,
                    merge_px=args.merge_px, ransac_thres=args.ransac_thres, ksize=args.ksize,
                    eval_type='coarse' if args.method == 'nc' else 'fine', io_thres=args.io_thres,
                    imsize=args.imsize)


if __name__ == '__main__':
    main()
