"""The reference's image-matching validation (utils/train/eval_epoch_immatch.py:12-98) with the per-pair statistics on
the device, and the pieces it needs: a reader for COLMAP's binary models (utils/colmap/data_loading.py:72-107) and the
histogram summaries of utils/eval/measure.py:115-161.

`eval_immatch_val_sets(net, data_root, ...)` prints the reference's lines and returns what it returns.  Per pair, the
matcher, the E-RANSAC and pose recovery of ``estimate_matches(verify=('E', ...))`` and the three Sampson-distance
histograms (``p2p_epipolar_histograms``) are enqueued on the device; the pair's record (match count, E-RANSAC count,
R|t, histograms) is copied, device to device, into a table that comes back in one copy at the end of the run.  The only
other device->host copy per pair is the mutual-match count the matcher itself reads.  The two image decodes of the next
pair run on a worker thread while the current pair is enqueued.

The pair lists that loop reads (dense/sparse/ov_pairs.npy) come from `precompute_immatch_val_ovs` /
`sav_model_multi_ov_pairs` (utils/colmap/data_loading.py:7-70): the image-overlap matrix is an integer Gram matrix of
per-image keypoint bitsets (``p2p_overlap_scores``), and the pairs of every threshold come out of one torch.nonzero.
"""
import ctypes as C
import os
import struct
import time
from argparse import Namespace

import numpy as np
import torch

from . import _lib
from . import pose as P
from .eval_helper import PairRunner, prefetch
from .verify import epipolar_histograms_into

EVAL_BINS = [0, 1e-2, 1, 5, 10, 25, 50, 100, 2500, 1e5]      # eval_epoch_immatch.py:85


# ---- COLMAP binary models (little-endian; https://colmap.github.io/format.html) --------------------------------------
CAMERA_MODELS = {0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5),
                 4: ('OPENCV', 8), 5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5),
                 8: ('SIMPLE_RADIAL_FISHEYE', 4), 9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12)}


class _Reader:
    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.buf = f.read()
        self.pos = 0

    def take(self, fmt):
        size = struct.calcsize(fmt)
        if self.pos + size > len(self.buf):
            raise ValueError(f'{self.path}: truncated at byte {self.pos}')
        vals = struct.unpack_from(fmt, self.buf, self.pos)
        self.pos += size
        return vals

    def skip(self, size):
        if self.pos + size > len(self.buf):
            raise ValueError(f'{self.path}: truncated at byte {self.pos}')
        self.pos += size

    def cstring(self):
        end = self.buf.find(b'\x00', self.pos)
        if end < 0:
            raise ValueError(f'{self.path}: truncated in a name at byte {self.pos}')
        s = self.buf[self.pos:end].decode('utf-8')
        self.pos = end + 1
        return s


def read_cameras_binary(path):
    """cameras.bin -> {camera_id: Namespace(id, model, width, height, params)}, in file order."""
    r = _Reader(path)
    cameras = {}
    for _ in range(r.take('<Q')[0]):
        cid, model_id, width, height = r.take('<iiQQ')
        if model_id not in CAMERA_MODELS:
            raise ValueError(f'{path}: unknown camera model id {model_id}')
        model, n_params = CAMERA_MODELS[model_id]
        params = np.array(r.take(f'<{n_params}d'))
        cameras[cid] = Namespace(id=cid, model=model, width=width, height=height, params=params)
    return cameras


_POINT2D = np.dtype([('xy', '<f8', (2,)), ('id', '<i8')])     # one 2D point of images.bin: x, y, point3D_id


def _read_images(path, points2D, copy):
    r = _Reader(path)
    images = {}
    for _ in range(r.take('<Q')[0]):
        props = r.take('<i7di')
        name = r.cstring()
        n2d = r.take('<Q')[0]
        start = r.pos
        r.skip(24 * n2d)
        im = Namespace(id=props[0], qvec=np.array(props[1:5]), tvec=np.array(props[5:8]), camera_id=props[8], name=name)
        if points2D:
            pts = np.frombuffer(r.buf, _POINT2D, n2d, start)
            im.xys = pts['xy'].copy() if copy else pts['xy']
            im.point3D_ids = pts['id'].copy() if copy else pts['id']
        images[props[0]] = im
    return images


def read_images_binary(path, points2D=False):
    """images.bin -> {image_id: Namespace(id, qvec, tvec, camera_id, name)}, in file order.  With points2D each image
    also carries xys (float64 [n, 2]) and point3D_ids (int64 [n], -1 where the keypoint has no 3D point); otherwise
    the 2D points are skipped."""
    return _read_images(path, points2D, copy=True)


def cam_params_to_matrix(params, model):
    """3x3 K of a camera (data_loading.py:85-98); the distortion terms of the radial models are dropped."""
    if model == 'SIMPLE_PINHOLE':
        f, cx, cy = params
        fx = fy = f
    elif model == 'PINHOLE':
        fx, fy, cx, cy = params
    elif model == 'SIMPLE_RADIAL':
        f, cx, cy, _ = params
        fx = fy = f
    elif model == 'RADIAL':
        f, cx, cy, _, _ = params
        fx = fy = f
    else:
        raise ValueError(f'camera model {model} is not supported (SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL)')
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])


def qvec2rotmat(qvec):
    """COLMAP's rotation of a quaternion (w, x, y, z), without normalising it."""
    w, x, y, z = qvec
    return np.array([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def load_model_ims(model_dir):
    """{image name: Namespace(name, K, c, q, R, id)} of a COLMAP model (data_loading.py:72-83, 100-107): c = -R^T t
    with COLMAP's unnormalised rotation R of q.  Images whose camera is absent are skipped."""
    cameras = read_cameras_binary(os.path.join(model_dir, 'cameras.bin'))
    images = read_images_binary(os.path.join(model_dir, 'images.bin'))
    ims = {}
    for im in images.values():
        cam = cameras.get(im.camera_id)
        if cam is None:
            continue
        R = qvec2rotmat(im.qvec)
        ims[im.name] = Namespace(name=im.name, K=cam_params_to_matrix(cam.params, cam.model), c=-R.T.dot(im.tvec),
                                 q=im.qvec, R=R, id=im.id)
    return ims


# ---- histogram summaries (measure.py:115-161) -------------------------------------------------------------------------
def inliers_distr_from_counts(counts, bins=EVAL_BINS, tag='', return_ratios=False):
    """check_inliers_distr from per-sample counts: one row per sample of len(bins) integers, the np.histogram(d, bins)
    counts followed by len(d).  Same string, ratios and early returns."""
    if len(counts) == 0:
        return (None, '') if return_ratios else ''
    inlier_ratios = []
    Npts = []
    for row in counts:
        N = int(row[-1])
        if N == 0:
            continue
        Npts.append(N)
        inlier_ratios.append(np.asarray(row[:-1], dtype=np.int64) / N)
    ratio_print = '{} Sample:{} N(mean/max/min):{:.0f}/{:.0f}/{:.0f}\nRatios(%):'.format(
        tag, len(counts), np.mean(Npts), np.max(Npts), np.min(Npts))
    ratios = []
    for val, low, high in zip(np.mean(inlier_ratios, axis=0), bins[0:-1], bins[1::]):
        ratio_print = '{} [{},{})={:.2f}'.format(ratio_print, low, high, 100 * val)
        ratios.append(100 * val)
    if return_ratios:
        return ratios, ratio_print
    return ratio_print


def check_inliers_distr(inlier_dists, bins=[0, 1e-2, 1, 5, 10, 25, 50, 100, 400, 2500, 1e5], tag='',
                        return_ratios=False):
    """measure.py:115-141: mean per-sample share (%) of the distances in each bin, with the sample sizes."""
    if not inlier_dists:
        return (None, '') if return_ratios else ''
    counts = [np.append(np.histogram(d, bins)[0], len(d)) for d in inlier_dists]
    return inliers_distr_from_counts(counts, bins, tag, return_ratios)


def check_data_hist(data_list, bins, tag='', return_hist=False):
    """measure.py:143-161: mean of the per-sample means and mean per-sample share (%) of the values in each bin."""
    if not data_list:
        return ''
    hists = []
    means = []
    for data in data_list:
        if len(data) == 0:
            continue
        hists.append(np.histogram(data, bins)[0] / len(data))
        means.append(np.mean(data))
    hist_print = f'{tag} mean={np.mean(means):.2f}'
    mean_hists = np.mean(hists, axis=0)
    for val, low, high in zip(mean_hists, bins[0:-1], bins[1::]):
        hist_print += ' [{},{})={:.2f}'.format(low, high, 100 * val)
    if return_hist:
        return mean_hists, hist_print
    return hist_print


# ---- the validation loop ----------------------------------------------------------------------------------------------
def select_pairs(data_root, sample_max=300, min_overlap=0.3):
    """[(scene, ims, pair names)] in os.listdir order: the pairs of dense/sparse/ov_pairs.npy[min_overlap], shuffled
    by np.random and cut to sample_max only when there are more (eval_epoch_immatch.py:19-37).  The caller seeds
    np.random."""
    out = []
    for scene in os.listdir(data_root):
        model_dir = os.path.join(data_root, scene, 'dense/sparse')
        ims = load_model_ims(model_dir)
        pair_names = np.load(os.path.join(model_dir, 'ov_pairs.npy'), allow_pickle=True).item()[min_overlap]
        if len(pair_names) > sample_max:
            np.random.shuffle(pair_names)
            pair_names = pair_names[0:sample_max]
        out.append((scene, ims, pair_names))
    return out


# A record is one float64 row of the device table: the kept-match count N, then the pose buffer of
# estimate_matches(verify=('E', ...)) up to the pose count (E [9], E-RANSAC count (int32), R [9], t [3], pose count),
# then the int32 counts [3][len(bins)] of p2p_epipolar_histograms.
_REC_POSE = 1 + 23


def _rec_len(n_edges):
    return _REC_POSE + (3 * n_edges + 1) // 2


def eval_pairs(net, pairs, ksize=2, eval_type='fine', io_thres=0.5, ncn_thres=0.0, imsize=1024, rthres=0.5,
               bins=EVAL_BINS):
    """The per-pair work of eval_epoch_immatch.py:39-80 on an explicit pair list [(im1_path, im2_path, im1, im2)], im1
    and im2 the load_model_ims records -> one Namespace per pair: status ('ok', 'match_failed', 'geo_failed'), N,
    n_inls, R, t, counts (int32 [3, len(bins)]: cdist, fdist, indist histograms, each ending with its sample size),
    terr, qerr (degrees; None where the reference has none)."""
    run = PairRunner(net, ksize, eval_type, io_thres, ncn_thres, imsize)
    n_edges = len(bins)
    table = torch.zeros(len(pairs), _rec_len(n_edges), dtype=torch.float64, device=run.dev)
    gts, failed = [], set()
    for i, ims in prefetch(pairs, lambda p: run.decode(p[:2])):
        _, _, im1, im2 = pairs[i]
        t_gt, q_gt = P.abs2relapose(im1.c, im2.c, im1.q, im2.q)
        F = P.pose2fund(im1.K, im2.K, P.quat2mat(q_gt), t_gt)
        gts.append((t_gt, q_gt))
        try:
            if isinstance(ims, Exception):
                raise ims
            packed, n = run.match(run.prepare(ims[0]), run.prepare(ims[1]), ('E', rthres, im1.K, im2.K))
        except Exception:
            failed.add(i)
            continue
        rec = table[i]
        epipolar_histograms_into(run.h, packed, 9, n, C.c_void_p(packed.data_ptr() + n * 9 * 8), 5, F,
                                 C.c_void_p(packed.data_ptr() + (n * 9 + 1) * 8 + 184), bins,
                                 C.c_void_p(rec.data_ptr() + _REC_POSE * 8))
        rec[:_REC_POSE].copy_(packed[n * 9:n * 9 + _REC_POSE])
    host = table.cpu().numpy()                        # the run's one copy of the records
    return [parse_record(None if i in failed else host[i], t_gt, q_gt, n_edges) for i, (t_gt, q_gt) in enumerate(gts)]


def parse_record(row, t_gt, q_gt, n_edges=len(EVAL_BINS)):
    """One pair's Namespace (see eval_pairs) from its host table row (None: the pair failed to load or match) and its
    ground-truth relative pose.  The pair is geo_failed when the E-RANSAC count is 0 (fewer than 5 matches or no model)
    or -1 (a coordinate is not finite); as in the reference it keeps its cdist and fdist histograms."""
    if row is None:
        return Namespace(status='match_failed', N=None, n_inls=None, R=None, t=None, counts=None, terr=None, qerr=None)
    N = int(row[0])
    count = int(row[10:11].view(np.int32)[0])
    counts = row[_REC_POSE:].view(np.int32)[:3 * n_edges].reshape(3, n_edges).copy()
    if count <= 0:
        return Namespace(status='geo_failed', N=N, n_inls=None, R=None, t=None, counts=counts, terr=None, qerr=None)
    R, t = row[11:20].reshape(3, 3).copy(), row[20:23].reshape(3, 1).copy()
    return Namespace(status='ok', N=N, n_inls=int(counts[2, -1]), R=R, t=t, counts=counts,
                     terr=float(P.cal_vec_angle_error(t.squeeze(), t_gt)),
                     qerr=float(P.cal_quat_angle_error(P.mat2quat(R), q_gt)))


def summarize(records, runtime, bins=EVAL_BINS):
    """The reference's closing lines (eval_epoch_immatch.py:81-98) from eval_pairs records -> (lines, qt_err_mean,
    pass_rate)."""
    ok = [r for r in records if r.status == 'ok']
    matched = [r for r in records if r.status != 'match_failed']
    qt = [max(r.terr, r.qerr) for r in ok]
    lines = [f'Pairs {len(records)} match_failed={len(records) - len(matched)} '
             f'geo_failed={len(matched) - len(ok)} num_matches={np.mean([r.N for r in matched]):.2f} '
             f'irat={np.mean([r.n_inls / r.N for r in ok]):.3f} time:{runtime:.2f}s']
    lines.append(inliers_distr_from_counts([r.counts[0] for r in matched], bins, 'cdist'))
    lines.append(inliers_distr_from_counts([r.counts[1] for r in matched], bins, 'fdist', return_ratios=True)[1])
    lines.append(inliers_distr_from_counts([r.counts[2] for r in ok], bins, 'indist', return_ratios=True)[1])
    pass_rate = np.array([100.0 * np.mean(np.array(qt) < thre) for thre in range(1, 11, 1)])
    qt_err_mean = np.mean(qt)
    qt_err_med = np.median(qt)
    lines.append('Pose err: qt_mean={:.2f}/{:.2f} qt<[1-10]deg:{}'.format(qt_err_mean, qt_err_med, pass_rate))
    return lines, qt_err_mean, pass_rate


def eval_immatch_val_sets(net, data_root='data/immatch_benchmark/val_dense', ksize=2, eval_type='fine', io_thres=0.5,
                          ncn_thres=0.0, imsize=1024, rthres=0.5, sample_max=300, min_overlap=0.3, lprint_=print):
    """utils/train/eval_epoch_immatch.py:12-98 -> (qt_err_mean, pass_rate), printing the same lines through lprint_.
    Scenes are the directories of data_root, each with dense/sparse/{cameras,images}.bin (COLMAP binary model),
    dense/sparse/ov_pairs.npy and dense/images."""
    net.eval()
    np.random.seed(0)
    lprint_(f'\n>>Eval on immatch: rthres={rthres} eval_type={eval_type} ov<{min_overlap} '
            f'nc={ncn_thres} ksize={ksize} io={io_thres} im={imsize}')
    start_time = time.time()
    pairs = []
    for scene, ims, pair_names in select_pairs(data_root, sample_max, min_overlap):
        im_dir = os.path.join(data_root, scene, 'dense/images')
        pairs += [(os.path.join(im_dir, a), os.path.join(im_dir, b), ims[a], ims[b]) for a, b in pair_names]
    records = eval_pairs(net, pairs, ksize, eval_type, io_thres, ncn_thres, imsize, rthres)
    lines, qt_err_mean, pass_rate = summarize(records, time.time() - start_time)
    for line in lines:
        lprint_(line)
    return qt_err_mean, pass_rate


# ---- validation pairs: the overlap precompute (utils/colmap/data_loading.py:7-70,
# data_pairs/precompute_immatch_val_ovs.py) ---------------------------------------------------------------------------
def overlap_scores_device(point3D_ids, device='cuda'):
    """p2p_overlap_scores on one int64 array of point3D_ids per image -> (scores [N, N] float64, counts [N] int32), CUDA
    tensors enqueued on the current stream: scores[i, j] = |A_i ∩ A_j| / max(|A_i|, |A_j|) for i < j, 1 on the
    diagonal and 0 below, A_i the indices of image i's keypoints with an id > 0.  Raises ZeroDivisionError, as the
    reference does, when two or more images have an empty A_i."""
    ids = [np.asarray(a, dtype=np.int64).reshape(-1) for a in point3D_ids]
    n = len(ids)
    if sum(1 for a in ids if not np.any(a > 0)) >= 2:
        raise ZeroDivisionError('division by zero')
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(a) for a in ids], out=offsets[1:])
    h = _lib.default_handle(torch.device(device))
    dev = h.device
    words = int((np.diff(offsets).max(initial=0) + 31) // 32)
    flat = torch.from_numpy(np.concatenate(ids) if n else np.zeros(0, dtype=np.int64)).to(dev)
    off = torch.from_numpy(offsets).to(dev)
    bits = torch.empty(n * words, dtype=torch.int32, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    scores = torch.empty(n, n, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_overlap_scores(h.h, _lib.ptr(flat), _lib.ptr(off),
                                            offsets.ctypes.data_as(C.POINTER(C.c_int64)), n, words, _lib.ptr(bits),
                                            _lib.ptr(counts), _lib.ptr(scores), h.stream()))
    return scores, counts


def cal_overlap_scores(im_ids, images, device='cuda'):
    """data_loading.py:54-70 -> (overlap_scores [N, N] float64, nums_3d [N] int64) as numpy, N = len(im_ids): the
    overlap of images i < j is the number of keypoint indices both have with a point3D_id > 0 over the larger of the
    two counts."""
    if len(im_ids) == 0:
        return np.eye(0), np.array([])          # the reference's empty result: a float64 nums_3d
    scores, counts = overlap_scores_device([images[i].point3D_ids for i in im_ids], device)
    return scores.cpu().numpy(), counts.cpu().numpy().astype(np.int64)


def _model_scores(model_dir, device):
    """(image names in images.bin order as an object array, the device overlap matrix) of a COLMAP model."""
    images = list(_read_images(os.path.join(model_dir, 'images.bin'), True, copy=False).values())
    names = np.empty(len(images), dtype=object)
    names[:] = [im.name for im in images]
    scores, _ = overlap_scores_device([im.point3D_ids for im in images], device)
    return names, scores


def _pairs_by_threshold(names, scores, thresholds):
    """The pair names of np.where((scores >= t) & (scores < 1)) for each t, each pair (max name, min name) by Python
    string order.  One mask [T, N, N] and one torch.nonzero, whose rows come grouped by threshold and row-major within
    a group (np.where's order): one device->host copy for nonzero's count and one for its rows."""
    if not thresholds:
        return []
    below = scores < 1
    mask = torch.stack([(scores >= t) & below for t in thresholds])
    idx = torch.nonzero(mask).to(torch.int32).cpu().numpy()
    rank = np.empty(len(names), dtype=np.int64)
    rank[sorted(range(len(names)), key=names.__getitem__)] = np.arange(len(names))
    bounds = np.searchsorted(idx[:, 0], np.arange(len(thresholds) + 1))
    out = []
    for k in range(len(thresholds)):
        i, j = idx[bounds[k]:bounds[k + 1], 1], idx[bounds[k]:bounds[k + 1], 2]
        swap = rank[i] < rank[j]
        out.append(list(zip(names[np.where(swap, j, i)].tolist(), names[np.where(swap, i, j)].tolist())))
    return out


def sav_model_multi_ov_pairs(model_dir, overlaps, device='cuda'):
    """data_loading.py:7-38: {overlap: pair names} of a COLMAP model, cached in model_dir/ov_pairs.npy.  A file holding
    every requested overlap is returned as it is; otherwise every requested overlap is recomputed (keys of the file that
    were not requested are dropped) and the file rewritten.  Prints the reference's lines."""
    sav_file_path = os.path.join(model_dir, 'ov_pairs.npy')
    if os.path.exists(sav_file_path):
        ov_pair_dict = np.load(sav_file_path, allow_pickle=True).item()
        if all(k in ov_pair_dict for k in overlaps):
            print('All overlaps have been computed.')
            return ov_pair_dict
    names, scores = _model_scores(model_dir, device)
    first = {}                                  # the reference's dict membership, for its skip rule
    for t in overlaps:
        first.setdefault(t, len(first))
    pairs = _pairs_by_threshold(names, scores, list(first))
    ov_pair_dict = {}
    for min_overlap in overlaps:
        if min_overlap in ov_pair_dict:
            print(f'ov>{min_overlap} exists, skip.')
            continue
        pair_names = pairs[first[min_overlap]]
        print(f'ov>{min_overlap} pairs: {len(pair_names)}')
        ov_pair_dict[min_overlap] = pair_names
    np.save(sav_file_path, ov_pair_dict)
    return ov_pair_dict


def load_model_ov_pairs(model_dir, min_overlap=0.3, device='cuda'):
    """data_loading.py:40-52: the pair names of one overlap threshold, computed from the model (no cache)."""
    names, scores = _model_scores(model_dir, device)
    pair_names = _pairs_by_threshold(names, scores, [min_overlap])[0]
    print('Loaded ov>{} pairs: {}'.format(min_overlap, len(pair_names)))
    return pair_names


def precompute_immatch_val_ovs(data_root, overlaps=(0.1, 0.2, 0.3, 0.4, 0.5), device='cuda'):
    """data_pairs/precompute_immatch_val_ovs.py: sav_model_multi_ov_pairs for every scene directory of data_root
    (os.listdir order), writing each scene's dense/sparse/ov_pairs.npy, with the script's printed lines."""
    overlaps = list(overlaps)
    scenes = os.listdir(data_root)
    print(f'Target scenes: {scenes}, ovs: {overlaps}\n')
    for scene in scenes:
        print(f'Start processing scene: {scene}')
        model_dir = os.path.join(data_root, scene, 'dense/sparse')
        t0 = time.time()
        sav_model_multi_ov_pairs(model_dir, overlaps, device)
        print(f'Finished, time {time.time() - t0}')


if __name__ == '__main__':
    import argparse
    parser = argparse.ArgumentParser(description='Write dense/sparse/ov_pairs.npy for every scene of a validation set.')
    parser.add_argument('--data_root', type=str, default='data/immatch_benchmark/val_as_train')
    precompute_immatch_val_ovs(parser.parse_args().data_root)
