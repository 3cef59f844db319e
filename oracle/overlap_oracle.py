"""numpy restatement of the reference's overlap precompute (utils/colmap/data_loading.py:7-70), for tests only.

cal_overlap_scores: the np.intersect1d double loop over the keypoint indices with a point3D_id > 0, divided by the
larger count in Python true division (raises ZeroDivisionError when two images have no such index).  pairs: the rule
np.where((ov >= t) & (ov < 1)) over the full matrix, each pair named (max(name_i, name_j), min(name_i, name_j)).
"""
import numpy as np


def cal_overlap_scores(point3D_ids):
    """point3D_ids: one array per image -> (ov [N, N] float64, nums_3d [N]) as the reference returns them."""
    n = len(point3D_ids)
    ov = np.eye(n)
    im_3ds = [np.where(np.asarray(p) > 0)[0] for p in point3D_ids]
    for i in range(n):
        for j in range(i + 1, n):
            ov[i, j] = len(np.intersect1d(im_3ds[i], im_3ds[j])) / max(len(im_3ds[i]), len(im_3ds[j]))
    return ov, np.array([len(v) for v in im_3ds])


def pairs(ov, names, t):
    """The pair names of threshold t, in np.where's row-major order."""
    out = []
    for i, j in np.vstack(np.where(np.logical_and(ov >= t, ov < 1))).T:
        out.append((max(names[i], names[j]), min(names[i], names[j])))
    return out


def exact_scores(point3D_ids):
    """The same matrix from an exact int64 Gram matrix X X^T of the 0/1 keypoint masks, for large seeded models."""
    n = len(point3D_ids)
    width = max([len(p) for p in point3D_ids], default=0)
    X = np.zeros((n, width), dtype=np.int64)
    for i, p in enumerate(point3D_ids):
        X[i, :len(p)] = np.asarray(p) > 0
    G = X @ X.T
    cnt = X.sum(1)
    ov = np.eye(n)
    iu = np.triu_indices(n, 1)
    ov[iu] = G[iu].astype(np.float64) / np.maximum(cnt[iu[0]], cnt[iu[1]]).astype(np.float64)
    return ov, cnt
