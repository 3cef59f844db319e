"""Time the GPU triangulation (triangulate_from_matches) and localization (localize_from_matches) on a seeded synthetic
model of realistic size, against the host flow: the numpy oracle for triangulation and cv2.solvePnPRansac for the
queries, on a subset (the oracle is a per-track Python loop).  Prints the card and its power limit.

    python bench_sfm.py [--images 500] [--pairs_per_image 20] [--matches 2000] [--queries 200] [--host_pairs 40]
"""
import argparse
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from oracle import sfm_oracle as O
from patch2pix_b200 import sfm as S
from patch2pix_b200.localize import rotmat_to_qvec
from patch2pix_b200.synth import _look_at, write_colmap_model

W, H, F, K1 = 1024, 768, 800.0, -0.05


def scene(seed, n_img, n_pts=100000):
    rng = np.random.default_rng(seed)
    X = rng.uniform([-40, -40, -5], [40, 40, 5], (n_pts, 3))
    poses = []
    for i in range(n_img):
        a = 2 * np.pi * i / n_img
        C = np.array([60 * np.cos(a), 60 * np.sin(a), rng.uniform(-2, 2)])
        R = _look_at(C, rng.uniform(-5, 5, 3), rng.uniform(-0.05, 0.05))
        poses.append((R, -R @ C))
    return rng, X, poses


def project(R, t, X):
    P = X @ R.T + t
    u, v = P[:, 0] / P[:, 2], P[:, 1] / P[:, 2]
    d = 1 + K1 * (u * u + v * v)
    x, y = F * u * d + W / 2, F * v * d + H / 2
    return x, y, (P[:, 2] > 0) & (x >= 0) & (x < W) & (y >= 0) & (y < H)


def matches(rng, X, pa, pb, n, cache={}):
    xa, ya, oka = cache[id(pa)] if id(pa) in cache else cache.setdefault(id(pa), project(*pa, X))
    xb, yb, okb = cache[id(pb)] if id(pb) in cache else cache.setdefault(id(pb), project(*pb, X))
    idx = np.nonzero(oka & okb)[0]
    idx = idx[rng.permutation(len(idx))[:n]]
    m = np.stack([xa[idx], ya[idx], xb[idx], yb[idx]], 1) + rng.normal(0, 0.5, (len(idx), 4))
    bad = rng.random(len(m)) < 0.1
    m[bad, 2] = rng.uniform(0, W, bad.sum())
    m[bad, 3] = rng.uniform(0, H, bad.sum())
    return m


def gpu_time(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=500)
    ap.add_argument('--pairs_per_image', type=int, default=20)
    ap.add_argument('--matches', type=int, default=2000)
    ap.add_argument('--queries', type=int, default=200)
    ap.add_argument('--query_pairs', type=int, default=20)
    ap.add_argument('--host_pairs', type=int, default=40)
    ap.add_argument('--host_queries', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    a = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'card: {smi or torch.cuda.get_device_name()}')
    rng, X, poses = scene(a.seed, a.images + a.queries)
    db, qp = poses[:a.images], poses[a.images:]
    tmp = tempfile.mkdtemp()
    names = [f'db/{i:05d}.jpg' for i in range(a.images)]
    write_colmap_model(tmp, [(1, 2, W, H, [F, W / 2, H / 2, K1])],
                       [(i + 1, rotmat_to_qvec(R), t, 1, names[i]) for i, (R, t) in enumerate(db)])
    pairs = [(names[i], names[(i + 1 + j) % a.images]) for i in range(a.images) for j in range(a.pairs_per_image)]
    t0 = time.perf_counter()
    idx = {n: i for i, n in enumerate(names)}
    mt = [torch.from_numpy(matches(rng, X, db[idx[p]], db[idx[q]], a.matches)).cuda() for p, q in pairs]
    print(f'{len(pairs)} database pairs, {sum(len(m) for m in mt)} matches (generated in '
          f'{time.perf_counter() - t0:.1f} s)')
    t_tri, sfm = gpu_time(lambda: S.triangulate_from_matches(tmp, pairs, mt))
    print(f'GPU triangulation: {t_tri:.3f} s  stats={sfm.stats}')
    qs, ret, qm = {}, [], []
    for k, (R, t) in enumerate(qp):
        qn = f'query/{k:04d}.jpg'
        qs[qn] = S.Namespace(model='SIMPLE_RADIAL', width=W, height=H, params=np.array([F, W / 2, H / 2, K1]))
        C = -R.T @ t
        near = np.argsort([np.linalg.norm(C + Rd.T @ td) for Rd, td in db])[:a.query_pairs]
        ret.append((qn, [names[j] for j in near]))
        qm += [torch.from_numpy(matches(rng, X, (R, t), db[j], a.matches)).cuda() for j in near]
    out = os.path.join(tmp, 'results.txt')
    t_loc, res = gpu_time(lambda: S.localize_from_matches(sfm, qs, ret, qm, out))
    print(f'GPU localization: {t_loc:.3f} s for {len(ret)} queries, {len(res["failed"])} failed')
    # host arm on a subset
    hp = pairs[:a.host_pairs]
    cameras, images, cams, img_cam, recs = S._model_tables(tmp)
    pt = S._pair_tables(images, cams, img_cam, recs, hp, 4.0)
    hm = [m.cpu().numpy() for m in mt[:a.host_pairs]]
    t0 = time.perf_counter()
    O.triangulate_host((cams, img_cam, recs), pt, hm)
    t_host = time.perf_counter() - t0
    t_sub, _ = gpu_time(lambda: S.triangulate_from_matches(tmp, hp, mt[:a.host_pairs]))
    print(f'triangulation, {len(hp)} pairs: numpy oracle {t_host:.2f} s, GPU {t_sub:.4f} s')
    import cv2
    t0 = time.perf_counter()
    for k in range(a.host_queries):
        rows, _ = O.query_rows([m.cpu().numpy() for m in qm[k * a.query_pairs:(k + 1) * a.query_pairs]],
                               [(0, idx[d]) for d in ret[k][1]], [S.camera_record('SIMPLE_RADIAL', qs[ret[k][0]].params)],
                               sfm.kp_xy, sfm.kp_key, sfm.kp_point, sfm.points, 4.0)
        if len(rows) >= 4:
            cv2.solvePnPRansac(rows[:, 2:], rows[:, :2], np.array([[F, 0, W / 2], [0, F, H / 2], [0, 0, 1]]), None,
                               reprojectionError=12.0, iterationsCount=10000, confidence=0.99999,
                               flags=cv2.SOLVEPNP_P3P)
    t_hq = (time.perf_counter() - t0) / a.host_queries
    print(f'localization per query: oracle rows + cv2.solvePnPRansac {t_hq:.3f} s, GPU {t_loc / len(ret):.5f} s')


if __name__ == '__main__':
    main()
