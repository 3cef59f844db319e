"""Throughput of absolute-pose RANSAC (patch2pix_b200.localize) against OpenCV, and of localize_inloc against a host flow.

    python bench_abspose.py [--queries 200] [--inloc_queries 8] [--inloc_db 4] [--rounds 1] [--out DIR]

  (a) find_absolute_poses over --queries seeded queries (synth.synthetic_abspose: 2k-8k rows, 20-50 % inliers, 1 px
      noise, 8 px threshold, conf 0.99999, 10000 iterations), one batched call, against a cv2.solvePnPRansac loop (P3P,
      same threshold, confidence and iteration cap) over the same queries.  Both arms' rotation and position errors
      against the true poses are printed (median, 90th percentile, share within 0.25 units and 2 degrees): the samplers
      and refinements differ, so the poses agree within RANSAC's randomness, not bit for bit.
  (b) localize_inloc with a seeded Patch2PixB200 on a synthetic InLoc tree (synth.synthetic_inloc_tree, 320 x 240
      images; under a temporary directory unless --out is given) against the host flow: estimate_matches_from_files
      per pair, the numpy lift of oracle/abspose_oracle.py, then cv2.solvePnPRansac per query at 48 px.
After one untimed pass of each GPU arm (OpenCV needs none), the arms alternate --rounds times, the fastest pass
reported; the OpenCV loop takes about half a second per query on the host.  Prints one JSON
line with the times, the comparisons, the card's name and its power limit.  Without cv2 the host arms are null.
"""
import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from oracle import abspose_oracle as A
from patch2pix_b200 import localize as L
from patch2pix_b200.synth import synthetic_abspose

TH, CONF, ITERS = 8.0, 0.99999, 10000


def log(msg):
    print(f'[{time.strftime("%H:%M:%S")}] {msg}', flush=True)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def errors(R, t, R0, t0):
    if R is None:
        return np.inf, np.inf
    ang = np.degrees(np.arccos(np.clip((np.trace(R0.T @ R) - 1) / 2, -1, 1)))
    return float(np.linalg.norm(-R.T @ np.ravel(t) + R0.T @ t0)), float(ang)


def stats(errs):
    e = np.array(errs, dtype=np.float64)
    return {'median_pos': float(np.median(e[:, 0])), 'p90_pos': float(np.percentile(e[:, 0], 90)),
            'median_deg': float(np.median(e[:, 1])), 'p90_deg': float(np.percentile(e[:, 1], 90)),
            'within_0.25_2deg': float(np.mean((e[:, 0] <= 0.25) & (e[:, 1] <= 2.0)))}


def cv2_pnp(cv2, p2, p3, K, th):
    if len(p2) < 4:
        return None, None
    ok, rv, tv, _ = cv2.solvePnPRansac(np.ascontiguousarray(p3), np.ascontiguousarray(p2), K, None,
                                       iterationsCount=ITERS, reprojectionError=th, confidence=CONF,
                                       flags=cv2.SOLVEPNP_P3P)
    return (cv2.Rodrigues(rv)[0], tv.ravel()) if ok else (None, None)


def bench_pnp(cv2, n_queries, rounds):
    rng = np.random.default_rng(7)
    scs = [synthetic_abspose(1000 + k, int(rng.integers(2000, 8001)), float(rng.uniform(0.5, 0.8)), 1.0)
           for k in range(n_queries)]
    p2, p3, Ks = [s['pts2d'] for s in scs], [s['pts3d'] for s in scs], [s['K'] for s in scs]
    log(f'pnp: {n_queries} queries, {sum(len(a) for a in p2)} rows')
    L.find_absolute_poses(p2, p3, Ks, TH, CONF, ITERS)
    ta, tb = [], []
    for r in range(rounds):
        log(f'pnp round {r}')
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gpu = L.find_absolute_poses(p2, p3, Ks, TH, CONF, ITERS)
        ta.append(time.perf_counter() - t0)
        if cv2 is not None:
            t0 = time.perf_counter()
            host = [cv2_pnp(cv2, a, b, K, TH) for a, b, K in zip(p2, p3, Ks)]
            tb.append(time.perf_counter() - t0)
    out = {'queries': n_queries, 'rows': int(sum(len(a) for a in p2)), 'gpu_batched_s': min(ta),
           'gpu_queries_per_s': n_queries / min(ta),
           'gpu_errors': stats([errors(R, t, s['R'], s['t']) for (R, t, _), s in zip(gpu, scs)])}
    if cv2 is not None:
        out.update({'cv2_loop_s': min(tb), 'cv2_queries_per_s': n_queries / min(tb),
                    'cv2_errors': stats([errors(R, t, s['R'], s['t']) for (R, t), s in zip(host, scs)])})
    return out


def host_inloc(cv2, net, root, ret):
    from PIL import Image
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    poses = {}
    for q, dbs in ret:
        rows = [A.lift_scan(L.read_scan(os.path.join(root, d + '.mat')), L.read_alignment(L.alignment_path(root, d)),
                            estimate_matches_from_files(net, os.path.join(root, q), os.path.join(root, d), 2, 0.0, True,
                                                        0.25, 'fine', 1024)[0]) for d in dbs]
        rows = np.concatenate(rows)
        w, h = Image.open(os.path.join(root, q)).size
        K = np.array([[L.INLOC_FOCAL, 0, w / 2], [0, L.INLOC_FOCAL, h / 2], [0, 0, 1.0]])
        poses[os.path.basename(q)] = cv2_pnp(cv2, rows[:, :2], rows[:, 2:], K, 48.0)
    return poses


def bench_inloc(cv2, root, n_q, n_db, rounds):
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_inloc_tree
    tree = synthetic_inloc_tree(root, 5, n_q, n_db)
    ret = L.read_retrieval(tree['pairs'])
    net = load_model(make_seeded_state_dict(0, nc_init='consensus'))
    res_path = os.path.join(root, 'results.txt')
    quiet = dict(lprint_=lambda s: None)
    log(f'inloc: {n_q} queries x {n_db} cutouts')
    L.localize_inloc(net, root, tree['pairs'], res_path, **quiet)
    if cv2 is not None:
        host_inloc(cv2, net, root, ret)
    ta, tb = [], []
    for r in range(rounds):
        log(f'inloc round {r}')
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = L.localize_inloc(net, root, tree['pairs'], res_path, **quiet)
        ta.append(time.perf_counter() - t0)
        if cv2 is not None:
            t0 = time.perf_counter()
            host = host_inloc(cv2, net, root, ret)
            tb.append(time.perf_counter() - t0)
    gt = L.read_results(tree['gt'])
    out = {'inloc_queries': n_q, 'inloc_pairs': n_q * n_db, 'localize_inloc_s': min(ta),
           'localize_recall': {str(k): v for k, v in L.eval_localization(res_path, gt)['recall'].items()},
           'localize_failed': len(res['failed'])}
    if cv2 is not None:
        hp = {n: (R, t) for n, (R, t) in host.items() if R is not None}
        out.update({'host_flow_s': min(tb),
                    'host_recall': {str(k): v for k, v in L.eval_localization(hp, gt)['recall'].items()},
                    'pose_gap_gpu_vs_host': [errors(*res['poses'][n][:2], *hp[n]) for n in sorted(hp)]})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--queries', type=int, default=200)
    ap.add_argument('--inloc_queries', type=int, default=8)
    ap.add_argument('--inloc_db', type=int, default=4)
    ap.add_argument('--rounds', type=int, default=1, help='timed passes of each arm, alternating')
    ap.add_argument('--out', default=None, help='directory for the synthetic tree (default: a temporary one)')
    args = ap.parse_args()
    try:
        import cv2
    except ImportError:
        cv2 = None
    out = {'pnp': bench_pnp(cv2, args.queries, args.rounds)}
    with tempfile.TemporaryDirectory() as tmp:
        out['inloc'] = bench_inloc(cv2, os.path.join(args.out or tmp, 'inloc'), args.inloc_queries, args.inloc_db,
                                   args.rounds)
    out['card'] = card()
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
