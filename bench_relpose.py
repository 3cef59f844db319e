"""Throughput of the relative-pose evaluation (patch2pix_b200.relpose) against a per-pair host flow with OpenCV.

    python bench_relpose.py [--out DIR] [--pairs 24] [--rounds 2]

Writes a seeded synthetic pair tree (synth.synthetic_relpose_tree, SuperGlue's text format, 640 x 480 images; under a
temporary directory unless --out is given), loads seeded 'consensus' weights and, after one untimed pass of each arm,
times two arms alternately (--rounds passes each, the fastest reported):
  (a) eval_relpose(net, ...): matching, per-pair-threshold E RANSAC, pose recovery and p2p_relpose_errors_batch on the
      device for every chunk of pairs, one table copy;
  (b) the host flow of SuperGlue / LoFTR: estimate_matches_from_files per pair, cv2.findEssentialMat on normalised
      points at ransac_thres / f_mean (RANSAC, conf 0.99999), cv2.recoverPose(..., 1e9, mask) of every returned E
      keeping the one with the most points, then the numpy errors of oracle/relpose_oracle.py;
and then, on the matches of (b) held in memory,
  (c) the batched RANSAC + error pass alone (eval_relpose with a callable returning the device rows) against
  (d) the per-pair cv2 loop with the numpy errors.
Prints both arms' AUCs (they differ within RANSAC's randomness: different samplers, one E against several) and one JSON
line with the times, the card and its power limit.  Without cv2 the host arms are null.
"""
import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from oracle import relpose_oracle as O
from patch2pix_b200 import relpose as RP

KW = dict(ksize=2, io_thres=0.25, ncn_thres=0.0, imsize=1024)
AUC_T = [5.0, 10.0, 20.0]
EPI = [5e-4]
RTHRES, CONF = 0.5, 0.99999


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def cv2_pose(cv2, m, p):
    """SuperGlue / LoFTR's estimate_pose + relative_pose_error on one pair's matches -> (pose error, counts)."""
    K0, K1 = p.K0, p.K1
    Rt_gt = np.concatenate([p.T_0to1[:3, :3].reshape(9), p.T_0to1[:3, 3]])
    intr = np.array([K0[0, 0], K0[1, 1], K0[0, 2], K0[1, 2], K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]])
    cnt = O.counts(O.epipolar_errors(m, intr, Rt_gt), EPI)
    if len(m) < 5:
        return np.inf, cnt
    k0 = (m[:, :2] - K0[[0, 1], [2, 2]][None]) / K0[[0, 1], [0, 1]][None]
    k1 = (m[:, 2:4] - K1[[0, 1], [2, 2]][None]) / K1[[0, 1], [0, 1]][None]
    thr = RTHRES / np.mean([K0[0, 0], K1[1, 1], K0[0, 0], K1[1, 1]])
    E, mask = cv2.findEssentialMat(k0, k1, np.eye(3), threshold=thr, prob=CONF, method=cv2.RANSAC)
    if E is None:
        return np.inf, cnt
    best, ret = 0, None
    for E_ in np.split(E, len(E) / 3):
        n, R, t, _ = cv2.recoverPose(E_, k0, k1, np.eye(3), 1e9, mask=mask)
        if n > best:
            best, ret = n, (R, t[:, 0])
    if ret is None:
        return np.inf, cnt
    est = np.concatenate([ret[0].reshape(9), ret[1]])
    return max(O.pose_errors(*O.pose_cosines(Rt_gt, est, 1))), cnt


def host_flow(cv2, net, pairs):
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    ms = [estimate_matches_from_files(net, p.path0, p.path1, KW['ksize'], KW['ncn_thres'], True, KW['io_thres'],
                                      'fine', KW['imsize'])[0] for p in pairs]
    return ms, [cv2_pose(cv2, m, p) for m, p in zip(ms, pairs)]


def summary(errs, counts):
    return O.pose_auc(errs, AUC_T), O.precision(counts, EPI)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the synthetic tree (default: a temporary one)')
    ap.add_argument('--pairs', type=int, default=24)
    ap.add_argument('--rounds', type=int, default=2, help='timed passes of each arm, alternating')
    args = ap.parse_args()
    try:
        import cv2
    except ImportError:
        cv2 = None
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_relpose_tree

    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(args.out or tmp, 'relpose')
        path, _ = synthetic_relpose_tree(root, 13, args.pairs, fmt='txt', size=(640, 480))
        pairs = RP.read_pairs(path, root)
        net = load_model(make_seeded_state_dict(0, nc_init='consensus'))
        quiet = dict(lprint_=lambda s: None)
        RP.eval_relpose(net, path, root, **quiet, **KW)
        if cv2 is not None:
            host_flow(cv2, net, pairs)
        ta, tb = [], []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = RP.eval_relpose(net, path, root, **quiet, **KW)
            torch.cuda.synchronize()
            ta.append(time.perf_counter() - t0)
            if cv2 is not None:
                t0 = time.perf_counter()
                ms, host = host_flow(cv2, net, pairs)
                tb.append(time.perf_counter() - t0)

        out = {'pairs': len(pairs), 'eval_relpose_s': min(ta), 'eval_pairs_per_s': len(pairs) / min(ta),
               'eval_auc': [res['auc'][t] for t in AUC_T], 'eval_prec': res['prec'][EPI[0]],
               'mean_matches': res['n_matches']}
        if cv2 is not None:
            h_auc, h_prec = summary([e for e, _ in host], [c for _, c in host])
            # (c) / (d): the RANSAC and error pass alone on the same matches
            dev_rows = {(p.path0, p.path1): torch.from_numpy(m).cuda() for p, m in zip(pairs, ms)}
            matcher = lambda a, b: dev_rows[(a, b)]
            RP.eval_relpose(matcher, path, root, **quiet)
            tc, td = [], []
            for _ in range(max(2, args.rounds)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res_c = RP.eval_relpose(matcher, path, root, **quiet)
                torch.cuda.synchronize()
                tc.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                [cv2_pose(cv2, m, p) for m, p in zip(ms, pairs)]
                td.append(time.perf_counter() - t0)
            out.update({'host_flow_s': min(tb), 'host_flow_pairs_per_s': len(pairs) / min(tb),
                        'host_auc': [h_auc[t] for t in AUC_T], 'host_prec': h_prec[EPI[0]],
                        'prec_equal': h_prec == res['prec'],
                        'batched_ransac_errors_ms': min(tc) * 1e3, 'cv2_loop_ms': min(td) * 1e3,
                        'batched_pairs_per_s': len(pairs) / min(tc), 'cv2_pairs_per_s': len(pairs) / min(td),
                        'batched_auc': [res_c['auc'][t] for t in AUC_T]})
        else:
            out.update({'host_flow_s': None, 'host_flow_pairs_per_s': None, 'host_auc': None,
                        'batched_ransac_errors_ms': None, 'cv2_loop_ms': None})
    out['card'] = card()
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
