"""Throughput of the image-matching validation loop (patch2pix_b200.evaluation) against the reference-style host flow.

    python bench_eval.py --out DIR [--pairs 50] [--scenes 2]

Writes a seeded synthetic validation tree under DIR (per scene: 1024x768 JPEGs, a COLMAP binary model, ov_pairs.npy),
loads seeded 'consensus' weights and times two arms on the same pairs, after one warm-up pair each:
  (a) eval_immatch_val_sets: matcher, E-RANSAC + pose and the Sampson histograms on the device, one table copy;
  (b) the reference's per-pair host flow (utils/train/eval_epoch_immatch.py:39-80): estimate_matches_from_files, numpy
      Sampson distances, cv2.findEssentialMat + cv2.recoverPose (utils/eval/geometry.py:32-48) and
      check_inliers_distr.
Prints both arms' summary lines, then one JSON line: pairs/s per arm, the host JPEG decode time of all pairs, the card
and its power limit.
"""
import argparse
import json
import os
import subprocess
import time

import numpy as np
import torch

from patch2pix_b200 import evaluation as E
from patch2pix_b200 import pose as P

KW = dict(ksize=2, io_thres=0.5, ncn_thres=0.0, imsize=1024, rthres=0.5)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def sampson(m, F):
    p1 = np.concatenate([m[:, 0:2], np.ones((len(m), 1))], 1)
    p2 = np.concatenate([m[:, 2:4], np.ones((len(m), 1))], 1)
    l2, l1 = F @ p1.T, F.T @ p2.T
    dd = np.sum(l2.T * p2, 1)
    return dd ** 2 / (1e-8 + l1[0] ** 2 + l1[1] ** 2 + l2[0] ** 2 + l2[1] ** 2)


def relapose_cv(p1, p2, K1, K2, rthres):
    """geometry.py:32-48: view 1 rescaled to view 2's focal length, principal points at the origin."""
    import cv2
    f1, f2 = K1[0, 0], K2[0, 0]
    p1 = (p1 - K1[:2, 2][None]) * f2 / f1
    p2 = p2 - K2[:2, 2][None]
    K = np.array([[f2, 0, 0], [0, f2, 0], [0, 0, 1]])
    Em, inls = cv2.findEssentialMat(p1, p2, cameraMatrix=K, method=cv2.FM_RANSAC, threshold=rthres)
    inls = np.where(inls > 0)[0]
    _, R, t, _ = cv2.recoverPose(Em, p1[inls], p2[inls], K)
    return inls, R, t


def host_arm(net, pairs):
    """The reference's loop body on the host, per pair; -> summary lines."""
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    cd, fd, ind, nm, irat, qt = [], [], [], [], [], []
    failed = geo = 0
    for p1, p2, im1, im2 in pairs:
        t_gt, q_gt = P.abs2relapose(im1.c, im2.c, im1.q, im2.q)
        F = P.pose2fund(im1.K, im2.K, P.quat2mat(q_gt), t_gt)
        try:
            m, _, c = estimate_matches_from_files(net, p1, p2, KW['ksize'], KW['ncn_thres'], True, KW['io_thres'],
                                                  'fine', KW['imsize'])
        except Exception:
            failed += 1
            continue
        fdist = sampson(m, F)
        cd.append(sampson(c, F))
        fd.append(fdist)
        nm.append(len(m))
        try:
            inls, R, t = relapose_cv(m[:, :2], m[:, 2:4], im1.K, im2.K, KW['rthres'])
        except Exception:
            geo += 1
            continue
        qt.append(max(P.cal_vec_angle_error(t.squeeze(), t_gt), P.cal_quat_angle_error(P.mat2quat(R), q_gt)))
        irat.append(len(inls) / len(m))
        ind.append(fdist[inls])
    pass_rate = np.array([100.0 * np.mean(np.array(qt) < thre) for thre in range(1, 11, 1)])
    return [f'Pairs {len(pairs)} match_failed={failed} geo_failed={geo} num_matches={np.mean(nm):.2f} '
            f'irat={np.mean(irat):.3f}',
            E.check_inliers_distr(cd, bins=E.EVAL_BINS, tag='cdist'),
            E.check_inliers_distr(fd, bins=E.EVAL_BINS, tag='fdist', return_ratios=True)[1],
            E.check_inliers_distr(ind, bins=E.EVAL_BINS, tag='indist', return_ratios=True)[1],
            'Pose err: qt_mean={:.2f}/{:.2f} qt<[1-10]deg:{}'.format(np.mean(qt), np.median(qt), pass_rate)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True, help='directory for the synthetic validation tree')
    ap.add_argument('--scenes', type=int, default=2)
    ap.add_argument('--pairs', type=int, default=50, help='pairs per scene')
    args = ap.parse_args()
    from PIL import Image
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_val_scene

    root = os.path.join(args.out, 'val')
    warm = os.path.join(args.out, 'warm')
    for k in range(args.scenes):
        synthetic_val_scene(root, f'scene{k}', k, [(1024, 768)] * args.pairs, ext='.jpg')
    synthetic_val_scene(warm, 'warm', 99, [(1024, 768)], ext='.jpg')
    net = load_model(make_seeded_state_dict(0, nc_init='consensus'))

    np.random.seed(0)
    pairs = []
    for scene, ims, names in E.select_pairs(root, 300, 0.3):
        d = os.path.join(root, scene, 'dense/images')
        pairs += [(os.path.join(d, a), os.path.join(d, b), ims[a], ims[b]) for a, b in names]

    t0 = time.perf_counter()
    for p1, p2, _, _ in pairs:
        np.asarray(Image.open(p1).convert('RGB'))
        np.asarray(Image.open(p2).convert('RGB'))
    decode_s = time.perf_counter() - t0

    E.eval_immatch_val_sets(net, warm, lprint_=lambda s: None, **KW)         # warm-up: one pair per arm
    lines_a = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    E.eval_immatch_val_sets(net, root, lprint_=lines_a.append, **KW)
    torch.cuda.synchronize()
    ta = time.perf_counter() - t0

    np.random.seed(0)
    warm_pairs = [(os.path.join(warm, 'warm/dense/images', a), os.path.join(warm, 'warm/dense/images', b), ims[a], ims[b])
                  for _, ims, names in E.select_pairs(warm, 300, 0.3) for a, b in names]
    host_arm(net, warm_pairs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lines_b = host_arm(net, pairs)
    tb = time.perf_counter() - t0

    print('(a) eval_immatch_val_sets:' + ''.join('\n  ' + s.strip('\n').replace('\n', '\n  ') for s in lines_a))
    print('(b) host flow:' + ''.join('\n  ' + s.replace('\n', '\n  ') for s in lines_b))
    print(json.dumps({'pairs': len(pairs), 'eval_pairs_per_s': len(pairs) / ta, 'host_flow_pairs_per_s': len(pairs) / tb,
                      'speedup': tb / ta, 'eval_s': ta, 'host_flow_s': tb, 'host_decode_s': decode_s,
                      'card': card()}), flush=True)


if __name__ == '__main__':
    main()
