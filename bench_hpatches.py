"""Throughput of the HPatches evaluation (patch2pix_b200.hpatches) against a per-pair host flow, and of its kernel.

    python bench_hpatches.py [--out DIR] [--seqs 12] [--rounds 2]

Writes a seeded synthetic HPatches tree (half i_, half v_ sequences, 1.ppm of 640..1024 px wide; under a temporary
directory unless --out is given), loads seeded 'consensus' weights and, after one untimed pass of each arm over the
whole tree (every image shape warmed up), times two arms alternately (--rounds passes each, the fastest reported):
  (a) eval_hpatches(net, ...): matching, H RANSAC and p2p_homography_errors on the device, one table copy;
  (b) the host flow: estimate_matches_from_files(..., verify=('H', 2.0)) per pair, then the numpy statistics of
      oracle/hpatches_oracle.py;
and, once,
  (c) p2p_homography_errors alone against the numpy statistics on 10^5 rows (CUDA events over repeated launches).
Checks that (a) and (b) give the same records (counts bit-exact outside a 1e-12 relative band around each threshold,
corner errors within 1e-12 relative) and prints one JSON line with the times, the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from oracle import hpatches_oracle as O
from patch2pix_b200 import hpatches as HP

KW = dict(ksize=2, io_thres=0.25, ncn_thres=0.0, imsize=1024)
THR = list(range(1, 11))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def host_flow(net, seqs):
    """Per pair: estimate_matches_from_files with H RANSAC, then the numpy statistics -> [(N, n_inliers, counts,
    corner error, the rows' errors)]."""
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    out = []
    for s in seqs:
        for k in range(2, 7):
            m, _, _, inl, model = estimate_matches_from_files(net, s.paths[0], s.paths[k - 1], KW['ksize'],
                                                              KW['ncn_thres'], True, KW['io_thres'], 'fine',
                                                              KW['imsize'], verify=('H', 2.0))
            n_inl = int(inl.sum()) if model is not None else 0
            d = O.reprojection_errors(m, s.H_gt[k - 2])
            ce = O.corner_error(s.H_gt[k - 2], model if model is not None else np.eye(3), n_inl, *s.size)
            out.append((len(m), n_inl, O.counts(d, THR), ce, d))
    return out


def same_records(recs, host):
    for r, (n, n_inl, c, ce, d) in zip(recs, host):
        if r.N != n or (n_inl > 0 and r.n_inliers != n_inl) or (n_inl == 0 and r.n_inliers > 0):
            return False
        for j, t in enumerate(THR):
            near = int(np.count_nonzero(np.abs(d - t) <= 1e-12 * t))
            if abs(int(r.counts[j]) - int(c[j])) > near:
                return False
        if r.counts[-1] != c[-1]:
            return False
        if not (r.corner_err == ce or abs(r.corner_err - ce) <= 1e-12 * abs(ce)):
            return False
    return len(recs) == len(host)


def kernel_arm(n=100_000, reps=200):
    rng = np.random.default_rng(0)
    H = np.array([[0.95, 0.08, 12.0], [-0.05, 1.03, -7.5], [1.2e-4, -0.8e-4, 1.0]])
    x = rng.uniform([0, 0], [1024, 768], (n, 2))
    px, py, _ = O.project(H, x[:, 0], x[:, 1])
    rows = np.concatenate([x, np.stack([px, py], 1) + rng.normal(0, 3.0, (n, 2))], 1)
    buf = np.zeros(10)
    buf[:9] = (H + 1e-4).reshape(9)
    buf[9:10].view(np.int32)[0] = n // 2
    rows_d, buf_d = torch.from_numpy(rows).cuda(), torch.from_numpy(buf).cuda()
    counts, ce = HP.homography_errors(rows_d, H, buf_d, 1024, 768, THR)
    exp_c = O.counts(O.reprojection_errors(rows, H), THR)
    exp_e = O.corner_error(H, buf[:9], n // 2, 1024, 768)
    ok = np.array_equal(counts.cpu().numpy(), exp_c) and float(ce.cpu()[0]) == exp_e
    for _ in range(10):
        HP.homography_errors(rows_d, H, buf_d, 1024, 768, THR)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        HP.homography_errors(rows_d, H, buf_d, 1024, 768, THR)
    e1.record()
    e1.synchronize()
    dev_ms = e0.elapsed_time(e1) / reps
    t0 = time.perf_counter()
    for _ in range(10):
        O.counts(O.reprojection_errors(rows, H), THR)
        O.corner_error(H, buf[:9], n // 2, 1024, 768)
    host_ms = (time.perf_counter() - t0) * 100
    return ok, dev_ms, host_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the synthetic tree (default: a temporary one)')
    ap.add_argument('--seqs', type=int, default=12, help='sequences (5 pairs each)')
    ap.add_argument('--rounds', type=int, default=2, help='timed passes of each arm, alternating')
    args = ap.parse_args()
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_hpatches_tree

    with tempfile.TemporaryDirectory() as tmp:
        out = args.out or tmp
        root = os.path.join(out, 'hpatches')
        rng = np.random.default_rng(1)
        names = [(f'{"iv"[j % 2]}_seq{j:02d}', (int(rng.integers(640, 1025)), int(rng.integers(480, 769))))
                 for j in range(args.seqs)]
        synthetic_hpatches_tree(root, 11, names)
        net = load_model(make_seeded_state_dict(0, nc_init='consensus'))
        seqs = HP.read_hpatches(root)

        # warm-up: one untimed pass of each arm over every image shape the timed passes use, then the two arms
        # alternately, twice; the faster pass of each arm is reported
        HP.eval_hpatches(net, root, lprint_=lambda s: None, **KW)
        host_flow(net, seqs)
        ta, tb = [], []
        for _ in range(args.rounds):
            lines = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = HP.eval_hpatches(net, root, lprint_=lines.append, **KW)
            torch.cuda.synchronize()
            ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            host = host_flow(net, seqs)
            tb.append(time.perf_counter() - t0)
        ta, tb = min(ta), min(tb)

    equal = same_records(res['records'], host)
    k_ok, k_dev_ms, k_host_ms = kernel_arm()
    print('(a) eval_hpatches:' + ''.join('\n  ' + s.strip('\n') for s in lines))
    print(json.dumps({'pairs': res['n_pairs'], 'records_equal': equal, 'eval_hpatches_s': ta, 'host_flow_s': tb,
                      'eval_pairs_per_s': res['n_pairs'] / ta, 'host_flow_pairs_per_s': res['n_pairs'] / tb,
                      'speedup': tb / ta, 'kernel_1e5_rows_ms': k_dev_ms, 'numpy_1e5_rows_ms': k_host_ms,
                      'kernel_equals_numpy': k_ok, 'card': card()}), flush=True)
    if not (equal and k_ok):
        raise SystemExit('records differ')


if __name__ == '__main__':
    main()
