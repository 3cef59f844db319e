"""Time match verification: p2p_find_model on the GPU against OpenCV on the host, on the same rows.

    python bench_verify.py [--calls 200] [--cpu-reps 20] [--batch-pairs 256] [--batch-calls 5]

Two workloads of 3200 rows each, for F and for H:
  * `fine`: the fine matches of one pair of bench.py's workload (640x480 synthetic_pair_shifted, consensus NC weights,
    ptmax 400, panc 8).  The seeded regressor is untrained, so these rows carry little consistent geometry and RANSAC
    tends to run to max_iters.
  * `scene`: synthetic_two_view with 50 % outliers and 0.5 px noise (planar for H), where the stopping bound ends
    RANSAC early.
Threshold 1 px for F and 2 px for H as in the reference's notebook, conf 0.999, at most 10000 iterations, seed 0.
GPU time: CUDA events around `--calls` back-to-back calls.  CPU time: host clock around `--cpu-reps` calls of
cv2.findFundamentalMat (USAC_ACCURATE) / cv2.findHomography (RANSAC), or null without cv2.
E (relative pose, the reference's matches2relapose_cv) runs on the same two workloads (the `scene` one non-planar)
with K at focal 500 px and the principal point at the image centre, 1 px, conf 0.999, at most 1000 iterations
(cv2's defaults): p2p_find_essential + p2p_recover_pose on its inliers against cv2.findEssentialMat (RANSAC) +
cv2.recoverPose.
DEGENSAC (F with the plane-degeneracy check, model 2 of p2p_find_model) runs on the `fine` workload and on `plane`, a
3200-row synthetic_dominant_plane scene (30 % outliers, 8 % of the inliers off the dominant plane, 0.5 px noise), at 1 px
against cv2.findFundamentalMat (USAC_ACCURATE); for `plane` it also reports the recall of the off-plane inliers.
Batch workload (`batch` in the output): --batch-pairs seeded pairs with row counts drawn uniformly from 300..3200
(synthetic_two_view, 40 % outliers, 0.5 px noise; planar for H; synthetic_dominant_plane for DEGENSAC), timed with CUDA
events as the K back-to-back single-pair calls (`ms_single`) and as one batched call (`ms_batch`), each the mean of
--batch-calls repetitions after a warm-up; for E both arms also run pose recovery on the inliers (`E+pose`).  The two
arms' outputs are compared byte for byte (`identical`).  `ms_cpu`: one pass of OpenCV over the K pairs on the host.
Prints one JSON line and writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

TH = {'F': 1.0, 'H': 2.0, 'DEGENSAC': 1.0}
MODEL = {'F': 0, 'H': 1, 'DEGENSAC': 2}


def fine_matches(dev):
    from argparse import Namespace
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_pair_shifted
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    cfg = Namespace(training=False, device=dev, regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=make_seeded_state_dict(0, nc_init='consensus'), change_stride=True, regressor_config=rc)
    net = Patch2PixB200(cfg)
    im1, im2 = synthetic_pair_shifted(0, 480, 640)
    with torch.no_grad():
        f1 = net.extract.forward_all(im1.to(dev), [], True)
        f2 = net.extract.forward_all(im2.to(dev), [], True)
        np.random.seed(0)
        fine, _, _ = net.match_from_feats(f1, f2, 2, ptmax=400)
    return fine[0].reshape(-1, 4).double().contiguous()


def scene_rows(kind, n, dev):
    from patch2pix_b200.synth import synthetic_two_view
    sc = synthetic_two_view(0, n, 0.5, 0.5, planar=kind == 'H')
    return torch.from_numpy(np.concatenate([sc['pts1'], sc['pts2']], 1)).to(dev)


def plane_rows(n, dev):
    from patch2pix_b200.synth import OFF_PLANE, synthetic_dominant_plane
    sc = synthetic_dominant_plane(0, n, 0.3, 0.08, 0.5)
    return torch.from_numpy(np.concatenate([sc['pts1'], sc['pts2']], 1)).to(dev), sc['label'] == OFF_PLANE


def time_one(kind, rows, calls, cpu_reps, off=None):
    from patch2pix_b200 import _lib
    from patch2pix_b200 import verify as V
    th, n = TH[kind], int(rows.shape[0])
    h = _lib.default_handle(rows.device)
    out = torch.empty(V.out_size(n), dtype=torch.float64, device=rows.device)
    model = MODEL[kind]
    for _ in range(5):
        V.find_model_into(h, model, rows, 4, n, None, th, 0.999, 10000, 0, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        V.find_model_into(h, model, rows, 4, n, None, th, 0.999, 10000, 0, out)
    e1.record()
    torch.cuda.synchronize()
    _, mask = V.parse_host(out.cpu().numpy(), n)
    res = {'rows': n, 'ms_gpu': e0.elapsed_time(e1) / calls, 'inliers_gpu': int(mask.sum()), 'ms_cpu': None,
           'inliers_cpu': None}
    if off is not None:
        res['off_plane_recall_gpu'] = float(mask[off].mean())
    try:
        import cv2
    except ImportError:
        return res
    pts = rows.cpu().numpy()
    p1, p2 = pts[:, :2].copy(), pts[:, 2:].copy()
    if kind in ('F', 'DEGENSAC'):
        run = lambda: cv2.findFundamentalMat(p1, p2, cv2.USAC_ACCURATE, th, 0.999, 10000)
    else:
        run = lambda: cv2.findHomography(p1, p2, cv2.RANSAC, th, maxIters=10000, confidence=0.999)
    _, cm = run()
    t0 = time.perf_counter()
    for _ in range(cpu_reps):
        run()
    res.update(ms_cpu=(time.perf_counter() - t0) * 1e3 / cpu_reps, inliers_cpu=None if cm is None else int(cm.sum()))
    if off is not None and cm is not None:
        res['off_plane_recall_cpu'] = float(cm.ravel()[off].astype(bool).mean())
    return res


def time_pose(rows, calls, cpu_reps):
    from patch2pix_b200 import _lib
    from patch2pix_b200 import pose as P
    n = int(rows.shape[0])
    K = np.array([[500.0, 0, 320.0], [0, 500.0, 240.0], [0, 0, 1]])
    intr = P.intrinsics(K, K)
    h = _lib.default_handle(rows.device)
    out = torch.zeros(P.out_size(n), dtype=torch.float64, device=rows.device)

    def run_gpu():
        P.find_essential_into(h, rows, 4, n, None, intr, 1.0, 0.999, 1000, 0, out)
        P.recover_pose_into(h, rows, 4, n, None, intr, out.data_ptr(), out.data_ptr() + 184, out)
    for _ in range(5):
        run_gpu()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        run_gpu()
    e1.record()
    torch.cuda.synchronize()
    _, emask, n_good, _, _, _ = P.parse_host(out.cpu().numpy(), n)
    res = {'rows': n, 'ms_gpu': e0.elapsed_time(e1) / calls, 'inliers_gpu': int(emask.sum()), 'good_gpu': n_good,
           'ms_cpu': None, 'inliers_cpu': None, 'good_cpu': None}
    try:
        import cv2
    except ImportError:
        return res
    pts = rows.cpu().numpy()
    p1, p2 = pts[:, :2].copy(), pts[:, 2:].copy()

    def run_cpu():
        E, m = cv2.findEssentialMat(p1, p2, K, cv2.RANSAC, 0.999, 1.0, maxIters=1000)
        if E is None or E.shape[0] != 3:
            return m, 0
        inl = np.where(m.ravel() > 0)[0]
        return m, cv2.recoverPose(E, p1[inl], p2[inl], K)[0]
    cm, good = run_cpu()
    t0 = time.perf_counter()
    for _ in range(cpu_reps):
        run_cpu()
    res.update(ms_cpu=(time.perf_counter() - t0) * 1e3 / cpu_reps, inliers_cpu=None if cm is None else int(cm.sum()),
               good_cpu=int(good))
    return res


def batch_pairs(kind, count, seed=0):
    from patch2pix_b200.synth import synthetic_dominant_plane, synthetic_two_view
    sizes = np.random.default_rng(seed).integers(300, 3201, count)
    out = []
    for k, n in enumerate(sizes):
        if kind == 'DEGENSAC':
            sc = synthetic_dominant_plane(1000 + k, int(n), 0.3, 0.08, 0.5)
        else:
            sc = synthetic_two_view(1000 + k, int(n), 0.4, 0.5, planar=kind == 'H')
        out.append(np.concatenate([sc['pts1'], sc['pts2']], 1))
    return out


def _events(fn, calls):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def time_batch(kind, count, calls, dev):
    """The K back-to-back single-pair calls against one batched call on the same device rows."""
    from patch2pix_b200 import _lib
    from patch2pix_b200 import pose as P
    from patch2pix_b200 import verify as V
    pairs = batch_pairs('F' if kind in ('E', 'E+pose') else kind, count)
    n = np.array([p.shape[0] for p in pairs])
    offsets = np.concatenate(([0], np.cumsum(n))).astype(np.int64)
    K, N = count, int(offsets[-1])
    rows = torch.from_numpy(np.concatenate(pairs)).to(dev)
    offs = torch.from_numpy(offsets).to(dev)
    views = [rows[offsets[k]:offsets[k + 1]] for k in range(K)]
    h = _lib.default_handle(dev)
    res = {'pairs': K, 'rows_total': N}
    if kind in ('F', 'H', 'DEGENSAC'):
        model, th = MODEL[kind], TH[kind]
        single = [torch.zeros(V.out_size(int(v)), dtype=torch.float64, device=dev) for v in n]
        batch = torch.zeros(V.batch_out_size(K, N), dtype=torch.float64, device=dev)
        b = batch.data_ptr()

        def run_single():
            for k in range(K):
                V.find_model_into(h, model, views[k], 4, int(n[k]), None, th, 0.999, 10000, 0, single[k])

        def run_batch():
            V.find_model_batch_into(h, model, rows, 4, offs, offsets, None, th, 0.999, 10000, 0, b,
                                    b + 8 * (9 * K + (K + 1) // 2), b + 72 * K)
        res['ms_single'], res['ms_batch'] = _events(run_single, calls), _events(run_batch, calls)
        got = V.parse_batch_host(batch.cpu().numpy(), offsets)
        want = [V.parse_host(o.cpu().numpy(), int(v)) for o, v in zip(single, n)]
        res['identical'] = all((g[0] is None) == (w[0] is None) and (g[0] is None or g[0].tobytes() == w[0].tobytes())
                               and np.array_equal(g[1], w[1]) for g, w in zip(got, want))
        res['inliers'] = int(sum(int(g[1].sum()) for g in got))
    else:
        pose = kind == 'E+pose'
        Kc = np.array([[500.0, 0, 320.0], [0, 500.0, 240.0], [0, 0, 1]])
        intr = P.intrinsics(Kc, Kc)
        intr_d = torch.from_numpy(np.tile(np.asarray(intr), (K, 1))).to(dev)
        single = [torch.zeros(P.out_size(int(v)), dtype=torch.float64, device=dev) for v in n]
        batch = torch.zeros(P.batch_out_size(K, N), dtype=torch.float64, device=dev)
        pp = P._batch_ptrs(batch, K, N)

        def run_single():
            for k in range(K):
                P.find_essential_into(h, views[k], 4, int(n[k]), None, intr, 1.0, 0.999, 1000, 0, single[k])
                if pose:
                    o = single[k].data_ptr()
                    P.recover_pose_into(h, views[k], 4, int(n[k]), None, intr, o, o + 184, single[k])

        def run_batch():
            P.find_essential_batch_into(h, rows, 4, offs, offsets, None, intr_d.data_ptr(), 1.0, 0.999, 1000, 0, pp['E'],
                                        pp['emask'], pp['cnt'])
            if pose:
                P.recover_pose_batch_into(h, rows, 4, offs, offsets, None, intr_d.data_ptr(), pp['E'], pp['emask'],
                                          pp['Rt'], pp['pmask'], pp['good'])
        res['ms_single'], res['ms_batch'] = _events(run_single, calls), _events(run_batch, calls)
        got = P._parse_batch(batch.cpu().numpy(), offsets, K, N)
        want = [P.parse_host(o.cpu().numpy(), int(v)) for o, v in zip(single, n)]
        keep = slice(0, 6) if pose else slice(0, 2)
        res['identical'] = all(all(np.asarray(a).tobytes() == np.asarray(b_).tobytes() if a is not None else b_ is None
                                   for a, b_ in zip(g[keep], w[keep])) for g, w in zip(got, want))
        res['inliers'] = int(sum(int(g[1].sum()) for g in got))
    res['speedup'] = res['ms_single'] / res['ms_batch']
    res['ms_cpu'] = None
    try:
        import cv2
    except ImportError:
        return res
    t0 = time.perf_counter()
    for p in pairs:
        p1, p2 = p[:, :2].copy(), p[:, 2:].copy()
        if kind in ('F', 'DEGENSAC'):
            cv2.findFundamentalMat(p1, p2, cv2.USAC_ACCURATE, TH[kind], 0.999, 10000)
        elif kind == 'H':
            cv2.findHomography(p1, p2, cv2.RANSAC, TH[kind], maxIters=10000, confidence=0.999)
        else:
            E, m = cv2.findEssentialMat(p1, p2, Kc, cv2.RANSAC, 0.999, 1.0, maxIters=1000)
            if pose and E is not None and E.shape[0] == 3:
                inl = np.where(m.ravel() > 0)[0]
                cv2.recoverPose(E, p1[inl], p2[inl], Kc)
    res['ms_cpu'] = (time.perf_counter() - t0) * 1e3
    return res


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--cpu-reps', type=int, default=20)
    ap.add_argument('--batch-pairs', type=int, default=256)
    ap.add_argument('--batch-calls', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError('bench_verify.py needs a CUDA device: there is no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device())
    fine = fine_matches(dev)
    line = {'metric': 'ms per verification call', 'card': card(), 'cpu_cores': os.cpu_count(),
            'config': {'th_px': TH, 'conf': 0.999, 'max_iters': 10000, 'seed': 0, 'calls': args.calls,
                       'cpu_reps': args.cpu_reps, 'cpu': 'cv2.findFundamentalMat USAC_ACCURATE (F, DEGENSAC) / cv2.findHomography RANSAC',
                       'E': {'th_px': 1.0, 'max_iters': 1000, 'K': 'focal 500 px, principal point (320, 240)',
                             'cpu': 'cv2.findEssentialMat RANSAC + cv2.recoverPose'}}}
    for kind in ('F', 'H'):
        line[kind] = {'fine': time_one(kind, fine, args.calls, args.cpu_reps),
                      'scene': time_one(kind, scene_rows(kind, fine.shape[0], dev), args.calls, args.cpu_reps)}
    prow, off = plane_rows(fine.shape[0], dev)
    line['DEGENSAC'] = {'fine': time_one('DEGENSAC', fine, args.calls, args.cpu_reps),
                        'plane': time_one('DEGENSAC', prow, args.calls, args.cpu_reps, off)}
    line['E'] = {'fine': time_pose(fine, args.calls, args.cpu_reps),
                 'scene': time_pose(scene_rows('E', fine.shape[0], dev), args.calls, args.cpu_reps)}
    if args.batch_pairs > 0:
        line['batch'] = {kind: time_batch(kind, args.batch_pairs, args.batch_calls, dev)
                         for kind in ('F', 'H', 'DEGENSAC', 'E', 'E+pose')}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
