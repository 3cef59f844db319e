"""Time the overlap precompute (patch2pix_b200.evaluation.sav_model_multi_ov_pairs) on a seeded COLMAP scene.

    python bench_ovs.py [--images 2500] [--keypoints 8000] [--host-images 300] [--reps 3] [--out DIR]

Writes a seeded images.bin (synth.synthetic_overlap_images: every image with --keypoints keypoints, a triangulated
fraction drawn per image from U(0.2, 0.6)) under DIR (a temporary directory by default, removed at the end) and times:
  - parse: images.bin with its 2D points (the host part);
  - upload: the flat point3D_ids and offsets to the device;
  - kernels: p2p_overlap_scores (pack + count), CUDA events over --reps launches;
  - pairs: the [T, N, N] masks, one torch.nonzero and the copy of its rows, for the five default thresholds;
  - sav_model_multi_ov_pairs end to end, from no ov_pairs.npy to the saved file, host clock, best of --reps.
On the first --host-images images it also times the reference's host loop (oracle/overlap_oracle.py: the
np.intersect1d double loop and the pair rule) and checks that the device's pair lists equal it.  Prints one JSON line
with the card and its power limit (nvidia-smi, read-only query).
"""
import argparse
import contextlib
import ctypes as C
import io
import json
import os
import shutil
import subprocess
import tempfile
import time

import numpy as np
import torch

from oracle import overlap_oracle as O
from patch2pix_b200 import _lib
from patch2pix_b200 import evaluation as E
from patch2pix_b200.synth import synthetic_overlap_images, write_colmap_model

OVERLAPS = [0.1, 0.2, 0.3, 0.4, 0.5]
CAMERA = [(1, 0, 1600, 1200, [1200.0, 800.0, 600.0])]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def quiet(fn, *a):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a)


def sync_clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def bench_scene(model_dir, reps):
    path = os.path.join(model_dir, 'images.bin')
    images, t_parse = sync_clock(lambda: list(E._read_images(path, True, copy=False).values()))
    ids = [im.point3D_ids for im in images]
    n = len(ids)
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(a) for a in ids], out=offsets[1:])
    words = int((np.diff(offsets).max() + 31) // 32)
    (flat, off), t_upload = sync_clock(lambda: (torch.from_numpy(np.concatenate(ids)).cuda(),
                                                torch.from_numpy(offsets).cuda()))
    bits = torch.empty(n * words, dtype=torch.int32, device='cuda')
    counts = torch.empty(n, dtype=torch.int32, device='cuda')
    scores = torch.empty(n, n, dtype=torch.float64, device='cuda')
    h = _lib.default_handle('cuda')

    def launch():
        _lib.check(h.lib.p2p_overlap_scores(h.h, _lib.ptr(flat), _lib.ptr(off),
                                            offsets.ctypes.data_as(C.POINTER(C.c_int64)), n, words, _lib.ptr(bits),
                                            _lib.ptr(counts), _lib.ptr(scores), h.stream()))
    launch()                                                     # warm-up
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        launch()
    ev[1].record()
    torch.cuda.synchronize()
    t_kernels = ev[0].elapsed_time(ev[1]) / 1e3 / reps
    names = np.empty(n, dtype=object)
    names[:] = [im.name for im in images]
    E._pairs_by_threshold(names, scores, OVERLAPS)               # warm-up
    pairs, t_pairs = sync_clock(lambda: E._pairs_by_threshold(names, scores, OVERLAPS))
    del images, ids, flat, off, bits, scores
    t_sav = []
    for _ in range(reps):
        f = os.path.join(model_dir, 'ov_pairs.npy')
        if os.path.exists(f):
            os.remove(f)
        _, t = sync_clock(lambda: quiet(E.sav_model_multi_ov_pairs, model_dir, OVERLAPS))
        t_sav.append(t)
    return {'images': n, 'keypoints': int(offsets[-1]), 'parse_s': t_parse, 'upload_s': t_upload,
            'kernels_s': t_kernels, 'pairs_s': t_pairs, 'sav_model_s': min(t_sav), 'sav_model_s_all': t_sav,
            'pairs_per_threshold': [len(p) for p in pairs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=2500)
    ap.add_argument('--keypoints', type=int, default=8000)
    ap.add_argument('--host-images', type=int, default=300, help='images of the host-loop comparison (0: skip it)')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None, help='directory for the seeded models (default: a temporary directory)')
    args = ap.parse_args()
    root = args.out or tempfile.mkdtemp(prefix='bench_ovs_')
    try:
        ims = synthetic_overlap_images(args.seed, args.images, n2d=args.keypoints, frac=(0.2, 0.6))
        full = os.path.join(root, 'full')
        write_colmap_model(full, CAMERA, ims)
        res = {'card': card(), 'full': bench_scene(full, args.reps)}
        if args.host_images:
            sub = ims[:args.host_images]
            sub_dir = os.path.join(root, 'host')
            write_colmap_model(sub_dir, CAMERA, sub)
            quiet(E.sav_model_multi_ov_pairs, sub_dir, OVERLAPS)                        # warm-up
            os.remove(os.path.join(sub_dir, 'ov_pairs.npy'))
            d, t_dev = sync_clock(lambda: quiet(E.sav_model_multi_ov_pairs, sub_dir, OVERLAPS))
            t0 = time.perf_counter()
            ov, _ = O.cal_overlap_scores([im[5] for im in sub])
            names = [im[4] for im in sub]
            host = {t: O.pairs(ov, names, t) for t in OVERLAPS}
            t_host = time.perf_counter() - t0
            n = len(sub)
            res['host'] = {'images': n, 'host_loop_s': t_host, 'sav_model_s': t_dev, 'pairs_equal': host == d,
                           'host_s_per_intersect': t_host / max(n * (n - 1) // 2, 1)}
            calls = args.images * (args.images - 1) // 2
            res['host_loop_estimate_full_s'] = calls * res['host']['host_s_per_intersect']
        print(json.dumps(res), flush=True)
    finally:
        if args.out is None:
            shutil.rmtree(root, ignore_errors=True)


if __name__ == '__main__':
    main()
