"""Generate the golden data of tests/test_eval_host.py by running the reference's own code on the CPU.

Run where the reference checkout is available (it does not travel with this repository):
    python tests/golden/make_eval_golden.py [/path/to/reference]
Writes tests/golden/eval_colmap/{cameras,images}.bin (a small COLMAP model written with the reference's
utils/colmap/read_write_model.py writers) and tests/golden/eval_golden.npz: the reference's load_model_ims output for
that model and the outputs of its check_inliers_distr / check_data_hist (utils/eval/measure.py:115-161) on seeded
lists of distances.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
sys.path.insert(0, REF)

from utils.colmap import read_write_model as rw                    # noqa: E402
from utils.colmap.data_loading import load_model_ims               # noqa: E402
from utils.eval.measure import check_data_hist, check_inliers_distr  # noqa: E402

EVAL_BINS = [0, 1e-2, 1, 5, 10, 25, 50, 100, 2500, 1e5]
DEFAULT_BINS = [0, 1e-2, 1, 5, 10, 25, 50, 100, 400, 2500, 1e5]


def write_model(out_dir, rng):
    """Four supported camera models and one unused OPENCV camera; images with unit and non-unit qvecs, 0 and many 2D
    points, and one whose camera is absent."""
    os.makedirs(out_dir, exist_ok=True)
    cams = {
        1: rw.Camera(id=1, model='SIMPLE_PINHOLE', width=1024, height=768, params=np.array([812.5, 512.25, 383.75])),
        2: rw.Camera(id=2, model='PINHOLE', width=800, height=600, params=np.array([701.125, 699.5, 400.5, 300.25])),
        5: rw.Camera(id=5, model='SIMPLE_RADIAL', width=1600, height=1200,
                     params=np.array([1199.91, 800.0, 600.0, -0.0324314])),
        7: rw.Camera(id=7, model='RADIAL', width=640, height=480, params=np.array([525.0, 319.5, 239.5, 0.01, -0.002])),
        9: rw.Camera(id=9, model='OPENCV', width=320, height=240, params=rng.uniform(-1, 1, 8)),
    }
    ims = {}
    cam_of = [1, 2, 5, 7, 1, 2, 42, 5]                  # 42: absent camera
    for k, cid in enumerate(cam_of):
        q = rng.normal(size=4)
        if k % 2 == 0:
            q /= np.linalg.norm(q)                      # odd k keep a non-unit qvec
        n2d = [0, 1, 1000, 5, 0, 250, 7, 2][k]
        ims[10 + 3 * k] = rw.Image(id=10 + 3 * k, qvec=q, tvec=rng.normal(scale=3.0, size=3), camera_id=cid,
                                   name=f'scene_{k:02d}/img_{k}.jpg', xys=rng.uniform(0, 1000, (n2d, 2)),
                                   point3D_ids=rng.integers(-1, 10 ** 6, n2d))
    rw.write_cameras_binary(cams, os.path.join(out_dir, 'cameras.bin'))
    rw.write_images_binary(ims, os.path.join(out_dir, 'images.bin'))


def dist_cases(rng):
    """Lists of per-pair distances: empty list, empty per-pair arrays, values on every edge, above 1e5, NaN, inf."""
    edges = np.array(EVAL_BINS + DEFAULT_BINS, dtype=np.float64)
    cases = [
        [],
        [np.array([])],
        [np.array([]), np.array([])],
        [rng.lognormal(1.0, 3.0, 200) for _ in range(5)],
        [np.array([]), rng.lognormal(0.0, 4.0, 50), np.array([]), rng.lognormal(2.0, 2.0, 7)],
        [edges, np.concatenate([edges, [1e5 * (1 + 1e-15), 2e5, 1e9, np.inf, np.nan, np.nan]]), rng.uniform(0, 1, 3)],
        [np.nextafter(edges, np.inf), np.nextafter(edges, -np.inf)],
        [rng.lognormal(1.0, 3.0, 1000), np.array([np.nan]), np.array([3.0])],
    ]
    return cases


def run(fn, *a, **kw):
    try:
        return fn(*a, **kw)
    except Exception as e:                               # the reference raises on some inputs; that is recorded too
        return {'raises': type(e).__name__}


def main():
    rng = np.random.default_rng(20261015)
    model_dir = os.path.join(HERE, 'eval_colmap')
    write_model(model_dir, rng)
    out = {}
    ims = load_model_ims(model_dir)
    out['im_names'] = np.array(list(ims.keys()))
    for f in ('K', 'c', 'q', 'R'):
        out['im_' + f] = np.stack([getattr(v, f) for v in ims.values()])
    out['im_id'] = np.array([v.id for v in ims.values()])
    results = []
    cases = dist_cases(rng)
    for i, case in enumerate(cases):
        out[f'case{i}_len'] = np.array(len(case))
        for j, d in enumerate(case):
            out[f'case{i}_{j}'] = d
        res = {}
        for bname, bins in (('eval', EVAL_BINS), ('default', DEFAULT_BINS)):
            res[f'distr_{bname}'] = run(check_inliers_distr, case, bins=bins, tag='fdist')
            r = run(check_inliers_distr, case, bins=bins, tag='indist', return_ratios=True)
            res[f'distr_ratios_{bname}'] = r if isinstance(r, dict) else [None if r[0] is None else
                                                                           [float(v) for v in r[0]], r[1]]
            res[f'hist_{bname}'] = run(check_data_hist, case, bins, tag='qt')
        res['distr_default_call'] = run(check_inliers_distr, case)
        results.append(res)
    out['results_json'] = np.array(json.dumps(results))
    np.savez(os.path.join(HERE, 'eval_golden.npz'), **out)
    print('wrote', model_dir, 'and eval_golden.npz with', len(cases), 'distance cases')


if __name__ == '__main__':
    main()
