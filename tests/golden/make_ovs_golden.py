"""Generate the golden data of tests/test_overlap_host.py and tests/test_gpu_overlap.py by running the reference's own
code on the CPU.

Run where a checkout of the reference (GrumpyZhou/patch2pix) is available; it does not travel with this repository:
    python tests/golden/make_ovs_golden.py /path/to/reference
Writes small COLMAP models under tests/golden/ovs_colmap/<case>/images.bin with the reference's
utils/colmap/read_write_model.py writer, and tests/golden/ovs_golden.npz with, per case, the reference's
read_images_binary point ids and xys, cal_overlap_scores matrix and counts (or the exception it raises), the pair lists
of load_model_ov_pairs' rule for a set of thresholds, and the dicts and printed lines of sav_model_multi_ov_pairs for a
fresh directory, a duplicated key, a complete file and an incomplete file.
"""
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1]
sys.path.insert(0, REF)

from utils.colmap import read_write_model as rw                                   # noqa: E402
from utils.colmap import data_loading as dl                                       # noqa: E402

THRESHOLDS = [-0.5, 0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.8, 1.0, float('nan')]
BIG = 2 ** 40


def _ids(rng, n2d, valid, pool=(1, BIG, 7, 123456)):
    """n2d ids: a positive id from `pool` at the indices in `valid`, -1 or 0 elsewhere."""
    ids = rng.choice([-1, 0], n2d)
    for k in valid:
        ids[k] = pool[k % len(pool)]
    return ids


def edge_case(rng):
    """Every n2d around the 32-bit word boundaries, ids -1 / 0 / 1 / 2^40, one image without a valid index, two
    identical sets and the exact ratios 3/10 and 1/5; image ids and names not in file order."""
    sets = [
        (0, []),                                          # no valid index (the only one)
        (1, [0]),
        (31, list(range(0, 31, 2))),
        (32, [0, 1, 2, 31]),
        (33, [32] + list(range(10))),
        (63, list(range(0, 63, 3))),
        (64, list(range(64))),
        (65, [0, 5, 31, 32, 33, 63, 64]),
        (65, [0, 5, 31, 32, 33, 63, 64]),                # the same set as the one before: overlap exactly 1
        (1000, sorted(rng.choice(1000, 400, replace=False).tolist())),
        (10, list(range(10))),                            # with the next one: 3 / 10
        (40, [0, 1, 2]),
        (200, [100, 101, 102, 103, 104]),                 # with the next one: 1 / 5
        (105, [104]),
    ]
    names = ['m.jpg', 'b/2.jpg', 'b/10.jpg', 'Z.png', 'a', 'zz.jpg', 'a.jpg', 'c1.jpg', 'c2.jpg', 'big.jpg', 'p10',
             'p3', 'q200', 'q105']
    iids = [17, 3, 99, 4, 5, 60, 7, 8, 1, 10, 11, 2, 13, 14]
    return [(iid, name, _ids(rng, n2d, valid, pool=(1, BIG) if k % 2 else (BIG, 1)))
            for k, (iid, name, (n2d, valid)) in enumerate(zip(iids, names, sets))]


def random_case(rng, n=40):
    out = []
    for k in range(n):
        n2d = int(rng.integers(40, 200))
        p = rng.uniform(0.1, 0.9)
        valid = np.nonzero(rng.uniform(size=n2d) < p)[0]
        out.append((1000 - 7 * k, f'img_{rng.integers(0, 10 ** 4):04d}_{k}.jpg', _ids(rng, n2d, valid)))
    return out


def write(case_dir, images, rng):
    os.makedirs(case_dir, exist_ok=True)
    ims = {}
    for iid, name, ids in images:
        xys = rng.integers(0, 4096, (len(ids), 2)) + rng.choice([0.0, 0.5, 0.25], (len(ids), 2))
        ims[iid] = rw.Image(id=iid, qvec=np.array([1.0, 0, 0, 0]), tvec=np.zeros(3), camera_id=1, name=name, xys=xys,
                            point3D_ids=np.asarray(ids, dtype=np.int64))
    rw.write_images_binary(ims, os.path.join(case_dir, 'images.bin'))


def captured(fn, *a):
    buf = io.StringIO()
    try:
        with contextlib.redirect_stdout(buf):
            res = fn(*a)
    except Exception as e:                                # the reference raises on some inputs; that is recorded too
        return {'raises': type(e).__name__}, buf.getvalue().splitlines()
    return res, buf.getvalue().splitlines()


def as_json(d):
    return d if 'raises' in d else [[repr(k), [list(p) for p in v]] for k, v in d.items()]


def main():
    rng = np.random.default_rng(20261016)
    cases = {
        'edge': edge_case(rng),
        'random40': random_case(rng),
        'two_empty': [(1, 'x.jpg', np.array([-1, 0, -1])), (2, 'y.jpg', np.zeros(0, np.int64)),
                      (3, 'w.jpg', np.array([5, 6]))],
        'one': [(5, 'solo.jpg', np.array([0, 3, -1, 9]))],
        'zero': [],
    }
    root = os.path.join(HERE, 'ovs_colmap')
    shutil.rmtree(root, ignore_errors=True)
    out, results = {}, {}
    for case, images in cases.items():
        case_dir = os.path.join(root, case)
        write(case_dir, images, rng)
        ims = rw.read_images_binary(os.path.join(case_dir, 'images.bin'))
        out[f'{case}_n'] = np.array(len(ims))
        for k, im in enumerate(ims.values()):
            out[f'{case}_ids_{k}'] = im.point3D_ids
            out[f'{case}_xys_{k}'] = im.xys
        res = {'names': [im.name for im in ims.values()], 'image_ids': list(ims)}
        sc, _ = captured(dl.cal_overlap_scores, list(ims), ims)
        if isinstance(sc, dict):
            res['cal_overlap_scores'] = sc
        else:
            out[f'{case}_ov'], out[f'{case}_nums'] = sc
            names = [im.name for im in ims.values()]
            res['pairs'] = {repr(t): [list(p) for p in np.vstack(np.where((sc[0] >= t) & (sc[0] < 1))).T.tolist()]
                            for t in THRESHOLDS}
            res['pair_names'] = {repr(t): [[max(names[i], names[j]), min(names[i], names[j])]
                                           for i, j in res['pairs'][repr(t)]] for t in THRESHOLDS}
        with tempfile.TemporaryDirectory() as tmp:
            shutil.copy(os.path.join(case_dir, 'images.bin'), tmp)
            runs = []
            for overlaps in ([0.1, 0.3, 0.3, 0.5], [0.3, 0.1], [0.2, 0.3, 0.2]):   # fresh+dup, complete, incomplete
                d, lines = captured(dl.sav_model_multi_ov_pairs, tmp, overlaps)
                runs.append({'overlaps': overlaps, 'dict': as_json(d), 'lines': lines,
                             'file': as_json(np.load(os.path.join(tmp, 'ov_pairs.npy'), allow_pickle=True).item())
                             if os.path.exists(os.path.join(tmp, 'ov_pairs.npy')) else None})
            res['sav_model_multi_ov_pairs'] = runs
            d, lines = captured(dl.load_model_ov_pairs, tmp, 0.3)
            res['load_model_ov_pairs'] = {'pairs': d if isinstance(d, dict) else [list(p) for p in d], 'lines': lines}
        results[case] = res
    out['results_json'] = np.array(json.dumps(results))
    np.savez_compressed(os.path.join(HERE, 'ovs_golden.npz'), **out)
    print('wrote', root, 'and ovs_golden.npz with', len(cases), 'cases')


if __name__ == '__main__':
    main()
