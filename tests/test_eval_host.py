"""Host side of patch2pix_b200.evaluation: the COLMAP reader and the histogram summaries against the reference's own
outputs (tests/golden/make_eval_golden.py), the counts-based summary, pair selection and record parsing."""
import json
import os
import shutil
import struct
import warnings
from argparse import Namespace

import numpy as np
import pytest

from patch2pix_b200 import evaluation as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
MODEL = os.path.join(GOLDEN, 'eval_colmap')
DEFAULT_BINS = [0, 1e-2, 1, 5, 10, 25, 50, 100, 400, 2500, 1e5]


@pytest.fixture(scope='module')
def golden():
    z = np.load(os.path.join(GOLDEN, 'eval_golden.npz'))
    cases = [[z[f'case{i}_{j}'] for j in range(int(z[f'case{i}_len']))]
             for i in range(sum(1 for k in z.files if k.endswith('_len')))]
    return z, cases, json.loads(str(z['results_json']))


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def test_load_model_ims_matches_reference(golden):
    z = golden[0]
    ims = E.load_model_ims(MODEL)
    assert list(ims) == list(z['im_names'])                 # file order, the image with an absent camera skipped
    for k, im in enumerate(ims.values()):
        for f in ('K', 'c', 'q', 'R'):
            assert _same(getattr(im, f), z['im_' + f][k]), (im.name, f)
        assert im.id == int(z['im_id'][k]) and im.name == z['im_names'][k]


def test_reader_fields():
    cams = E.read_cameras_binary(os.path.join(MODEL, 'cameras.bin'))
    assert [c.model for c in cams.values()] == ['SIMPLE_PINHOLE', 'PINHOLE', 'SIMPLE_RADIAL', 'RADIAL', 'OPENCV']
    assert [len(c.params) for c in cams.values()] == [3, 4, 4, 5, 8]
    assert (cams[5].width, cams[5].height) == (1600, 1200)
    images = E.read_images_binary(os.path.join(MODEL, 'images.bin'))
    assert len(images) == 8 and images[28].camera_id == 42          # the image whose camera is absent is read
    with pytest.raises(ValueError):
        E.cam_params_to_matrix(cams[9].params, 'OPENCV')


def _truncations(path):
    size = os.path.getsize(path)
    return sorted({1, 7, 8, 9, 20, 40, 64, 70, 71, 73, size // 3, size // 2, size - 25, size - 1} & set(range(size)))


@pytest.mark.parametrize('name', ['cameras.bin', 'images.bin'])
def test_truncated_model_raises(tmp_path, name):
    src = os.path.join(MODEL, name)
    data = open(src, 'rb').read()
    other = 'images.bin' if name == 'cameras.bin' else 'cameras.bin'
    shutil.copy(os.path.join(MODEL, other), tmp_path / other)
    for cut in _truncations(src):
        (tmp_path / name).write_bytes(data[:cut])
        with pytest.raises(ValueError):
            E.load_model_ims(str(tmp_path))


def test_name_without_terminator_raises(tmp_path):
    blob = struct.pack('<Q', 1) + struct.pack('<i7di', 1, 1, 0, 0, 0, 0, 0, 0, 1) + b'no_nul.jpg'
    (tmp_path / 'images.bin').write_bytes(blob)
    with pytest.raises(ValueError):
        E.read_images_binary(str(tmp_path / 'images.bin'))


def _call(fn, *a, **kw):
    try:
        r = fn(*a, **kw)
    except Exception as e:
        return {'raises': type(e).__name__}
    if isinstance(r, tuple):
        return [None if r[0] is None else [float(v) for v in r[0]], r[1]]
    return r


def test_summaries_match_reference(golden):
    _, cases, results = golden
    with warnings.catch_warnings():         # the reference's means of empty lists warn; outputs are compared
        warnings.simplefilter('ignore')
        for case, res in zip(cases, results):
            for bname, bins in (('eval', E.EVAL_BINS), ('default', DEFAULT_BINS)):
                assert _call(E.check_inliers_distr, case, bins=bins, tag='fdist') == res[f'distr_{bname}']
                assert _call(E.check_inliers_distr, case, bins=bins, tag='indist', return_ratios=True) == \
                    res[f'distr_ratios_{bname}']
                assert _call(E.check_data_hist, case, bins, tag='qt') == res[f'hist_{bname}']
            assert _call(E.check_inliers_distr, case) == res['distr_default_call']


def test_counts_helper_equals_list_helper(golden):
    _, cases, _ = golden
    rng = np.random.default_rng(3)
    cases = cases + [[rng.lognormal(1.0, 3.0, int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 9)))]
                     for _ in range(30)]
    with warnings.catch_warnings():         # the reference's means of empty lists warn; outputs are compared
        warnings.simplefilter('ignore')
        for case in cases:
            for bins in (E.EVAL_BINS, DEFAULT_BINS):
                counts = [np.append(np.histogram(d, bins)[0], len(d)).astype(np.int32) for d in case]
                for rr in (False, True):
                    assert _call(E.inliers_distr_from_counts, counts, bins, 'x', rr) == \
                        _call(E.check_inliers_distr, case, bins, 'x', rr)


def _tree(root, scenes):
    for scene, pairs in scenes.items():
        d = os.path.join(root, scene, 'dense', 'sparse')
        os.makedirs(d)
        shutil.copy(os.path.join(MODEL, 'cameras.bin'), d)
        shutil.copy(os.path.join(MODEL, 'images.bin'), d)
        np.save(os.path.join(d, 'ov_pairs.npy'), {0.3: pairs, 0.5: pairs[:3]})


def test_pair_selection_rule(tmp_path):
    """The reference's rule restated: one np.random.seed(0), scenes in os.listdir order, a shuffle (the permutation
    np.random draws for that length) only for scenes with more than sample_max pairs."""
    scenes = {f's{k}': [(f'a{k}_{i}.jpg', f'b{k}_{i}.jpg') for i in range(n)]
              for k, n in enumerate([12, 5, 30, 7, 8])}
    _tree(str(tmp_path), scenes)
    sample_max = 7
    np.random.seed(0)
    got = E.select_pairs(str(tmp_path), sample_max, 0.3)
    np.random.seed(0)
    expect = []
    for scene in os.listdir(str(tmp_path)):
        pairs = scenes[scene]
        if len(pairs) > sample_max:
            pairs = [pairs[i] for i in np.random.permutation(len(pairs))[:sample_max]]
        expect.append((scene, pairs))
    assert [(s, [tuple(p) for p in ps]) for s, _, ps in got] == expect
    assert [len(ps) for _, ps in expect] == [min(len(scenes[s]), sample_max) for s, _ in expect]
    assert all(set(ims) == set(E.load_model_ims(MODEL)) for _, ims, _ in got)


def _row(N, count, R, t, counts):
    row = np.zeros(E._rec_len(counts.shape[1]))
    row[0] = N
    row[10:11].view(np.int32)[0] = count
    row[11:20] = np.asarray(R).reshape(9)
    row[20:23] = np.asarray(t).reshape(3)
    row[E._REC_POSE:].view(np.int32)[:counts.size] = counts.reshape(-1)
    return row


def test_parse_record_classification():
    from patch2pix_b200 import pose as P
    ne = len(E.EVAL_BINS)
    counts = np.arange(3 * ne, dtype=np.int32).reshape(3, ne)
    q = np.array([0.9, 0.1, -0.3, 0.2])
    q = q / np.linalg.norm(q)
    R = P.quat2mat(q)
    t = np.array([0.3, -0.2, 0.9])
    for bad in (0, -1):
        r = E.parse_record(_row(40, bad, R, t, counts), t, q)
        assert r.status == 'geo_failed' and r.N == 40 and np.array_equal(r.counts, counts) and r.terr is None
    r = E.parse_record(_row(40, 17, R, t, counts), t, q)
    assert r.status == 'ok' and r.n_inls == counts[2, -1] and r.terr < 1e-4 and r.qerr < 1e-4
    assert E.parse_record(None, t, q).status == 'match_failed'


def test_summarize_equals_list_based_lines():
    """summarize on records equals the reference's closing lines computed from the distance lists."""
    rng = np.random.default_rng(5)
    ne = len(E.EVAL_BINS)
    records, cd, fd, ind, qt, nm, irat = [], [], [], [], [], [], []
    for k in range(12):
        st = ['ok', 'ok', 'geo_failed', 'match_failed'][k % 4]
        if st == 'match_failed':
            records.append(E.parse_record(None, None, None))
            continue
        N = int(rng.integers(0, 60)) if st == 'geo_failed' else int(rng.integers(5, 60))
        c, f = rng.lognormal(2, 3, N), rng.lognormal(1, 3, N)
        mask = rng.random(N) < 0.6
        mask[0] = True
        counts = np.stack([np.append(np.histogram(x, E.EVAL_BINS)[0], len(x)) for x in (c, f, f[mask])])
        cd.append(c)
        fd.append(f)
        nm.append(N)
        if st == 'ok':
            terr, qerr = rng.uniform(0, 12, 2)
            records.append(Namespace(status='ok', N=N, n_inls=int(mask.sum()), counts=counts, terr=terr, qerr=qerr))
            ind.append(f[mask])
            qt.append(max(terr, qerr))
            irat.append(mask.sum() / N)
        else:
            records.append(Namespace(status='geo_failed', N=N, n_inls=None, counts=counts, terr=None, qerr=None))
    lines, mean, pr = E.summarize(records, 1.25)
    expect = [f'Pairs 12 match_failed=3 geo_failed=3 num_matches={np.mean(nm):.2f} irat={np.mean(irat):.3f} '
              f'time:1.25s',
              E.check_inliers_distr(cd, bins=E.EVAL_BINS, tag='cdist'),
              E.check_inliers_distr(fd, bins=E.EVAL_BINS, tag='fdist', return_ratios=True)[1],
              E.check_inliers_distr(ind, bins=E.EVAL_BINS, tag='indist', return_ratios=True)[1]]
    pass_rate = np.array([100.0 * np.mean(np.array(qt) < thre) for thre in range(1, 11, 1)])
    expect.append('Pose err: qt_mean={:.2f}/{:.2f} qt<[1-10]deg:{}'.format(np.mean(qt), np.median(qt), pass_rate))
    assert lines == expect and mean == np.mean(qt) and np.array_equal(pr, pass_rate)



def test_eval_kernel_compiles_without_spills(tmp_path):
    import re
    import subprocess
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'eval.cu'), '-o', str(tmp_path / 'e.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    found = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', r.stdout + r.stderr)
    spills = [int(st) + int(ld) for st, ld in found]
    assert spills == [0], spills                  # one kernel, no spills
