"""The relative-pose evaluation's host side (patch2pix_b200.relpose, oracle/relpose_oracle.py): the numpy restatement of
the kernel and of the statistics on hand-made cases, the pair-list readers on synthetic files, and the CLI."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import relpose_oracle as O
from patch2pix_b200 import relpose as RP
from patch2pix_b200.synth import _rotation, synthetic_relpose_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rt(R, t):
    return np.concatenate([np.asarray(R, dtype=np.float64).reshape(9), np.asarray(t, dtype=np.float64)])


def test_identity_pose_has_zero_error():
    Rt = _rt(_rotation(np.array([0.05, -0.02, 0.03])), [0.7, 0.1, -0.2])
    cr, ct = O.pose_cosines(Rt, Rt, 10)
    assert cr == pytest.approx(1.0, abs=1e-15) and ct == pytest.approx(1.0, abs=1e-15)
    assert O.pose_errors(1.0, 1.0) == (0.0, 0.0)


@pytest.mark.parametrize('deg', [1.0, 10.0, 30.0, 90.0, 179.0])
def test_known_rotation_error(deg):
    R = _rotation(np.array([0.0, 0.0, math.radians(deg)]))
    cr, ct = O.pose_cosines(_rt(np.eye(3), [1, 0, 0]), _rt(R, [3, 0, 0]), 5)
    r_err, t_err = O.pose_errors(cr, ct)
    assert r_err == pytest.approx(deg, abs=1e-6) and t_err == 0.0


@pytest.mark.parametrize('deg,folded', [(40.0, 40.0), (90.0, 90.0), (150.0, 30.0), (180.0, 0.0)])
def test_translation_direction_error_is_folded(deg, folded):
    a = math.radians(deg)
    cr, ct = O.pose_cosines(_rt(np.eye(3), [2, 0, 0]), _rt(np.eye(3), [math.cos(a), math.sin(a), 0]), 5)
    assert O.pose_errors(cr, ct)[1] == pytest.approx(folded, abs=1e-6)


def test_no_model_gives_nan_cosines_and_inf_errors():
    Rt = _rt(np.eye(3), [1, 0, 0])
    cr, ct = O.pose_cosines(Rt, Rt, 0)
    assert math.isnan(cr) and math.isnan(ct)
    assert O.pose_errors(cr, ct) == (np.inf, np.inf)
    assert O.pose_errors(1.0, 1.0, failed=True) == (np.inf, np.inf)


def test_cosines_are_clipped():
    R = np.eye(3) * (1 + 1e-12)                    # trace slightly above 3
    cr, _ = O.pose_cosines(_rt(np.eye(3), [1, 0, 0]), _rt(R, [1, 0, 0]), 1)
    assert cr == 1.0


def test_exact_correspondences_have_zero_epipolar_error():
    # R = I, t along x: E x0 = (0, -1, v0), so x1^T E x0 = v0 - v1 = 0 exactly when the rows share y and both views
    # have the same intrinsics
    intr = np.array([500.0, 500.0, 320.0, 240.0, 500.0, 500.0, 320.0, 240.0])
    rng = np.random.default_rng(0)
    y = rng.uniform(0, 480, 200)
    rows = np.stack([rng.uniform(0, 640, 200), y, rng.uniform(0, 640, 200), y], 1)
    e = O.epipolar_errors(rows, intr, _rt(np.eye(3), [0.8, 0, 0]))
    assert np.all(e == 0.0)
    assert list(O.counts(e, [1e-12, 5e-4])) == [200, 200, 200]


def test_epipolar_errors_of_true_correspondences():
    from patch2pix_b200.synth import synthetic_two_view
    s = synthetic_two_view(3, 300, 0.3, 0.0, focal2=430.0)
    intr = np.array([500.0, 500.0, 320.0, 240.0, 430.0, 430.0, 320.0, 240.0])
    e = O.epipolar_errors(np.concatenate([s['pts1'], s['pts2']], 1), intr, _rt(s['R'], s['t']))
    assert np.all(e[s['inlier']] < 1e-20) and np.median(e[~s['inlier']]) > 1e-3
    c = O.counts(e, [5e-4])
    assert c[1] == 300 and c[0] >= s['inlier'].sum()


def test_auc_hand_made():
    # one pair at 2.5 degrees: the recall curve is (0, 0) -> (2.5, 1) -> (5, 1)
    assert O.pose_auc([2.5], [5])[5] == 0.75
    # errors exactly at a threshold fall outside it
    a = O.pose_auc([5.0, 5.0, 10.0], [5, 10, 20])
    assert a[5] == 0.0
    assert a[10] == pytest.approx((5 / 6 + 10 / 3) / 10)          # (0, 0) (5, 1/3) (5, 2/3) (10, 2/3)
    assert a[20] == pytest.approx((5 / 6 + 25 / 6 + 10) / 20)     # ... (10, 1) (20, 1)
    assert O.pose_auc([0.0, 0.0], [5])[5] == 1.0
    assert O.pose_auc([np.inf] * 4, [5, 10, 20]) == {5: 0.0, 10: 0.0, 20: 0.0}
    assert all(math.isnan(v) for v in O.pose_auc([], [5, 10]).values())
    rng = np.random.default_rng(1)
    errs = np.concatenate([rng.exponential(6.0, 50), [np.inf] * 7, [5.0, 10.0]])
    assert RP.pose_auc(errs, [5, 10, 20]) == O.pose_auc(errs, [5, 10, 20])


def test_precision():
    rows = [[3, 4, 10], [0, 0, 0], [1, 2, 2]]
    assert O.precision(rows, [1e-4, 5e-4]) == {1e-4: pytest.approx((0.3 + 0 + 0.5) / 3),
                                              5e-4: pytest.approx((0.4 + 0 + 1.0) / 3)}
    assert all(math.isnan(v) for v in O.precision(np.zeros((0, 3)), [1e-4, 5e-4]).values())
    from argparse import Namespace
    recs = [Namespace(counts=np.array(r, dtype=np.int32)) for r in rows]
    assert RP.precision(recs, [1e-4, 5e-4]) == O.precision(rows, [1e-4, 5e-4])
    assert all(math.isnan(v) for v in RP.precision([], [5e-4]).values())


def test_pair_thresholds():
    from argparse import Namespace
    K0 = np.array([[500.0, 0, 320], [0, 510.0, 240], [0, 0, 1]])
    K1 = np.array([[400.0, 0, 300], [0, 420.0, 250], [0, 0, 1]])
    T = np.eye(4)
    T[0, 3] = 1.0
    intr, Rt, px = RP.pair_arrays([Namespace(K0=K0, K1=K1, T_0to1=T)], 0.5)
    assert np.array_equal(intr[0], [500, 510, 320, 240, 400, 420, 300, 250])
    assert np.array_equal(Rt[0], _rt(np.eye(3), [1, 0, 0]))
    f_mean = (500 + 420 + 500 + 420) / 4
    # the engine's threshold in camera coordinates, px_th / ((fx1 + fy1) / 2), is the protocol's 0.5 / f_mean
    assert px[0] / ((400 + 420) / 2) == pytest.approx(0.5 / f_mean, rel=1e-15)


# ---- readers ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fmt', ['txt', 'npz'])
def test_readers_on_synth_files(tmp_path, fmt):
    path, gts = synthetic_relpose_tree(str(tmp_path), 5, 3, fmt=fmt, size=(96, 64))
    pairs = RP.read_pairs(path, str(tmp_path))
    assert len(pairs) == 3
    for k, (p, g) in enumerate(zip(pairs, gts)):
        assert p.name0 == f'images/pair{k:03d}_0.png' and p.name1 == f'images/pair{k:03d}_1.png'
        assert os.path.isfile(p.path0) and os.path.isfile(p.path1)
        assert np.array_equal(p.K0, g['K0']) and np.array_equal(p.K1, g['K1'])
        if fmt == 'txt':
            assert np.array_equal(p.T_0to1, g['T_0to1'])           # %.17g reads back exactly
        else:
            assert np.allclose(p.T_0to1, g['T_0to1'], rtol=0, atol=1e-12)
    again, _ = synthetic_relpose_tree(str(tmp_path / 'again'), 5, 3, fmt=fmt, size=(96, 64))
    from PIL import Image
    for p in pairs:
        a = np.array(Image.open(p.path1))
        b = np.array(Image.open(os.path.join(str(tmp_path / 'again'), p.name1)))
        assert np.array_equal(a, b) and a.shape == (64, 96, 3) and a.any()


def _line(rot=(0, 0), t=(1.0, 0.0, 0.0), n_vals=34):
    K = [500, 0, 320, 0, 500, 240, 0, 0, 1]
    T = [1, 0, 0, t[0], 0, 1, 0, t[1], 0, 0, 1, t[2], 0, 0, 0, 1]
    vals = (K + K + T)[:n_vals] + [0] * max(0, n_vals - 34)
    return ' '.join(['a.png', 'b.png', str(rot[0]), str(rot[1])] + [repr(float(v)) for v in vals])


@pytest.mark.parametrize('line,match', [
    (_line(rot=(0, 90)), 'EXIF rotation'),
    (_line(rot=(180, 0)), 'EXIF rotation'),
    (_line(t=(0.0, 0.0, 0.0)), 'zero norm'),
    (_line(n_vals=33), '38 fields'),
    (_line(n_vals=35), '38 fields'),
    (_line().replace('320.0', 'x20', 1), 'x20'),
    ('a.png b.png', '38 fields'),
])
def test_text_reader_rejects(tmp_path, line, match):
    f = tmp_path / 'pairs.txt'
    f.write_text(_line() + '\n\n' + line + '\n')
    with pytest.raises(ValueError, match=match) as e:
        RP.read_pairs(str(f), str(tmp_path))
    assert 'pairs.txt:3' in str(e.value)


def test_npz_reader_rejects(tmp_path):
    path, _ = synthetic_relpose_tree(str(tmp_path), 1, 2, fmt='npz', size=(32, 32))
    z = dict(np.load(path, allow_pickle=True))
    bad = dict(z)
    bad['poses'] = z['poses'].copy()
    bad['poses'][2] = bad['poses'][3] = np.eye(4)            # pair 1: the same camera twice
    np.savez(str(tmp_path / 'same.npz'), **bad)
    with pytest.raises(ValueError, match=r'pair_infos\[1\].*zero norm'):
        RP.read_pairs(str(tmp_path / 'same.npz'), str(tmp_path))
    del bad['intrinsics']
    np.savez(str(tmp_path / 'nok.npz'), **bad)
    with pytest.raises(ValueError, match='intrinsics'):
        RP.read_pairs(str(tmp_path / 'nok.npz'), str(tmp_path))


def test_cli_help():
    r = subprocess.run([sys.executable, '-m', 'patch2pix_b200.relpose', '--help'], cwd=ROOT, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0 and '--pairs' in r.stdout and '--data_root' in r.stdout
