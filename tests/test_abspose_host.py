"""Absolute pose and the InLoc protocol on the host: the P3P oracle against OpenCV, the oracle's RANSAC on synthetic
2D-3D matches, the scan-lift oracle against grid_sample, the InLoc readers, the results file, eval_localization and
the CLI's rejections.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import abspose_oracle as A
from patch2pix_b200 import localize as L
from patch2pix_b200.synth import synthetic_abspose, synthetic_inloc_tree


def _rot(v):
    th = np.linalg.norm(v)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]]) / th
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def test_p3p_contains_true_pose_and_agrees_with_opencv():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(0)
    checked = tight = 0
    for _ in range(200):
        R0, t0 = _rot(rng.normal(0, 0.7, 3)), rng.normal(0, 1, 3) + [0, 0, 8]
        X = rng.uniform(-2, 2, (3, 3))
        Xc = X @ R0.T + t0
        if (Xc[:, 2] < 1).any():
            continue
        j = Xc / np.linalg.norm(Xc, axis=1, keepdims=True)
        sols = A.solve_p3p(j, X)
        err = min(np.abs(m[:9] - R0.ravel()).max() + np.abs(m[9:] - t0).max() for m in sols)
        assert err < 1e-4                       # near a double root the polished roots lose digits
        tight += err < 1e-8
        uv = Xc[:, :2] / Xc[:, 2:]
        n, rv, tv = cv2.solveP3P(X.reshape(3, 1, 3), uv.reshape(3, 1, 2), np.eye(3), None, flags=cv2.SOLVEPNP_P3P)
        cv = [np.concatenate([cv2.Rodrigues(r)[0].ravel(), t.ravel()]) for r, t in zip(rv, tv)]
        for m in sols:                          # every oracle pose is one of OpenCV's
            assert min(np.abs(m - c).max() for c in cv) < 1e-4
        checked += 1
    assert checked > 150 and tight > 0.95 * checked


def test_quartic_roots_polished_and_sorted():
    r = A.quartic_roots([24.0, -50.0, 35.0, -10.0, 1.0])       # (v - 1)(v - 2)(v - 3)(v - 4)
    assert np.allclose(r, [1, 2, 3, 4], atol=1e-12) and r == sorted(r)
    assert A.quartic_roots([1.0, 0.0, 1.0, 0.0, 0.0]) == []     # degree drop


@pytest.mark.parametrize('ratio,noise', [(0.5, 0.0), (0.7, 1.0)])
def test_oracle_ransac_recovers_pose(ratio, noise):
    sc = synthetic_abspose(3, 1500, ratio, noise)
    rows = np.concatenate([sc['pts2d'], sc['pts3d']], 1)
    intr = L._camera(sc['K'])
    m, mask, c = A.find_absolute_pose(rows, intr, 4.0)
    R, t = m[:9].reshape(3, 3), m[9:]
    ang = np.degrees(np.arccos(np.clip((np.trace(sc['R'].T @ R) - 1) / 2, -1, 1)))
    dpos = np.linalg.norm(-R.T @ t + sc['R'].T @ sc['t'])
    assert (mask & sc['inlier']).sum() >= 0.98 * sc['inlier'].sum()
    if noise == 0:
        assert ang < 1e-6 and dpos < 1e-8 and c == sc['inlier'].sum()
    else:
        assert ang < 0.1 and dpos < 0.02


def test_oracle_bad_rows():
    sc = synthetic_abspose(4, 50, 0.2, 0.0)
    rows = np.concatenate([sc['pts2d'], sc['pts3d']], 1)
    rows[7, 3] = np.nan
    m, mask, c = A.find_absolute_pose(rows, L._camera(sc['K']), 2.0)
    assert c == -1 and np.isnan(m).all() and not mask.any()
    assert A.find_absolute_pose(rows[:3][:, :5] * 0 + 1, L._camera(sc['K']), 2.0)[2] == 0


def test_lift_oracle_matches_grid_sample():
    rng = np.random.default_rng(5)
    H, W = 37, 53
    scan = rng.normal(0, 10, (H, W, 3))
    scan[5:9, 10:20] = np.nan                           # holes: bilinear NaN near them, nearest may recover
    scan[20, 30] = np.nan
    pts = np.concatenate([rng.uniform([0, 0], [W - 1, H - 1], (400, 2)),
                          [[0, 0], [W - 1, H - 1], [W - 1, 0], [9.5, 8.5], [10.5, 6.5], [30, 20], [29.5, 19.5]]])
    g = torch.from_numpy(pts / np.array([W - 1, H - 1]) * 2 - 1)[None, None]
    s = torch.from_numpy(scan).permute(2, 0, 1)[None]
    lin = torch.nn.functional.grid_sample(s, g, mode='bilinear', align_corners=True)[0, :, 0].T.numpy()
    nn = torch.nn.functional.grid_sample(s, g, mode='nearest', align_corners=True)[0, :, 0].T.numpy()
    ref = np.where(np.isnan(lin), nn, lin)
    got = A.sample_scan(scan, pts[:, 0], pts[:, 1])
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.allclose(got[ok], ref[ok], rtol=1e-12, atol=1e-12)
    assert np.isnan(got).any(1).sum() > 0 and (~np.isnan(got).any(1)).sum() > 300
    # lift: rows dropped (outside or NaN), order kept, alignment applied
    Ta = np.eye(4)
    Ta[:3, :3], Ta[:3, 3] = _rot(np.array([0.1, -0.2, 0.3])), [100, -20, 5]
    m = np.concatenate([rng.uniform(0, 100, (pts.shape[0], 2)), pts], 1)
    m = np.concatenate([m, [[1, 2, -0.5, 3], [1, 2, W - 0.5, 3], [1, 2, np.nan, 3]]])
    rows = A.lift_scan(scan, Ta, m)
    keep = ~np.isnan(ref).any(1)
    assert rows.shape == (keep.sum(), 5)
    assert np.array_equal(rows[:, :2], m[:len(pts)][keep, :2])
    assert np.allclose(rows[:, 2:], ref[keep] @ Ta[:3, :3].T + Ta[:3, 3], rtol=0, atol=1e-9)


def test_inloc_readers_and_results_roundtrip(tmp_path):
    tree = synthetic_inloc_tree(str(tmp_path), 0, 2, 3, size=(64, 48))
    ret = L.read_retrieval(tree['pairs'])
    assert [q for q, _ in ret] == list(tree['queries']) and all(len(d) == 3 for _, d in ret)
    assert [d for _, ds in ret for d in ds] == list(tree['db'])
    db = ret[1][1][2]
    scan = L.read_scan(str(tmp_path / (db + '.mat')))
    assert scan.shape == (48, 64, 3) and scan.flags.c_contiguous and np.isnan(scan).any()
    Ta = L.read_alignment(L.alignment_path(str(tmp_path), db))
    assert L.alignment_path('/r', 'database/cutouts/DUC1/005/DUC_cutout_005_0_0.jpg') == \
        '/r/database/alignments/DUC1/transformations/DUC_trans_005.txt'
    # the scan in world coordinates reprojects into its cutout
    K, R, t = tree['db'][db]
    X = scan.reshape(-1, 3) @ Ta[:3, :3].T + Ta[:3, 3]
    ok = ~np.isnan(X).any(1)
    P = X[ok] @ R.T + t
    v, u = np.mgrid[0:48, 0:64]
    uv = np.stack([u.ravel(), v.ravel()], 1)[ok]
    assert np.abs(P[:, :2] / P[:, 2:] * K[0, 0] + K[:2, 2] - uv).max() < 1e-6
    gt = L.read_results(tree['gt'])
    assert set(gt) == {q.split('/')[-1] for q in tree['queries']}
    for q, (K, R, t) in tree['queries'].items():
        Rr, tr = gt[q.split('/')[-1]]
        assert np.abs(Rr - R).max() < 1e-12 and np.abs(tr - t).max() < 1e-12
    out = tmp_path / 'res.txt'
    L.write_results(str(out), [(n, R, t) for n, (R, t) in gt.items()])
    back = L.read_results(str(out))
    assert all(np.abs(back[n][0] - gt[n][0]).max() < 1e-14 and np.array_equal(back[n][1], gt[n][1]) for n in gt)
    bad = tmp_path / 'bad.txt'
    bad.write_text('a b c\n')
    with pytest.raises(ValueError, match='expected 2 fields'):
        L.read_retrieval(str(bad))
    with pytest.raises(ValueError, match='expected 8 fields'):
        L.read_results(str(bad))
    with pytest.raises(ValueError, match='lines 7-10'):
        L.read_alignment(str(bad))


def test_quaternion_roundtrip():
    rng = np.random.default_rng(1)
    for v in list(rng.normal(0, 2, (50, 3))) + [np.array([np.pi, 0, 0]), np.array([0, np.pi - 1e-9, 0])]:
        R = _rot(v)
        q = L.rotmat_to_qvec(R)
        assert q[0] >= 0 and abs(np.linalg.norm(q) - 1) < 1e-12
        assert np.abs(L.qvec_to_rotmat(q) - R).max() < 1e-9


def test_eval_localization_hand_made():
    R0, t0 = np.eye(3), np.zeros(3)
    gt = {'a': (R0, t0), 'b': (R0, t0), 'c': (R0, t0), 'd': (R0, t0)}
    res = {'a': (R0, np.array([0.2, 0, 0])),                       # 0.2 m, 0 deg
           'b': (_rot(np.radians([0, 0, 12.0])), t0),             # 0 m, 12 deg
           'c': (R0, np.array([0, 0.7, 0]))}                      # 0.7 m; d missing
    out = L.eval_localization(res, gt)
    assert out['recall'] == {(0.25, 10.0): 0.25, (0.5, 10.0): 0.25, (1.0, 10.0): 0.5}
    assert abs(out['errors']['b'][1] - 12.0) < 1e-9 and out['errors']['d'] == (np.inf, np.inf)
    assert np.isnan(L.eval_localization({}, {})['recall'][(0.25, 10.0)])


def test_cli_rejections(tmp_path, capsys):
    with pytest.raises(SystemExit):
        L.main([])                                                  # required arguments
    pairs = tmp_path / 'pairs.txt'
    pairs.write_text('q d\n')
    base = ['--ckpt', str(tmp_path / 'missing.pth'), '--data_root', str(tmp_path), '--pairs', str(pairs),
            '--results', str(tmp_path / 'r.txt')]
    for argv, msg in ((base, 'ckpt'), (base[:3] + [str(tmp_path / 'nodir')] + base[4:], 'data_root'),
                      (base[:5] + [str(tmp_path / 'nofile')] + base[6:], 'pairs'),
                      (base + ['--method', 'sift'], 'method')):
        with pytest.raises(SystemExit):
            L.main(argv)
        assert msg in capsys.readouterr().err
    (tmp_path / 'c.pth').write_text('')
    with pytest.raises(SystemExit):
        L.main(['--ckpt', str(tmp_path / 'c.pth')] + base[2:] + ['--ransac_thres', '0'])
    assert 'ransac_thres' in capsys.readouterr().err
