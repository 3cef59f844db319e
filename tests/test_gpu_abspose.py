"""GPU absolute pose (p2p_find_absolute_pose_batch, p2p_lift_scan) against the numpy oracle (oracle/abspose_oracle.py)
and OpenCV.

The device scores in fp32 and the oracle in fp64, so inlier decisions may differ on rows whose squared reprojection
error lies within the derived per-row bound of oracle/ransac_bound.py (decision_bound) of th^2; every comparison below
exempts exactly those rows and nothing else, as test_gpu_pose.py does."""
import numpy as np
import pytest
import torch

from oracle import abspose_oracle as A
from oracle import ransac_bound as RB
from patch2pix_b200 import localize as L
from patch2pix_b200.synth import synthetic_abspose

pytestmark = pytest.mark.gpu
TH = 4.0


def _scene(seed=0, n=1000, ratio=0.5, noise=0.5):
    sc = synthetic_abspose(seed, n, ratio, noise)
    return sc, np.concatenate([sc['pts2d'], sc['pts3d']], 1), L._camera(sc['K'])


def _near(m, rows, intr, mean, th2):
    e = A.errors(m, rows, intr, mean)[0]
    return ~(np.abs(e - th2) > RB.decision_bound(4, m, rows, th2, intr, mean))


def _well_conditioned(rows, intr, mean, hyp, seed):
    """The oracle's rating of a sample: its quartic's real roots are well separated from each other, the valid poses'
    denominators are not small, and the sample's triangle is not thin."""
    idx, ok = A.V.draw_samples(seed, [hyp], rows.shape[0], 3)
    if not ok[0]:
        return False
    j, X = A.bearings(rows[idx[0]], intr), rows[idx[0], 2:5] - mean
    e = np.cross(X[1] - X[0], X[2] - X[0])
    if np.linalg.norm(e) < 1e-2 * np.linalg.norm(X[1] - X[0]) * np.linalg.norm(X[2] - X[0]):
        return False
    q = A.p3p_quartic(j, X)
    r = np.roots(np.asarray(q[0])[::-1])
    real = r[np.abs(r.imag) < 1e-6 * (1 + np.abs(r))].real
    if len(real) != len(A.quartic_roots(q[0])):
        return False
    re = np.sort(real)
    _, ca, _, cg, _ = q[1]
    if len(re) and np.abs(cg - re * ca).min() < 1e-3:
        return False
    return len(re) < 2 or np.diff(re).min() > 1e-2 * (1 + np.abs(re).max())


def test_hypotheses_match_oracle():
    sc, rows, intr = _scene(seed=1)
    count, seed = 512, 3
    gm, gc = L.first_absolute_pose_hypotheses(sc['pts2d'], sc['pts3d'], sc['K'], TH, count, seed=seed)
    mean = rows[:, 2:5].mean(0)
    om, ov = A.hypotheses(rows, intr, np.arange(count), seed, mean)
    th2 = TH * TH
    checked = models = 0
    for i in range(count):
        if not _well_conditioned(rows, intr, mean, i, seed):
            continue
        checked += 1
        o = [k for k in range(4) if ov[i * 4 + k]]
        g = [k for k in range(4) if gc[i * 4 + k] >= 0]
        assert len(o) == len(g), (i, o, g)
        for k, kk in zip(o, g):
            assert np.abs(gm[i * 4 + kk] - om[i * 4 + k]).max() < 1e-6, (i, k)
            cnt = int((A.errors(om[i * 4 + k], rows, intr, mean)[0] < th2).sum())
            nb = int(_near(om[i * 4 + k], rows, intr, mean, th2).sum())
            assert abs(int(gc[i * 4 + kk]) - cnt) <= nb, (i, k, gc[i * 4 + kk], cnt, nb)
            models += 1
    assert checked > 0.8 * count and models >= checked, (checked, models)


def _compare_final(mask_gpu, rows, intr, seed):
    """GPU mask against the oracle's, except near-threshold rows, when the oracle's winning margin exceeds their
    number.  Returns whether the comparison applied."""
    tr = {}
    m, omask, _ = A.find_absolute_pose(rows, intr, TH, seed=seed, trace=tr)
    mean = rows[:, 2:5].mean(0)
    centred = np.concatenate([m[:9], m[9:] + m[:9].reshape(3, 3) @ mean])
    near = _near(centred, rows, intr, mean, TH * TH)
    if tr['margin'] <= int(near.sum()):
        return False
    diff = mask_gpu != omask
    assert not (diff & ~near).any(), (np.nonzero(diff & ~near)[0][:10], tr)
    return True


@pytest.mark.parametrize('ratio', [0.5, 0.7])
def test_final_mask_matches_oracle(ratio):
    sc, rows, intr = _scene(seed=2, n=1500, ratio=ratio, noise=0.8)
    R, t, mask = L.find_absolute_pose(sc['pts2d'], sc['pts3d'], sc['K'], TH, seed=4)
    assert R.shape == (3, 3) and t.shape == (3,) and mask.dtype == bool and mask.shape == (1500,)
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-9
    applied = _compare_final(mask, rows, intr, 4)
    assert (mask & sc['inlier']).sum() >= 0.97 * sc['inlier'].sum()
    assert applied or abs(int(mask.sum()) - A.find_absolute_pose(rows, intr, TH, seed=4)[2]) <= 3


def test_batched_equals_single_and_bad_rows():
    scs = [synthetic_abspose(10 + k, n, r, 0.7) for k, (n, r) in enumerate([(900, 0.4), (3, 0.0), (2500, 0.6),
                                                                            (40, 0.2), (1200, 0.5)])]
    p2, p3, Ks = [s['pts2d'] for s in scs], [s['pts3d'] for s in scs], [s['K'] for s in scs]
    many = L.find_absolute_poses(p2, p3, Ks, TH, seed=7)
    th_each = L.find_absolute_poses(p2, p3, Ks, [TH] * len(scs), seed=7)
    for k in range(len(scs)):
        one = L.find_absolute_pose(p2[k], p3[k], Ks[k], TH, seed=7)
        for a, b, c in zip(many[k], one, th_each[k]):
            if a is None:
                assert b is None and c is None
            else:
                assert np.array_equal(a, b) and np.array_equal(a, c), k
    assert many[1][0] is None and not many[1][2].any()          # 3 rows: no model
    assert all(many[k][0] is not None for k in (0, 2, 3, 4))
    # a per-query threshold takes effect per query
    diff = L.find_absolute_poses(p2, p3, Ks, [TH, TH, 1.0, TH, TH], seed=7)
    assert np.array_equal(diff[0][2], many[0][2]) and np.array_equal(diff[4][0], many[4][0])
    assert diff[2][2].sum() < many[2][2].sum()
    # CUDA tensors: a non-finite row gives NaN for that query only, without a sync
    t2 = [torch.from_numpy(x).cuda() for x in p2]
    t3 = [torch.from_numpy(x.copy()).cuda() for x in p3]
    t3[3][5, 1] = float('nan')
    res = L.find_absolute_poses(t2, t3, Ks, TH, seed=7)
    assert torch.isnan(res[3][0]).all() and torch.isnan(res[3][1]).all() and not res[3][2].any()
    assert torch.isnan(res[1][0]).all()
    for k in (0, 2, 4):
        assert np.array_equal(res[k][0].cpu().numpy(), many[k][0]) and np.array_equal(res[k][2].cpu().numpy(),
                                                                                       many[k][2])
    with pytest.raises(ValueError, match='not finite'):
        L.find_absolute_poses([p2[3]], [t3[3].cpu().numpy()], Ks[3], TH)
    from patch2pix_b200.verify import batch_chunk_pairs
    assert 1 < batch_chunk_pairs(L.ENTRY_ABSPOSE) <= 65535


def _errs(sc, R, t):
    ang = np.degrees(np.arccos(np.clip((np.trace(sc['R'].T @ R) - 1) / 2, -1, 1)))
    return ang, np.linalg.norm(-R.T @ t + sc['R'].T @ sc['t'])


def test_accuracy_noise_free_and_against_opencv():
    cv2 = pytest.importorskip('cv2')
    for seed in range(4):
        sc = synthetic_abspose(100 + seed, 2000, 0.6, 0.0)
        R, t, mask = L.find_absolute_pose(sc['pts2d'], sc['pts3d'], sc['K'], TH)
        ang, dp = _errs(sc, R, t)
        assert ang < 0.01 and dp < 1e-6 * 20.0, (seed, ang, dp)        # scene depth up to 20 units
    # A threshold near the noise: LO keeps a refit only while the inlier count grows, so at a threshold far above the
    # noise (every inlier already in the minimal sample's set) the pose stays the sample's, where OpenCV refines.
    for seed in range(4):
        sc = synthetic_abspose(200 + seed, 3000, 0.6, 1.0)
        R, t, mask = L.find_absolute_pose(sc['pts2d'], sc['pts3d'], sc['K'], 2.0)
        ok, rv, tv, inl = cv2.solvePnPRansac(sc['pts3d'], sc['pts2d'], sc['K'], None, iterationsCount=10000,
                                             reprojectionError=2.0, confidence=0.99999, flags=cv2.SOLVEPNP_P3P)
        assert ok
        ga, gp = _errs(sc, R, t)
        ca, cp = _errs(sc, cv2.Rodrigues(rv)[0], tv.ravel())
        assert ga <= 2 * ca + 0.02 and gp <= 2 * cp + 0.01, (seed, ga, ca, gp, cp)


def test_lift_matches_oracle_bit_for_bit():
    rng = np.random.default_rng(9)
    items, ref = [], []
    for c in range(3):
        H, W = int(rng.integers(30, 90)), int(rng.integers(30, 90))
        scan = rng.normal(0, 30, (H, W, 3)) + 1000.0
        for _ in range(5):
            y0, x0 = int(rng.integers(0, H - 4)), int(rng.integers(0, W - 4))
            scan[y0:y0 + int(rng.integers(1, 6)), x0:x0 + int(rng.integers(1, 6))] = np.nan
        Ta = np.eye(4)
        Ta[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        Ta[:3, 3] = rng.normal(0, 100, 3)
        m = np.concatenate([rng.uniform(0, 500, (700, 2)), rng.uniform([-2, -2], [W + 1, H + 1], (700, 2))], 1)
        m[::50, 2] = np.round(m[::50, 2])                         # on pixel centres
        m[1::50, 2:4] = np.floor(m[1::50, 2:4]) + 0.5             # ties of the nearest pixel
        items.append((scan, Ta, m))
        ref.append(A.lift_scan(scan, Ta, m))
    got = L.lift_scans(items)
    ref = np.concatenate(ref)
    assert got.shape == ref.shape and ref.shape[0] > 1000
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))
