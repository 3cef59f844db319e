"""GPU F RANSAC with the DEGENSAC degeneracy check (model 2 of p2p_find_model, p2p_test_degeneracy) against the numpy
oracle (oracle/degensac_oracle.py), and matches2relapose_degensac against the numpy chain of geometry.py:50-71.

As in test_gpu_verify.py, the device scores F in fp32 and the oracle in fp64, so final inlier decisions may differ on rows
whose Sampson error lies within the derived per-row bound of oracle/ransac_bound.py of px_th^2; comparisons exempt
exactly those rows.  The degeneracy test is compared on well-conditioned samples whose points are not within BAND of
h_th^2 under an induced H."""
import numpy as np
import pytest
import torch

from oracle import degensac_oracle as D
from oracle import ransac_bound as RB
from oracle import verify_oracle as V
from patch2pix_b200.synth import OFF_PLANE, PLANE, synthetic_dominant_plane, synthetic_two_view
from test_gpu_verify import _canon, _compare_final as _compare_final_f, _dtoh, _well_conditioned

pytestmark = pytest.mark.gpu
# The plane tests run in fp64 on the device (h_inlier64, with affine2's fixed rounding of H x1), so they differ from the
# oracle's fp64 transfer error only by fp64 rounding: a relative band of 1e-4 of h_th^2 is far wider than that.  The
# fp32 final F decisions use the derived bound instead.
BAND = 1e-4


def _dominant(seed, n=1000, **kw):
    sc = synthetic_dominant_plane(seed, n, 0.3, 0.08, 0.5, **kw)
    return sc, np.concatenate([sc['pts1'], sc['pts2']], 1)


def _near_h(F, rows7, T, h_th2):
    """Whether any point of the sample lies within the band of h_th^2 under any induced H the test evaluates."""
    P = V.normalise(rows7, T)
    Fn = D.normalise_f(F, T)
    for tri in D.TRIPLETS:
        Hn = D.induced_homography(Fn, P[list(tri)])
        if Hn is None:
            continue
        H, ok = V.denormalise(1, Hn.reshape(9), T)
        if ok[0] and (np.abs(V.errors(1, H[0], rows7)[0] - h_th2) <= BAND * h_th2).any():
            return True
    return False


def test_degeneracy_hook_matches_oracle():
    from patch2pix_b200.verify import first_degeneracy, first_hypotheses
    sc, rows = _dominant(1)
    count, seed, th = 2048, 3, 1.0
    tri, H = first_degeneracy(sc['pts1'], sc['pts2'], th, count, seed=seed)
    _, gc = first_hypotheses(0, sc['pts1'], sc['pts2'], th, count, seed=seed)
    T = V.normalisation(rows)
    otri, oH = D.degeneracy_hypotheses(rows, T, np.arange(count), seed, th)
    om, ov = V.hypotheses(0, rows, T, np.arange(count), seed)
    idx, _ = V.draw_samples(seed, np.arange(count), rows.shape[0], 7)
    assert np.array_equal(tri == -2, gc < 0)
    h_th2 = (2.0 * th) ** 2
    flagged = clean = 0
    for i in range(count):
        if not _well_conditioned(0, rows, T, i, seed):
            continue
        for k in range(3):
            s = 3 * i + k
            if not ov[s] or gc[s] < 0 or _near_h(om[s], rows[idx[i]], T, h_th2):
                continue
            assert tri[s] == otri[s], (i, k, tri[s], otri[s])
            if otri[s] >= 0:
                assert np.abs(_canon(H[s]) - _canon(oH[s])).max() < 1e-4, (i, k)
                flagged += 1
            else:
                clean += 1
    assert flagged > 200 and clean > 1000, (flagged, clean)


def _compare_final(rows, gmask, th, seed=0, **kw):
    tr = {}
    M, omask, _ = D.find_model(rows, th, seed=seed, trace=tr, **kw)
    assert M is not None
    near = ~(np.abs(V.errors(0, M, rows)[0] - th * th) > RB.decision_bound(0, M, rows, th * th))
    if tr['margin'] <= int(near.sum()):
        return False
    diff = gmask != omask
    assert not (diff & ~near).any(), (np.nonzero(diff & ~near)[0][:10], tr)
    return True


@pytest.mark.parametrize('scene, seed', [('plane', 2), ('plane', 3), ('plane', 13), ('general', 2), ('general', 9)])
def test_final_result_matches_oracle(scene, seed):
    from patch2pix_b200.verify import find_fundamental_matrix
    if scene == 'plane':
        sc, rows = _dominant(seed)
    else:
        sc = synthetic_two_view(seed, 1000, 0.5, 0.5)
        rows = np.concatenate([sc['pts1'], sc['pts2']], 1)
    F, mask = find_fundamental_matrix(sc['pts1'], sc['pts2'], 1.0, seed=4, degeneracy_check=True)
    assert F is not None and F.shape == (3, 3) and F.dtype == np.float64 and mask.dtype == bool
    applied = _compare_final(rows, mask, 1.0, seed=4)
    assert applied or abs(int(mask.sum()) - int(D.find_model(rows, 1.0, seed=4)[2])) <= 3
    # without the check the call is model 0, unchanged
    F0, mask0 = find_fundamental_matrix(sc['pts1'], sc['pts2'], 1.0, seed=4)
    assert F0 is not None
    _compare_final_f(0, rows, mask0, 1.0, seed=4)


def test_recovers_off_plane_inliers_on_the_device():
    from patch2pix_b200.verify import find_fundamental_matrix
    rec = []
    for seed in range(20):
        sc, _ = _dominant(seed)
        F, mask = find_fundamental_matrix(sc['pts1'], sc['pts2'], 1.0, degeneracy_check=True)
        assert F is not None and mask[sc['label'] == PLANE].mean() >= 0.9
        rec.append(mask[sc['label'] == OFF_PLANE].mean())
    assert np.median(rec) >= 0.9 and min(rec) >= 0.8, rec


def test_results_are_deterministic():
    from patch2pix_b200 import _lib
    from patch2pix_b200.verify import find_fundamental_matrix
    h = _lib.default_handle(torch.device('cuda', torch.cuda.current_device()))
    for sc in (_dominant(5, n=3000)[0], synthetic_two_view(5, 3000, 0.6, 0.5)):
        p1 = torch.from_numpy(sc['pts1']).cuda()
        p2 = torch.from_numpy(sc['pts2']).cuda()
        outs = []
        for sms in (0, 0, 66):
            h.set_option('num_sms', sms)
            F, mask = find_fundamental_matrix(p1, p2, 1.0, seed=7, degeneracy_check=True)
            outs.append((F.cpu().numpy().tobytes(), mask.cpu().numpy().tobytes()))
        h.set_option('num_sms', 0)
        assert outs[0] == outs[1] == outs[2]


def test_edge_cases():
    from patch2pix_b200.verify import find_fundamental_matrix, first_degeneracy
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 500, (6, 2))
    F, mask = find_fundamental_matrix(p, p + 3.0, 1.0, degeneracy_check=True)
    assert F is None and mask.shape == (6,) and not mask.any()
    q = rng.uniform(0, 500, (100, 2))
    q[17, 1] = np.nan
    with pytest.raises(ValueError):
        find_fundamental_matrix(q, q + 1.0, 1.0, degeneracy_check=True)
    Ft, mt = find_fundamental_matrix(torch.from_numpy(q).cuda(), torch.from_numpy(q + 1.0).cuda(), 1.0,
                                     degeneracy_check=True)
    assert torch.isnan(Ft).all() and not mt.any()
    # a purely planar scene: every inlier is coplanar, so samples of inliers are degenerate (the oracle flags 77 % of
    # them at this noise) and the plane is kept whatever F the parallax rounds settle on
    sc = synthetic_two_view(5, 1000, 0.3, 0.5, planar=True)
    rows = np.concatenate([sc['pts1'], sc['pts2']], 1)
    tri, _ = first_degeneracy(sc['pts1'], sc['pts2'], 1.0, 1024, seed=3)
    idx, _ = V.draw_samples(3, np.arange(1024), 1000, 7)
    slots = np.repeat(sc['inlier'][idx].all(1), 3) & (tri > -2)
    assert slots.sum() > 50 and (tri[slots] >= 0).mean() > 0.6
    F, mask = find_fundamental_matrix(sc['pts1'], sc['pts2'], 1.0, degeneracy_check=True)
    assert F is not None and (mask & sc['inlier']).sum() >= 0.95 * sc['inlier'].sum()
    assert _compare_final(rows, mask, 1.0) or abs(int(mask.sum()) - int(D.find_model(rows, 1.0)[2])) <= 3
    # 2^20 rows
    sc, _ = _dominant(8, n=1 << 20)
    F, mask = find_fundamental_matrix(sc['pts1'], sc['pts2'], 1.0, max_iters=2048, degeneracy_check=True)
    assert F is not None and mask.shape == (1 << 20,)
    assert mask[sc['label'] == PLANE].mean() >= 0.95 and mask[sc['label'] == OFF_PLANE].mean() >= 0.8


def _angle(R1, R2):
    return np.degrees(np.arccos(np.clip((np.trace(R1.T @ R2) - 1) / 2, -1, 1)))


def _t_angle(t, tg):
    t = np.asarray(t, dtype=np.float64).ravel()
    return np.degrees(np.arccos(np.clip(abs(t @ tg) / (np.linalg.norm(t) * np.linalg.norm(tg)), -1, 1)))


def test_matches2relapose_degensac_matches_the_numpy_chain():
    cv2 = pytest.importorskip('cv2')
    from patch2pix_b200.pose import matches2relapose, matches2relapose_degensac
    errs, errs_e = [], []
    for seed in range(6):
        sc, _ = _dominant(seed, focal2=650.0)
        K1, K2 = sc['K1'], sc['K2']
        E, inls, R, t = matches2relapose_degensac(sc['pts1'], sc['pts2'], K1, K2, rthres=1.0)
        # geometry.py:50-71 with oracle model 2 in place of pydegensac
        f1, f2 = K1[0, 0], K2[0, 0]
        p1 = (sc['pts1'] - K1[:2, 2][None]) * f2 / f1
        p2 = sc['pts2'] - K2[:2, 2][None]
        rows = np.concatenate([p1, p2], 1)
        K = np.diag([f2, f2, 1.0])
        mask = np.zeros(len(rows), dtype=bool)
        mask[inls] = True
        applied = _compare_final(rows, mask, 1.0)
        oF, omask, _ = D.find_model(rows, 1.0)
        oE = K.T @ oF @ K
        oi = np.where(omask)[0]
        _, oR, ot, _ = cv2.recoverPose(oE, p1[oi], p2[oi], K)
        if applied and np.array_equal(mask, omask):
            assert _angle(R, oR) < 1e-4 and _t_angle(t, ot.ravel()) < 1e-3
        assert _angle(R, oR) < 0.5
        errs.append((_angle(R, sc['R']), _t_angle(t, sc['t'])))
        _, _, Re, te = matches2relapose(sc['pts1'], sc['pts2'], K1, K2, rthres=1.0)
        errs_e.append((_angle(Re, sc['R']), _t_angle(te, sc['t'])))
    errs, errs_e = np.array(errs), np.array(errs_e)
    # measured on the oracle: rotation error below E RANSAC's on every scene; translation error below on average
    # (E RANSAC loses one scene entirely) but not on every scene
    assert errs[:, 0].mean() < errs_e[:, 0].mean() and errs[:, 1].mean() < errs_e[:, 1].mean(), (errs, errs_e)
    assert errs[:, 0].max() < 0.5, errs


def test_estimate_matches_degensac_pipeline(consensus_sd):
    from patch2pix_b200.eval_helper import _finalize, estimate_matches, load_model
    from patch2pix_b200.synth import synthetic_pair_shifted
    net = load_model(consensus_sd)
    im1, im2 = synthetic_pair_shifted(2, 240, 320)
    m, s, c, inl, F = estimate_matches(net, im1, im2, eval_type='coarse', verify=('DEGENSAC', 1.0))
    m0, s0, c0 = estimate_matches(net, im1, im2, eval_type='coarse')
    assert np.array_equal(m, m0) and np.array_equal(s, s0) and np.array_equal(c, c0)
    assert F is not None and inl.shape == (len(m),) and inl.dtype == bool
    if len(m) >= 7:
        _compare_final(m, inl, 1.0)
    with torch.no_grad():
        cm, sc = net.predict_coarse(im1.cuda(), im2.cuda())
    up = (1.0, 1.0, 1.0, 1.0)
    _, n_tail = _dtoh(lambda: _finalize(net, None, sc[0], cm[0], float('-inf'), up, ('DEGENSAC', 1.0)))
    _, n_plain = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse'))
    _, n_ver = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse', verify=('DEGENSAC', 1.0)))
    assert n_tail == 1 and n_ver == n_plain
