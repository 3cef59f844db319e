"""GPU relative pose (p2p_find_essential / p2p_recover_pose) against the numpy oracle (oracle/pose_oracle.py) and OpenCV.

The device scores in fp32 and the oracle in fp64, so inlier decisions may differ on rows whose Sampson error lies within
the derived per-row bound of oracle/ransac_bound.py (decision_bound) of th^2; every comparison below exempts exactly
those rows and nothing else, as test_gpu_verify.py does."""
import numpy as np
import pytest
import torch

from oracle import pose_oracle as P
from oracle import ransac_bound as RB
from patch2pix_b200.synth import synthetic_two_view
from test_gpu_verify import _dtoh

pytestmark = pytest.mark.gpu
TH = 1.5
INTR = [500.0, 500.0, 320.0, 240.0, 500.0, 500.0, 320.0, 240.0]


def _scene(seed=0, n=1000, ratio=0.5, noise=0.5, **kw):
    sc = synthetic_two_view(seed, n, ratio, noise, **kw)
    return sc, np.concatenate([sc['pts1'], sc['pts2']], 1)


def _near(E, cam, th2):
    e = P.errors(E, cam)[0]
    return ~(np.abs(e - th2) > RB.decision_bound(3, E, cam, th2))


def _canon(M):
    M = np.asarray(M, dtype=np.float64).reshape(9)
    M = M / np.linalg.norm(M)
    return M * np.sign(M[np.argmax(np.abs(M))])


def _well_conditioned(cam, hyp, seed):
    """The oracle's rating of a sample: its 5 x 9 system has a clear rank gap and the real roots of the degree-10
    polynomial are well separated from each other and from complex pairs."""
    idx, ok = P.V.draw_samples(seed, [hyp], cam.shape[0], P.SAMPLE)
    if not ok[0]:
        return False
    A = P.V.f7_rows(cam[idx])
    sv = np.linalg.svd(A[0], compute_uv=False)
    if sv[-1] < 1e-4 * sv[0]:
        return False
    ns, _ = P.V.null_space(A)
    Bm, okg = P.gauss_jordan(P.constraints(ns))
    if not okg[0]:
        return False
    _, d = P.degree10(Bm)
    r = np.roots(d[0, ::-1])
    real = r[np.abs(r.imag) == 0].real
    near_real = r[np.abs(r.imag) < 1e-3 * (1 + np.abs(r.real))]
    if len(near_real) != len(real) or (np.abs(real) > 1e3).any():
        return False
    re = np.sort(real)
    return len(re) < 2 or np.diff(re).min() > 1e-3 * (1 + np.abs(re).max())


def test_essential_hypotheses_match_oracle():
    from patch2pix_b200.pose import first_essential_hypotheses
    sc, rows = _scene(seed=1)
    count, seed = 1024, 3
    gm, gc = first_essential_hypotheses(sc['pts1'], sc['pts2'], sc['K1'], sc['K2'], TH, count, seed=seed)
    cam = P.to_camera(rows, INTR)
    th2 = P.threshold(TH, INTR) ** 2
    om, ov = P.hypotheses(cam, np.arange(count), seed)
    sl = P.SLOTS
    checked = models = 0
    for i in range(count):
        if not _well_conditioned(cam, i, seed):
            continue
        checked += 1
        o = [k for k in range(sl) if ov[i * sl + k]]
        g = [k for k in range(sl) if gc[i * sl + k] >= 0]
        assert len(o) == len(g), (i, o, g)
        for k in o:
            oc = _canon(om[i * sl + k])
            d = [np.abs(_canon(gm[i * sl + j]) - oc).max() for j in g]
            j = g[int(np.argmin(d))]
            assert min(d) < 1e-4, (i, k, min(d))
            cnt = int((P.errors(om[i * sl + k], cam)[0] < th2).sum())
            nb = int(_near(om[i * sl + k], cam, th2).sum())
            assert abs(int(gc[i * sl + j]) - cnt) <= nb, (i, k, gc[i * sl + j], cnt, nb)
            models += 1
    assert checked > 0.5 * count and models > checked, (checked, models)


def _compare_final(rows, intr, gmask, th, seed=0, **kw):
    """GPU mask against the oracle's, except near-threshold rows, when the oracle's winning margin exceeds their
    number.  Returns whether the comparison applied."""
    tr = {}
    E, omask, _ = P.find_essential(rows, intr, th, seed=seed, trace=tr, **kw)
    assert E is not None
    near = _near(E, P.to_camera(rows, intr), P.threshold(th, intr) ** 2)
    if tr['margin'] <= int(near.sum()):
        return False
    diff = gmask != omask
    assert not (diff & ~near).any(), (np.nonzero(diff & ~near)[0][:10], tr)
    return True


@pytest.mark.parametrize('ratio', [0.3, 0.6])
def test_final_mask_and_pose_match_oracle_and_opencv(ratio):
    cv2 = pytest.importorskip('cv2')
    from patch2pix_b200.pose import find_essential_matrix, recover_pose
    sc, rows = _scene(seed=2, ratio=ratio)
    E, mask = find_essential_matrix(sc['pts1'], sc['pts2'], sc['K1'], sc['K2'], TH, seed=4)
    assert E is not None and E.shape == (3, 3) and E.dtype == np.float64 and mask.dtype == bool
    assert abs(np.linalg.norm(E) - 1) < 1e-12
    applied = _compare_final(rows, INTR, mask, TH, seed=4)
    lab = sc['inlier']
    assert (mask & lab).sum() >= 0.9 * lab.sum()
    assert applied or abs(int(mask.sum()) - int(P.find_essential(rows, INTR, TH, seed=4)[2])) <= 3
    # pose recovery on the GPU's own E
    n, R, t, good = recover_pose(E, sc['pts1'], sc['pts2'], sc['K1'], sc['K2'], mask)
    on, oR, ot, ogood = P.recover_pose(E, rows, INTR, mask)
    cn, cR, ct, cm = cv2.recoverPose(E, sc['pts1'], sc['pts2'], sc['K1'], mask=mask.astype(np.uint8).copy())
    assert n == on == cn and np.array_equal(good, ogood) and np.array_equal(good, cm.ravel() > 0)
    assert np.abs(R - oR).max() < 1e-9 and np.abs(t.ravel() - ot).max() < 1e-9
    assert np.abs(R - cR).max() < 1e-9 and np.abs(t - ct).max() < 1e-9
    assert not (good & ~mask).any()


def test_matches2relapose_with_different_focal_lengths():
    from patch2pix_b200.pose import matches2relapose
    sc, _ = _scene(seed=6, n=800, ratio=0.4, focal2=650.0)
    K1, K2 = sc['K1'], sc['K2']
    E, inls, R, t = matches2relapose(sc['pts1'], sc['pts2'], K1, K2, rthres=TH)
    # the reference's rescaling (geometry.py:35-45) fed to the oracle
    f1, f2 = K1[0, 0], K2[0, 0]
    p1 = (sc['pts1'] - K1[:2, 2][None]) * f2 / f1
    p2 = sc['pts2'] - K2[:2, 2][None]
    rows = np.concatenate([p1, p2], 1)
    intr = [f2, f2, 0.0, 0.0, f2, f2, 0.0, 0.0]
    mask = np.zeros(len(rows), dtype=bool)
    mask[inls] = True
    applied = _compare_final(rows, intr, mask, TH, max_iters=1000)
    oE, omask, _ = P.find_essential(rows, intr, TH, max_iters=1000)
    _, oR, ot, _ = P.recover_pose(oE, rows[omask], intr)
    ang = np.degrees(np.arccos(np.clip((np.trace(R.T @ oR) - 1) / 2, -1, 1)))
    if applied and np.array_equal(mask, omask):
        assert ang < 1e-4 and np.abs(t.ravel() - ot).max() < 1e-6
    assert ang < 0.5
    # and both are near the scene's pose
    assert np.degrees(np.arccos(np.clip((np.trace(R.T @ sc['R']) - 1) / 2, -1, 1))) < 1.0
    assert np.dot(t.ravel(), sc['t'] / np.linalg.norm(sc['t'])) > np.cos(np.radians(4.0))


def test_results_are_deterministic():
    from patch2pix_b200 import _lib
    from patch2pix_b200.pose import find_essential_matrix, recover_pose
    h = _lib.default_handle(torch.device('cuda', torch.cuda.current_device()))
    sc, _ = _scene(seed=5, n=3000, ratio=0.6)
    p1 = torch.from_numpy(sc['pts1']).cuda()
    p2 = torch.from_numpy(sc['pts2']).cuda()
    outs = []
    for sms in (0, 0, 66):
        h.set_option('num_sms', sms)
        E, mask = find_essential_matrix(p1, p2, sc['K1'], sc['K2'], TH, seed=7)
        n, R, t, good = recover_pose(E, p1, p2, sc['K1'], sc['K2'], mask)
        outs.append(tuple(x.cpu().numpy().tobytes() for x in (E, mask, n, R, t, good)))
    h.set_option('num_sms', 0)
    assert outs[0] == outs[1] == outs[2]


def test_edge_cases():
    from patch2pix_b200.pose import find_essential_matrix, recover_pose
    K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 500, (4, 2))
    E, mask = find_essential_matrix(p, p + 3.0, K, K, 1.0)
    assert E is None and mask.shape == (4,) and not mask.any()
    E, mask = find_essential_matrix(np.zeros((0, 2)), np.zeros((0, 2)), K, K, 1.0)
    assert E is None and mask.shape == (0,)
    q = rng.uniform(0, 500, (100, 2))
    q[17, 1] = np.nan
    with pytest.raises(ValueError):
        find_essential_matrix(q, q + 1.0, K, K, 1.0)
    Et, mt = find_essential_matrix(torch.from_numpy(q).cuda(), torch.from_numpy(q + 1.0).cuda(), K, K, 1.0)
    assert torch.isnan(Et).all() and not mt.any()
    with pytest.raises(RuntimeError):
        find_essential_matrix(p, p, K * np.array([[-1.0], [1], [1]]), K, 1.0)     # negative focal length
    # a zero E gives no pose
    sc, _ = _scene(seed=3, n=200, ratio=0.2)
    n, R, t, good = recover_pose(np.zeros((3, 3)), sc['pts1'], sc['pts2'], sc['K1'], sc['K2'])
    assert n == 0 and not R.any() and not t.any() and not good.any()
    # 2^20 rows with a small iteration budget
    sc, rows = _scene(seed=8, n=1 << 20, ratio=0.3)
    E, mask = find_essential_matrix(sc['pts1'], sc['pts2'], sc['K1'], sc['K2'], TH, max_iters=64)
    lab = sc['inlier']
    assert E is not None and mask.shape == (1 << 20,)
    assert (mask & lab).sum() >= 0.95 * lab.sum() and (mask & ~lab).sum() <= 0.02 * (~lab).sum()
    n, R, t, good = recover_pose(E, sc['pts1'], sc['pts2'], sc['K1'], sc['K2'], mask)
    assert n >= 0.95 * (mask & lab).sum()
    assert np.degrees(np.arccos(np.clip((np.trace(R.T @ sc['R']) - 1) / 2, -1, 1))) < 0.5


def test_estimate_matches_pose_pipeline(consensus_sd):
    from patch2pix_b200.eval_helper import _finalize, estimate_matches, load_model
    from patch2pix_b200.synth import shifted_pair_offset, synthetic_pair_shifted
    net = load_model(consensus_sd)
    im1, im2 = synthetic_pair_shifted(2, 240, 320)
    dx, dy = shifted_pair_offset(2)
    K = np.array([[320.0, 0, 160], [0, 320.0, 120], [0, 0, 1]])
    m, s, c, inl, E, R, t = estimate_matches(net, im1, im2, eval_type='coarse', verify=('E', 1.0, K, K))
    m0, s0, c0 = estimate_matches(net, im1, im2, eval_type='coarse')
    assert np.array_equal(m, m0) and np.array_equal(s, s0) and np.array_equal(c, c0)
    assert E is not None and inl.shape == (len(m),) and inl.dtype == bool
    # the second view is the first shifted by (-dx, -dy) px: a camera translation parallel to the image plane
    assert np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))) < 2.0, R
    shift = np.array([dx, dy, 0.0]) / np.hypot(dx, dy)
    assert abs(np.dot(t.ravel(), shift)) > np.cos(np.radians(5.0)), (t.ravel(), dx, dy)
    exact = (m[:, 2] - m[:, 0] == -dx) & (m[:, 3] - m[:, 1] == -dy)
    assert exact.sum() > 20 and inl[exact].mean() >= 0.9
    # pose estimation adds no device->host copy
    with torch.no_grad():
        cm, sc = net.predict_coarse(im1.cuda(), im2.cuda())
    up = (1.0, 1.0, 1.0, 1.0)
    _, n_tail = _dtoh(lambda: _finalize(net, None, sc[0], cm[0], float('-inf'), up, ('E', 1.0, K, K)))
    _, n_plain = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse'))
    _, n_pose = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse', verify=('E', 1.0, K, K)))
    assert n_tail == 1 and n_pose == n_plain
