"""GPU match verification (p2p_find_model / p2p_sampson_distance) against the numpy oracle (oracle/verify_oracle.py).

The device scores in fp32 and the oracle in fp64, so inlier decisions may differ on rows whose error lies within the
derived per-row bound of oracle/ransac_bound.py (decision_bound) of px_th^2; every comparison below exempts exactly those
rows and nothing else."""
import numpy as np
import pytest
import torch

from oracle import ransac_bound as RB
from oracle import verify_oracle as V
from patch2pix_b200.synth import synthetic_two_view

pytestmark = pytest.mark.gpu


def _scene(kind, seed=0, n=1000, ratio=0.5, noise=0.5):
    sc = synthetic_two_view(seed, n, ratio, noise, planar=kind == 1)
    return sc, np.concatenate([sc['pts1'], sc['pts2']], 1)


def _near(kind, model, rows, th2):
    e = V.errors(kind, model, rows)[0]
    return ~(np.abs(e - th2) > RB.decision_bound(kind, model, rows, th2))


def _canon(M):
    M = np.asarray(M, dtype=np.float64).reshape(9)
    M = M / np.linalg.norm(M)
    return M * np.sign(M[np.argmax(np.abs(M))])


def _well_conditioned(kind, rows, T, hyp, seed):
    """The oracle's rating of a sample: its linear system has a clear rank gap, no near-collinear triple (H), and the
    real roots of the cubic are well separated (F)."""
    s = V.SAMPLE[kind]
    idx, ok = V.draw_samples(seed, [hyp], rows.shape[0], s)
    if not ok[0]:
        return False
    P = V.normalise(rows[idx], T)
    A = (V.f7_rows(P) if kind == 0 else V.h4_rows(P))[0]
    sv = np.linalg.svd(A, compute_uv=False)
    if sv[-1] < 1e-4 * sv[0]:
        return False
    if kind == 1:
        for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
            for i in (0, 2):
                o = (P[0, b, i] - P[0, a, i]) * (P[0, c, i + 1] - P[0, a, i + 1]) - \
                    (P[0, b, i + 1] - P[0, a, i + 1]) * (P[0, c, i] - P[0, a, i])
                if abs(o) < 1e-3:
                    return False
        return True
    ns, _ = V.null_space(A[None])
    N1, N2 = ns[0]
    D = N1 - N2
    v = [np.linalg.det((N2 + l * D).reshape(3, 3)) for l in (0.0, 1.0, -1.0, 2.0)]
    a2 = 0.5 * (v[1] + v[2]) - v[0]
    odd = 0.5 * (v[1] - v[2])
    a3 = (v[3] - v[0] - 4 * a2 - 2 * odd) / 6
    r = np.roots([a3, a2, odd - a3, v[0]])
    if np.abs(a3) < 1e-6 * max(abs(a2), abs(odd), abs(v[0])):
        return False
    near_real = r[np.abs(r.imag) < 1e-3 * (1 + np.abs(r.real))]
    real = r[np.abs(r.imag) == 0]
    if len(near_real) != len(real):
        return False
    re = np.sort(real.real)
    return len(re) < 2 or np.diff(re).min() > 1e-3 * (1 + np.abs(re).max())


@pytest.mark.parametrize('kind, th', [(0, 1.0), (1, 2.0)])
def test_hypotheses_match_oracle(kind, th):
    from patch2pix_b200.verify import first_hypotheses
    sc, rows = _scene(kind, seed=1)
    count, seed, th2 = 2048, 3, th * th
    gm, gc = first_hypotheses(kind, sc['pts1'], sc['pts2'], th, count, seed=seed)
    T = V.normalisation(rows)
    om, ov = V.hypotheses(kind, rows, T, np.arange(count), seed)
    sl = V.SLOTS[kind]
    checked = models = 0
    for i in range(count):
        if not _well_conditioned(kind, rows, T, i, seed):
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
            cnt = int((V.errors(kind, om[i * sl + k], rows)[0] < th2).sum())
            nb = int(_near(kind, om[i * sl + k], rows, th2).sum())
            assert abs(int(gc[i * sl + j]) - cnt) <= nb, (i, k, gc[i * sl + j], cnt, nb)
            models += 1
    assert checked > 0.5 * count and models > 0.25 * count, (checked, models)


def _compare_final(kind, rows, gmask, th, seed=0, **kw):
    """GPU mask against the oracle's, except near-threshold rows, when the oracle's winning margin exceeds their
    number.  Returns whether the comparison applied."""
    tr = {}
    M, omask, c = V.find_model(kind, rows, th, seed=seed, trace=tr, **kw)
    assert M is not None
    near = _near(kind, M, rows, th * th)
    if tr['margin'] <= int(near.sum()):
        return False
    diff = gmask != omask
    assert not (diff & ~near).any(), (np.nonzero(diff & ~near)[0][:10], tr)
    return True


@pytest.mark.parametrize('kind, th, ratio', [(0, 1.0, 0.3), (0, 1.0, 0.6), (1, 2.0, 0.3), (1, 2.0, 0.7)])
def test_final_result_matches_oracle(kind, th, ratio):
    from patch2pix_b200.verify import find_fundamental_matrix, find_homography
    sc, rows = _scene(kind, seed=2, ratio=ratio)
    fn = find_fundamental_matrix if kind == 0 else find_homography
    M, mask = fn(sc['pts1'], sc['pts2'], th, seed=4)
    assert M is not None and M.shape == (3, 3) and M.dtype == np.float64 and mask.dtype == bool
    applied = _compare_final(kind, rows, mask, th, seed=4)
    # sanity bound only (the oracle comparison above is the check): even the true model keeps P(chi2(1) < 4) = 0.954 of
    # the F inliers at 1 px and sigma 0.5 px, and an estimated F a few percent fewer
    lab = sc['inlier']
    assert (mask & lab).sum() >= 0.85 * lab.sum()
    assert applied or abs(int(mask.sum()) - int(V.find_model(kind, rows, th, seed=4)[2])) <= 3


def test_results_are_deterministic():
    from patch2pix_b200 import _lib
    from patch2pix_b200.verify import find_fundamental_matrix, find_homography
    h = _lib.default_handle(torch.device('cuda', torch.cuda.current_device()))
    for kind, fn, th in ((0, find_fundamental_matrix, 1.0), (1, find_homography, 2.0)):
        sc, _ = _scene(kind, seed=5, n=3000, ratio=0.6)
        p1 = torch.from_numpy(sc['pts1']).cuda()
        p2 = torch.from_numpy(sc['pts2']).cuda()
        outs = []
        for sms in (0, 0, 66):
            h.set_option('num_sms', sms)
            M, mask = fn(p1, p2, th, seed=7)
            outs.append((M.cpu().numpy().tobytes(), mask.cpu().numpy().tobytes()))
        h.set_option('num_sms', 0)
        assert outs[0] == outs[1] == outs[2]


def test_edge_cases():
    from patch2pix_b200.verify import find_fundamental_matrix, find_homography
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 500, (6, 2))
    M, mask = find_fundamental_matrix(p, p + 3.0, 1.0)
    assert M is None and mask.shape == (6,) and not mask.any()
    M, mask = find_homography(p[:3], p[:3] + 3.0, 1.0)
    assert M is None and not mask.any()
    M, mask = find_homography(np.zeros((0, 2)), np.zeros((0, 2)), 1.0)
    assert M is None and mask.shape == (0,)
    q = rng.uniform(0, 500, (100, 2))
    q[17, 1] = np.nan
    with pytest.raises(ValueError):
        find_fundamental_matrix(q, q + 1.0, 1.0)
    q[17, 1] = np.inf
    with pytest.raises(ValueError):
        find_homography(q, q + 1.0, 1.0)
    # CUDA tensor input: NaN model on non-finite input, zero model without one
    Mt, mt = find_homography(torch.from_numpy(q).cuda(), torch.from_numpy(q + 1.0).cuda(), 1.0)
    assert torch.isnan(Mt).all() and not mt.any()
    Mt, mt = find_fundamental_matrix(torch.from_numpy(p).cuda(), torch.from_numpy(p).cuda(), 1.0)
    assert (Mt == 0).all() and not mt.any()
    # 2^20 rows
    sc, _ = _scene(1, seed=8, n=1 << 20, ratio=0.5)
    M, mask = find_homography(sc['pts1'], sc['pts2'], 2.0, max_iters=2048)
    lab = sc['inlier']
    assert M is not None and mask.shape == (1 << 20,)
    assert (mask & lab).sum() >= 0.95 * lab.sum() and (mask & ~lab).sum() <= 0.01 * (~lab).sum()


def test_sampson_distance_matches_oracle():
    from patch2pix_b200.verify import sampson_distance
    sc, rows = _scene(0, seed=9, n=5000, ratio=0.5, noise=1.0)
    d = sampson_distance(sc['pts1'], sc['pts2'], sc['F'])
    np.testing.assert_allclose(d, V.sampson_distance(rows, sc['F']), rtol=1e-9, atol=1e-18)
    dt = sampson_distance(torch.from_numpy(sc['pts1']).cuda(), torch.from_numpy(sc['pts2']).cuda(),
                          torch.from_numpy(sc['F']).cuda())
    assert dt.is_cuda and np.array_equal(dt.cpu().numpy(), d)


def _dtoh(fn):
    """fn()'s result and the device->host copies it made.  The profiler can drop the device activity a session records
    first: on an H100, after earlier sessions in the same process, every other session lost a short call's kernels and
    copy.  So the window opens with copy-free matmuls and fn() runs after them."""
    from torch.profiler import ProfilerActivity, profile
    pad = torch.full((2048, 2048), 1.0 / 2048, device='cuda')
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(60):
            pad = pad @ pad
        out = fn()
        torch.cuda.synchronize()
    return out, sum(1 for e in prof.events() if 'Memcpy DtoH' in e.name)


def test_estimate_matches_verify_pipeline(consensus_sd):
    from patch2pix_b200.eval_helper import _finalize, estimate_matches, load_model
    from patch2pix_b200.synth import shifted_pair_offset, synthetic_pair_shifted
    net = load_model(consensus_sd)
    im1, im2 = synthetic_pair_shifted(2, 240, 320)
    dx, dy = shifted_pair_offset(2)
    m, s, c, inl, H = estimate_matches(net, im1, im2, eval_type='coarse', verify=('H', 2.0))
    m0, s0, c0 = estimate_matches(net, im1, im2, eval_type='coarse')
    assert np.array_equal(m, m0) and np.array_equal(s, s0) and np.array_equal(c, c0)
    assert H is not None and inl.shape == (len(m),) and inl.dtype == bool
    corners = np.array([[0, 0, 1], [319, 0, 1], [0, 239, 1], [319, 239, 1]], dtype=np.float64)
    mapped = corners @ H.T
    mapped = mapped[:, :2] / mapped[:, 2:3]
    assert np.abs(mapped - (corners[:, :2] - [dx, dy])).max() < 0.5, (H, dx, dy)
    exact = (m[:, 2] - m[:, 0] == -dx) & (m[:, 3] - m[:, 1] == -dy)
    assert exact.sum() > 20 and inl[exact].mean() >= 0.9
    # verification adds no device->host copy: the tail after the matcher still copies exactly once
    with torch.no_grad():
        cm, sc = net.predict_coarse(im1.cuda(), im2.cuda())
    up = (1.0, 1.0, 1.0, 1.0)
    _, n_tail = _dtoh(lambda: _finalize(net, None, sc[0], cm[0], float('-inf'), up, ('H', 2.0)))
    _, n_plain = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse'))
    _, n_ver = _dtoh(lambda: estimate_matches(net, im1, im2, eval_type='coarse', verify=('H', 2.0)))
    assert n_tail == 1 and n_ver == n_plain
    # fine: the seeded regressor is untrained, so the oracle on the same rows is the reference
    mf, sf, cf, inf_, Hf = estimate_matches(net, im1, im2, eval_type='fine', verify=('H', 2.0))
    mf0, _, _ = estimate_matches(net, im1, im2, eval_type='fine')
    assert np.array_equal(mf, mf0)
    if Hf is not None:
        _compare_final(1, mf, inf_, 2.0, seed=0)
