"""GPU side of the validation loop: p2p_epipolar_histograms against p2p_sampson_distance and a numpy oracle, and
eval_immatch_val_sets / eval_pairs end to end against a host recomputation through estimate_matches_from_files."""
import os

import numpy as np
import pytest
import torch

from patch2pix_b200 import evaluation as E
from patch2pix_b200 import pose as P
from patch2pix_b200.synth import synthetic_two_view, synthetic_val_scene
from patch2pix_b200.verify import epipolar_histograms, sampson_distance

pytestmark = pytest.mark.gpu
EDGE_BAND = 1e-12


def _np_sampson(rows, F):
    """utils/eval/measure.py:18-40 in numpy fp64."""
    p1 = np.concatenate([rows[:, 0:2], np.ones((len(rows), 1))], 1)
    p2 = np.concatenate([rows[:, 2:4], np.ones((len(rows), 1))], 1)
    l2, l1 = F @ p1.T, F.T @ p2.T
    dd = np.sum(l2.T * p2, 1)
    return dd ** 2 / (1e-8 + l1[0] ** 2 + l1[1] ** 2 + l2[0] ** 2 + l2[1] ** 2)


def _hist(d, edges):
    return np.append(np.histogram(d, edges)[0], len(d))


def _near_edge(d, edges):
    e = np.asarray(edges, dtype=np.float64)
    return (np.abs(d[:, None] - e[None, :]) <= EDGE_BAND * np.maximum(np.abs(e[None, :]), 1e-300)).any(1)


def _rows9(seed=0, n=3000):
    """[n, 9] rows as p2p_finalize_matches packs them: refined (x1, y1, x2, y2), a score, coarse (x1, y1, x2, y2)."""
    sc = synthetic_two_view(seed, n, 0.5, 1.0)
    rng = np.random.default_rng(seed)
    ref = np.concatenate([sc['pts1'], sc['pts2']], 1)
    rows = np.concatenate([ref, rng.random((n, 1)), ref + rng.normal(0, 4.0, (n, 4))], 1)
    return rows, sc['F'] * 1e3


@pytest.mark.parametrize('stride', [4, 9])
def test_histograms_equal_sampson_distance(stride):
    rows, F = _rows9()
    n = len(rows)
    rt = torch.from_numpy(np.ascontiguousarray(rows[:, :stride])).cuda()
    d = sampson_distance(rt[:, 0:2].contiguous(), rt[:, 2:4].contiguous(), torch.from_numpy(F).cuda()).cpu().numpy()
    dc = sampson_distance(torch.from_numpy(rows[:, 5:7]).cuda(), torch.from_numpy(rows[:, 7:9]).cuda(),
                          torch.from_numpy(F).cuda()).cpu().numpy()
    mask = np.random.default_rng(1).random(n) < 0.4
    edges = E.EVAL_BINS
    coarse = 5 if stride == 9 else -1
    for m in (n, 1234, 0):
        n_dev = torch.tensor(float(m), dtype=torch.float64, device='cuda')
        got = epipolar_histograms(rt, F, edges, coarse, torch.from_numpy(mask).cuda(), n_dev).cpu().numpy()
        assert np.array_equal(got[1], _hist(d[:m], edges)), m
        assert np.array_equal(got[2], _hist(d[:m][mask[:m]], edges)), m
        assert np.array_equal(got[0], _hist(dc[:m], edges) if coarse >= 0 else np.zeros(len(edges))), m
    got = epipolar_histograms(rt, F, edges).cpu().numpy()          # no mask, no n_dev, no coarse columns
    assert np.array_equal(got[1], _hist(d, edges)) and not got[0].any() and not got[2].any()
    empty = torch.zeros(0, stride, dtype=torch.float64, device='cuda')
    assert not epipolar_histograms(empty, F, edges, coarse).cpu().numpy().any()


def test_histograms_against_numpy_oracle():
    rows, F = _rows9(seed=3, n=20000)
    edges = E.EVAL_BINS
    mask = np.random.default_rng(2).random(len(rows)) < 0.5
    got = epipolar_histograms(torch.from_numpy(rows).cuda(), F, edges, 5, torch.from_numpy(mask).cuda()).cpu().numpy()
    for k, (d, sel) in enumerate(((_np_sampson(rows[:, 5:9], F), None), (_np_sampson(rows[:, :4], F), None),
                                  (_np_sampson(rows[:, :4], F), mask))):
        d = d if sel is None else d[sel]
        near = _near_edge(d, edges)
        exp = _hist(d, edges)
        assert got[k, -1] == exp[-1]
        assert np.abs(got[k, :-1] - exp[:-1]).sum() <= 2 * near.sum(), (k, got[k], exp)


def test_histograms_exact_values():
    """Rows with exact distances: F = [[0,0,0],[0,0,0],[0,a,0]] gives d = y1^2 (den = a^2 absorbs eps), and
    F = [[0,0,0],[0,0,a],[0,3a,0]] gives d = (y2 + 3 y1)^2 / 10 (den = 10 a^2), so y2 = 1000 lands on 1e5."""
    a = 2.0 ** 14
    edges = E.EVAL_BINS
    inf, nan = np.inf, np.nan
    F1 = np.array([[0, 0, 0], [0, 0, 0], [0, a, 0]], dtype=np.float64)
    y1 = np.array([0, 1, 50, 0.1, 1e3, 400, 316, 317, 10, 5, 2, 3])
    r1 = np.stack([np.full_like(y1, 7.0), y1, np.full_like(y1, 3.0), np.full_like(y1, 4.0)], 1)
    r1 = np.concatenate([r1, [[inf, 1, 2, 3], [1, nan, 2, 3], [1, 2, inf, 3], [nan, nan, nan, nan]]])
    F2 = np.array([[0, 0, 0], [0, 0, a], [0, 3 * a, 0]], dtype=np.float64)
    y2 = np.array([1000.0, 1001.0, 999.0, 2000.0, 0.0])
    r2 = np.stack([np.zeros_like(y2), np.zeros_like(y2), np.zeros_like(y2), y2], 1)
    for rows, F in ((r1, F1), (r2, F2)):
        d = _np_sampson(rows, F)
        got = epipolar_histograms(torch.from_numpy(rows).cuda(), F, edges).cpu().numpy()
        assert np.array_equal(got[1], _hist(d, edges)), (got[1], d)
    assert _np_sampson(r2[:1], F2)[0] == 1e5 and _np_sampson(r1[:3], F1).tolist() == [0.0, 1.0, 2500.0]


def test_invalid_edges_raise():
    rows = torch.zeros(4, 4, dtype=torch.float64, device='cuda')
    F = np.eye(3)
    for edges in ([1.0], list(range(17)), [0, 1, 1, 2], [0, 2, 1], [0, np.nan, 2], [0, 1, np.inf], [-np.inf, 0]):
        with pytest.raises(RuntimeError):
            epipolar_histograms(rows, F, edges)


def test_histograms_deterministic():
    from patch2pix_b200 import _lib
    rows, F = _rows9(seed=5, n=50000)
    rt = torch.from_numpy(rows).cuda()
    mask = torch.from_numpy(np.random.default_rng(0).random(len(rows)) < 0.3).cuda()
    h = _lib.default_handle(rt.device)
    outs = []
    for sms in (0, 0, 17, 132):
        h.set_option('num_sms', sms)
        outs.append(epipolar_histograms(rt, F, E.EVAL_BINS, 5, mask).cpu().numpy())
    h.set_option('num_sms', 0)
    assert all(np.array_equal(o, outs[0]) for o in outs)


# ---- end to end -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('val'))
    synthetic_val_scene(root, 'sceneA', 1, [(320, 240), (256, 192), (320, 256), (288, 224), (320, 240)])
    synthetic_val_scene(root, 'sceneB', 2, [(256, 192), (320, 240), (224, 160)], missing=(1,))
    return root


def _pairs(root, sample_max):
    np.random.seed(0)
    out = []
    for scene, ims, names in E.select_pairs(root, sample_max, 0.3):
        d = os.path.join(root, scene, 'dense/images')
        out += [(os.path.join(d, a), os.path.join(d, b), ims[a], ims[b]) for a, b in names]
    return out


KW = dict(ksize=2, io_thres=0.5, ncn_thres=0.0, imsize=1024, rthres=0.5)


@pytest.mark.parametrize('eval_type', ['fine', 'coarse'])
def test_eval_end_to_end_matches_host(net, tree, eval_type):
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    sample_max = 3
    pairs = _pairs(tree, sample_max)
    assert len(pairs) == 6                                  # sceneA cut to 3 of its 5 pairs, sceneB keeps its 3
    lines = []
    E.eval_immatch_val_sets(net, tree, eval_type=eval_type, sample_max=sample_max, lprint_=lines.append, **KW)
    recs = E.eval_pairs(net, pairs, eval_type=eval_type, **KW)
    assert sum(r.status == 'match_failed' for r in recs) == 1
    cd, fd, ind, nm, irat, qt, host_recs = [], [], [], [], [], [], []
    for (p1, p2, im1, im2), r in zip(pairs, recs):
        if not (os.path.exists(p1) and os.path.exists(p2)):
            assert r.status == 'match_failed'
            continue
        t_gt, q_gt = P.abs2relapose(im1.c, im2.c, im1.q, im2.q)
        F = P.pose2fund(im1.K, im2.K, P.quat2mat(q_gt), t_gt)
        m, _, c, inl, Em, R, t = estimate_matches_from_files(net, p1, p2, KW['ksize'], KW['ncn_thres'], True,
                                                             KW['io_thres'], eval_type, KW['imsize'],
                                                             verify=('E', KW['rthres'], im1.K, im2.K))
        cdist, fdist = _np_sampson(np.asarray(c), F), _np_sampson(np.asarray(m), F)
        if eval_type == 'coarse':
            assert np.array_equal(r.counts[0], r.counts[1])
        assert r.N == len(m)
        for k, d in ((0, cdist), (1, fdist)) + (((2, fdist[inl]),) if r.status == 'ok' else ()):
            exp = _hist(d, E.EVAL_BINS)
            assert r.counts[k, -1] == exp[-1]
            assert np.abs(r.counts[k, :-1] - exp[:-1]).sum() <= 2 * _near_edge(d, E.EVAL_BINS).sum(), (k, r.counts[k])
        cd.append(cdist)
        fd.append(fdist)
        nm.append(len(m))
        if Em is None:
            assert r.status == 'geo_failed'
            continue
        assert r.status == 'ok' and r.n_inls == inl.sum()
        assert np.array_equal(r.R, R) and np.array_equal(r.t, t)
        terr = P.cal_vec_angle_error(t.squeeze(), t_gt)
        qerr = P.cal_quat_angle_error(P.mat2quat(R), q_gt)
        assert abs(r.terr - terr) <= 1e-9 and abs(r.qerr - qerr) <= 1e-9
        ind.append(fdist[inl])
        irat.append(inl.sum() / len(m))
        qt.append(max(terr, qerr))
    n_ok = len(qt)
    assert n_ok >= 1
    expect = [f'Pairs {len(pairs)} match_failed=1 geo_failed={len(nm) - n_ok} num_matches={np.mean(nm):.2f} '
              f'irat={np.mean(irat):.3f} time:',
              E.check_inliers_distr(cd, bins=E.EVAL_BINS, tag='cdist'),
              E.check_inliers_distr(fd, bins=E.EVAL_BINS, tag='fdist', return_ratios=True)[1],
              E.check_inliers_distr(ind, bins=E.EVAL_BINS, tag='indist', return_ratios=True)[1]]
    pass_rate = np.array([100.0 * np.mean(np.array(qt) < thre) for thre in range(1, 11, 1)])
    expect.append('Pose err: qt_mean={:.2f}/{:.2f} qt<[1-10]deg:{}'.format(np.mean(qt), np.median(qt), pass_rate))
    assert lines[0].startswith('\n>>Eval on immatch: rthres=0.5 eval_type=' + eval_type)
    assert lines[1].startswith(expect[0]) and lines[2:] == expect[1:], (lines, expect)


def test_eval_device_to_host_copies(net, tree):
    from torch.profiler import ProfilerActivity, profile
    from patch2pix_b200.preprocess import load_im_flexible
    pairs = [p for p in _pairs(tree, 300) if os.path.exists(p[0]) and os.path.exists(p[1])][:3]

    def dtoh(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if 'Memcpy DtoH' in e.name)

    x1, _ = load_im_flexible(pairs[0][0], 2, net.upsample, imsize=1024, device=net.device, handle=net._handle)
    x2, _ = load_im_flexible(pairs[0][1], 2, net.upsample, imsize=1024, device=net.device, handle=net._handle)
    with torch.no_grad():
        net.predict_fine(x1.unsqueeze(0), x2.unsqueeze(0))           # warm-up
        n_pf = dtoh(lambda: net.predict_fine(x1.unsqueeze(0), x2.unsqueeze(0)))
    E.eval_pairs(net, pairs, **KW)                                    # warm-up
    n_eval = dtoh(lambda: E.eval_pairs(net, pairs, **KW))
    assert n_pf >= 1 and n_eval == len(pairs) * n_pf + 1, (n_pf, n_eval)
