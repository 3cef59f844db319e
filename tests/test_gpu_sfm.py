"""The Aachen triangulation and localization on the GPU (csrc/sfm.cu, patch2pix_b200/sfm.py) against the numpy oracle
(oracle/sfm_oracle.py), stage by stage on seeded noisy matches with outliers and distortion; determinism across runs
and chunkings; ground-truth matches; a seeded Patch2PixB200 against the host composition; failure handling."""
import os

import numpy as np
import pytest
import torch

from oracle import sfm_oracle as O
from patch2pix_b200 import localize as L
from patch2pix_b200 import sfm as S
from patch2pix_b200.synth import aachen_gt_matcher, synthetic_aachen_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return synthetic_aachen_tree(str(tmp_path_factory.mktemp('aachen')), 4, 6, 4)


def _noisy(tree, seed, step=6):
    """Ground-truth matches with 0.5 px noise, 10 % outliers, some duplicates and a few invalid endpoints."""
    rng = np.random.default_rng(seed)
    match = aachen_gt_matcher(tree, step=step)
    pairs = S.read_pairs(tree['db_pairs'])
    out = []
    for a, b in pairs:
        m = match(os.path.join(tree['images'], a), os.path.join(tree['images'], b))
        m = m + rng.normal(0, 0.5, m.shape)
        bad = rng.random(len(m)) < 0.1
        m[bad, 2:] = rng.uniform(0, 320, (bad.sum(), 2)) * [1, 0.75]
        m = np.concatenate([m, m[rng.integers(0, len(m), 20)]])
        m[rng.integers(0, len(m), 3), 0] = np.nan
        m[rng.integers(0, len(m), 3), 3] = -1.0
        out.append(np.clip(m, -5, None))
    return pairs, out


def _tables(tree, pairs):
    cameras, images, cams, img_cam, recs = S._model_tables(tree['model'])
    return (cams, img_cam, recs), S._pair_tables(images, cams, img_cam, recs, pairs, 4.0), images


def test_stages_match_oracle(tree):
    pairs, mt = _noisy(tree, 0)
    mtab, ptab, images = _tables(tree, pairs)
    ref = O.triangulate_host(mtab, ptab, mt)
    sfm = S.triangulate_from_matches(tree['model'], pairs, mt)
    # keypoints: ids, means and keys bit for bit
    np.testing.assert_array_equal(sfm.kp_key, ref['kp_key'])
    assert np.array_equal(sfm.kp_xy.view(np.int64), ref['kp_xy'].view(np.int64))
    assert sfm.stats['n_dropped_endpoints'] == ref['dropped'] > 0
    assert sfm.stats['n_edges'] == len(ref['edges'])
    assert sfm.stats['n_tracks'] == len(ref['tracks'])
    # components: scipy as a second opinion on the oracle's union-find
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    e = np.array(ref['edges']).reshape(-1, 2)
    n = len(ref['kp_xy'])
    _, lab = connected_components(coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n)), directed=False)
    first = {}
    for i, l in enumerate(lab):
        first.setdefault(l, i)
    np.testing.assert_array_equal(ref['labels'], [first[l] for l in lab])
    # points within 1e-9 relative, the same keypoint -> point assignment
    assert len(sfm.points) == len(ref['points']) > 100
    np.testing.assert_allclose(sfm.points, ref['points'], rtol=1e-9, atol=0)
    np.testing.assert_array_equal(sfm.kp_point, ref['kp_point'])
    np.testing.assert_array_equal(sfm.point_len, ref['point_len'])
    np.testing.assert_allclose(sfm.point_err, ref['point_err'], rtol=1e-9)


def test_query_rows_match_oracle(tree):
    from patch2pix_b200 import _lib
    import ctypes as C
    pairs, mt = _noisy(tree, 1)
    sfm = S.triangulate_from_matches(tree['model'], pairs, mt)
    qs = S.read_queries_with_intrinsics(tree['queries'])
    ret = L.read_retrieval(tree['query_pairs'])
    rng = np.random.default_rng(2)
    match = aachen_gt_matcher(tree, step=5)
    qm, pimg = [], []
    for k, (q, dbs) in enumerate(ret):
        for d in dbs:
            m = match(os.path.join(tree['images'], q), os.path.join(tree['images'], d))
            m = m + rng.normal(0, 1.0, m.shape)
            qm.append(np.clip(m, -2, None))
            pimg.append((k, sfm.index[d]))
    cams = [S.camera_record(qs[q].model, qs[q].params) for q, _ in ret]
    rows_ref, off_ref = O.query_rows(qm, pimg, cams, sfm.kp_xy, sfm.kp_key, sfm.kp_point, sfm.points, 4.0)
    # the device rows through the same entry points localize_from_matches uses
    dev = torch.device('cuda')
    h = _lib.default_handle(dev)
    lib, st = h.lib, h.stream()
    kp_key, kp_xy, kp_point, pts = sfm.device_arrays(dev)
    offsets = np.concatenate([[0], np.cumsum([len(m) for m in qm])]).astype(np.int64)
    M, P, K = int(offsets[-1]), len(qm), len(ret)
    m4 = torch.from_numpy(np.concatenate(qm)).to(dev)
    off_d = torch.from_numpy(offsets).to(dev)
    pim_d = torch.from_numpy(np.array(pimg, np.int32).reshape(-1)).to(dev)
    cams_d = torch.from_numpy(np.stack(cams)).to(dev)
    intr_d = torch.from_numpy(np.stack(cams)[:, 1:5].copy()).to(dev)
    qcam = torch.arange(K, dtype=torch.int32, device=dev)
    q_xy = torch.empty(M, 2, dtype=torch.float64, device=dev)
    q_key = torch.empty(M, dtype=torch.int64, device=dev)
    q_of = torch.empty(M, dtype=torch.int32, device=dev)
    q_n = torch.empty(M, 2, dtype=torch.float64, device=dev)
    cnt = torch.zeros(2, dtype=torch.int64, device=dev)
    rows = torch.empty(M, 5, dtype=torch.float64, device=dev)
    q_off = torch.empty(K + 1, dtype=torch.int64, device=dev)
    p = _lib.ptr
    _lib.check(lib.p2p_sfm_keypoints(h.h, p(m4), M, p(off_d), P, p(pim_d), 0, 4.0, p(q_xy), p(q_key), p(q_of), p(cnt),
                                     st))
    _lib.check(lib.p2p_sfm_undistort(h.h, p(q_xy), p(q_key), M, p(cnt), p(qcam), p(cams_d), p(q_n), st))
    _lib.check(lib.p2p_sfm_query_rows(h.h, p(m4), M, p(off_d), P, p(pim_d), K, 4.0, p(q_of), p(q_key), p(q_n),
                                      p(intr_d), p(kp_key), p(kp_xy), p(kp_point), len(sfm.kp_key), p(pts), p(rows),
                                      p(q_off), st))
    off = q_off.cpu().numpy()
    np.testing.assert_array_equal(off, off_ref)
    got = rows[:off[-1]].cpu().numpy()
    assert len(got) > 100 and np.array_equal(got.view(np.int64), rows_ref.view(np.int64))


def test_determinism_and_chunking(tree, tmp_path):
    match = aachen_gt_matcher(tree, step=6)
    kw = dict(lprint_=lambda s: None)
    a = S.localize_aachen(match, tree['images'], tree['model'], tree['db_pairs'], tree['query_pairs'],
                          tree['queries'], str(tmp_path / 'a.txt'), **kw)
    b = S.localize_aachen(match, tree['images'], tree['model'], tree['db_pairs'], tree['query_pairs'],
                          tree['queries'], str(tmp_path / 'b.txt'), chunk_pairs=1, chunk_queries=1, **kw)
    for k in ('kp_xy', 'kp_key', 'kp_point', 'points', 'point_len', 'point_err'):
        assert np.array_equal(getattr(a['sfm'], k), getattr(b['sfm'], k)), k
    for n, (R, t, c) in a['poses'].items():
        assert np.array_equal(b['poses'][n][0], R) and np.array_equal(b['poses'][n][1], t) and b['poses'][n][2] == c
    assert open(tmp_path / 'a.txt').read() == open(tmp_path / 'b.txt').read()
    # exact matches at the defaults: every query within Aachen's middle bin.  The finest bin is not reached by every
    # query: the scene is one plane, and at 12 px, far above the noise, the P3P RANSAC keeps its sample's pose
    assert not a['failed'] and not a['failed_pairs']
    ev = L.eval_localization(str(tmp_path / 'a.txt'), tree['gt'], thresholds=S.AACHEN_THRESHOLDS)
    assert ev['recall'][(0.5, 5.0)] == 1.0 and ev['recall'][(0.25, 2.0)] >= 0.75, ev['errors']
    # the written model reads back to the same localization
    a['sfm'].write(str(tmp_path / 'sfm'))
    back = S.load_sfm_model(str(tmp_path / 'sfm'))
    np.testing.assert_array_equal(back.kp_key, a['sfm'].kp_key)
    c = S.localize_sfm(match, back, tree['images'], tree['queries'], tree['query_pairs'], str(tmp_path / 'c.txt'),
                       **kw)
    assert open(tmp_path / 'c.txt').read() == open(tmp_path / 'a.txt').read() and c['n_queries'] == 4


def test_ground_truth_points_on_surface(tree):
    match = aachen_gt_matcher(tree, step=7)
    pairs = S.read_pairs(tree['db_pairs'])
    mt = [match(os.path.join(tree['images'], a), os.path.join(tree['images'], b)) for a, b in pairs]
    sfm = S.triangulate_from_matches(tree['model'], pairs, mt, merge_px=1e-4)
    sc = tree['scene']
    assert len(sfm.points) > 100
    dist = np.abs((sfm.points - sc['O']) @ sc['n'])
    assert dist.max() < 1e-6 * 7.0, dist.max()          # relative to the 5-7 m from the cameras to the plane


def test_failures_stay_local(tree, tmp_path):
    match = aachen_gt_matcher(tree, step=6)
    pairs = S.read_pairs(tree['db_pairs'])

    def flaky(p0, p1):
        if p0.endswith(pairs[1][0]) and p1.endswith(pairs[1][1]):
            raise RuntimeError('db boom')
        if p0.endswith('query/0002.png'):
            raise RuntimeError('query boom')
        return match(p0, p1)
    res = S.localize_aachen(flaky, tree['images'], tree['model'], tree['db_pairs'], tree['query_pairs'],
                            tree['queries'], str(tmp_path / 'r.txt'), lprint_=lambda s: None)
    assert [p for p, _ in res['failed_pairs']] == [pairs[1]]
    assert [q for q, _ in res['failed']] == ['query/0002.png']
    w = L.read_results(str(tmp_path / 'r.txt'))
    assert len(w) == 4 and np.array_equal(w['0002.png'][0], np.eye(3)) and not w['0002.png'][1].any()
    # the model without pair 1 is the model of the other pairs' matches
    rest = [p for i, p in enumerate(pairs) if i != 1]
    ref = S.triangulate_from_matches(tree['model'], rest, [match(os.path.join(tree['images'], a),
                                                                 os.path.join(tree['images'], b)) for a, b in rest])
    assert np.array_equal(res['sfm'].points, ref.points)


def test_patch2pix_matches_host_composition(tree, tmp_path):
    from patch2pix_b200.eval_helper import estimate_matches_from_files, load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    net = load_model(make_seeded_state_dict(0, nc_init='consensus'))
    kw = dict(ksize=2, io_thres=0.25, imsize=320)
    res = S.localize_aachen(net, tree['images'], tree['model'], tree['db_pairs'], tree['query_pairs'],
                            tree['queries'], str(tmp_path / 'r.txt'), chunk_pairs=4, chunk_queries=3,
                            lprint_=lambda s: None, **kw)

    def em(a, b):
        return estimate_matches_from_files(net, os.path.join(tree['images'], a), os.path.join(tree['images'], b),
                                           kw['ksize'], 0.0, True, kw['io_thres'], 'fine', kw['imsize'])[0]
    pairs = S.read_pairs(tree['db_pairs'])
    sfm = S.triangulate_from_matches(tree['model'], pairs, [em(a, b) for a, b in pairs])
    ret = L.read_retrieval(tree['query_pairs'])
    host = S.localize_from_matches(sfm, tree['queries'], ret, [em(q, d) for q, dbs in ret for d in dbs],
                                   str(tmp_path / 'h.txt'))
    assert sfm.stats['n_matches'] > 0
    for k in ('kp_xy', 'kp_key', 'kp_point', 'points'):
        assert np.array_equal(getattr(res['sfm'], k), getattr(sfm, k)), k
    assert [q for q, _ in res['failed']] == [q for q, _ in host['failed']]
    for n, (R, t, c) in host['poses'].items():
        assert np.array_equal(res['poses'][n][0], R) and np.array_equal(res['poses'][n][1], t), n
