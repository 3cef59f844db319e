"""localize_inloc end to end on synthetic InLoc-layout trees: with a seeded Patch2PixB200 it writes the poses of the host
composition (estimate_matches_from_files -> the oracle's scan lift -> find_absolute_poses), whatever the chunking;
with ground-truth matches every query is localized within the tightest threshold."""
import os

import numpy as np
import pytest

from oracle import abspose_oracle as A
from patch2pix_b200 import localize as L
from patch2pix_b200.synth import inloc_gt_matcher, synthetic_inloc_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


def test_patch2pix_matches_host_composition(net, tmp_path):
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    root = str(tmp_path)
    tree = synthetic_inloc_tree(root, 1, 3, 2)
    kw = dict(ksize=2, io_thres=0.25, imsize=320)
    res = L.localize_inloc(net, root, tree['pairs'], str(tmp_path / 'r.txt'), chunk_queries=2, lprint_=lambda s: None,
                           **kw)
    ret = L.read_retrieval(tree['pairs'])
    p2, p3, Ks = [], [], []
    for q, dbs in ret:
        rows = []
        for d in dbs:
            m = estimate_matches_from_files(net, os.path.join(root, q), os.path.join(root, d), kw['ksize'], 0.0,
                                            True, kw['io_thres'], 'fine', kw['imsize'])[0]
            rows.append(A.lift_scan(L.read_scan(os.path.join(root, d + '.mat')),
                                    L.read_alignment(L.alignment_path(root, d)), m))
        rows = np.concatenate(rows)
        p2.append(rows[:, :2])
        p3.append(rows[:, 2:])
        Ks.append([L.INLOC_FOCAL, L.INLOC_FOCAL, 160.0, 120.0])
    host = L.find_absolute_poses(p2, p3, Ks, 48.0)
    failed = {q for q, _ in res['failed']}
    written = L.read_results(str(tmp_path / 'r.txt'))
    assert len(written) == 3 and sum(len(r) for r in p2) > 0
    for (q, _), (R, t, _) in zip(ret, host):
        name = os.path.basename(q)
        Rg, tg, cnt = res['poses'][name]
        if R is None:
            assert q in failed and np.array_equal(Rg, np.eye(3)) and not tg.any()
        else:
            assert q not in failed and cnt > 0
            assert np.array_equal(Rg, R) and np.array_equal(tg, t), name
            assert np.abs(written[name][0] - R).max() < 1e-12 and np.abs(written[name][1] - t).max() < 1e-9


def test_ground_truth_matches_localize_every_query(tmp_path):
    root = str(tmp_path)
    tree = synthetic_inloc_tree(root, 2, 4, 3)
    matcher = inloc_gt_matcher(tree)
    out = str(tmp_path / 'r.txt')
    # 320 x 240 images at InLoc's focal length see 6 degrees of a plane: poses 0.5 m apart reproject every match within
    # a few pixels, so the exact matches are held to 1 px
    kw = dict(ransac_thres=1.0, lprint_=lambda s: None)
    res = L.localize_inloc(matcher, root, tree['pairs'], out, **kw)
    assert not res['failed'] and res['n_queries'] == 4
    ev = L.eval_localization(out, tree['gt'])
    assert ev['recall'][(0.25, 10.0)] == 1.0, ev['errors']
    # the chunking changes no pose; a matcher that raises fails only its query, written as the identity
    one = L.localize_inloc(matcher, root, tree['pairs'], str(tmp_path / 'r1.txt'), chunk_queries=1, **kw)
    for n, (R, t, c) in res['poses'].items():
        assert np.array_equal(one['poses'][n][0], R) and np.array_equal(one['poses'][n][1], t)

    def flaky(q, d):
        if q.endswith('IMG_0001.JPG'):
            raise RuntimeError('boom')
        return matcher(q, d)
    bad = L.localize_inloc(flaky, root, tree['pairs'], str(tmp_path / 'r2.txt'), **kw)
    assert [q for q, _ in bad['failed']] == ['query/iphone7/IMG_0001.JPG']
    w = L.read_results(str(tmp_path / 'r2.txt'))
    assert len(w) == 4 and np.array_equal(w['IMG_0001.JPG'][0], np.eye(3)) and not w['IMG_0001.JPG'][1].any()
    for n in ('IMG_0000.JPG', 'IMG_0002.JPG', 'IMG_0003.JPG'):
        assert np.array_equal(bad['poses'][n][0], res['poses'][n][0])
