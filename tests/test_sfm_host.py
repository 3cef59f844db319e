"""CPU checks of the Aachen triangulation protocol: the numpy oracle (oracle/sfm_oracle.py) on hand-built cases, the
file readers, the model write/read round trip, the CLI's argument errors, and the whole protocol rehearsed with the
oracle and cv2.solvePnPRansac on a synthetic tree with exact matches."""
import math
import os

import numpy as np
import pytest

from oracle import sfm_oracle as O
from patch2pix_b200 import sfm as S
from patch2pix_b200.evaluation import read_cameras_binary, read_images_binary


def test_merge_means_and_id_order():
    # image 1's endpoints come first in input order but its keys sort after image 0's
    m = [np.array([[9.0, 1.0, 1.0, 1.0], [10.0, 2.0, 2.5, 3.0], [1.0, 9.0, 1.0, 1.0]])]
    img, x, y = O.endpoints(m, [(1, 0)])
    kp_xy, kp_key, kp_of, dropped = O.keypoints(img, x, y, 4.0)
    # image 0: cell (0, 0) holds (1, 1), (2.5, 3), (1, 1); image 1: cells (2, 0) and (0, 2)
    assert dropped == 0 and len(kp_xy) == 3
    np.testing.assert_array_equal(kp_xy[0], [(1.0 + 2.5 + 1.0) / 3, (1.0 + 3.0 + 1.0) / 3])
    assert list(kp_key >> np.uint64(44)) == [0, 1, 1]
    assert kp_xy[1].tolist() == [9.5, 1.5] and kp_xy[2].tolist() == [1.0, 9.0]
    assert kp_of.tolist() == [1, 0, 1, 0, 2, 0]


def test_merge_drops_bad_endpoints():
    m = [np.array([[np.nan, 1.0, 1.0, 1.0], [-0.5, 2.0, 4.0 * (1 << 22), 3.0]])]
    img, x, y = O.endpoints(m, [(0, 1)])
    kp_xy, _, kp_of, dropped = O.keypoints(img, x, y, 4.0)
    assert dropped == 3 and kp_of.tolist() == [-1, 0, -1, -1] and len(kp_xy) == 1


def test_one_to_one_rule_and_chain():
    # pair (A, B): A1 -> B1 first, A1 -> B2 is not first for A1, A2 -> B1 is not first for B1
    kp_n = np.ones((4, 2))
    kp_of = np.array([0, 2, 0, 3, 1, 2])
    E, thr = np.zeros((1, 9)), np.ones(1)
    E[0, 0] = 1e-9
    edges, n_first = O.edges(kp_of, [3], E, thr, kp_n)
    assert edges == [(0, 2)] and n_first == 1
    # a chain A1 - B1 - A2 across two pairs is one component labelled by its smallest id
    lab = O.components(5, [(0, 2), (1, 2)])
    assert lab.tolist() == [0, 0, 0, 3, 4]
    obs, tr, rej = O.tracks(lab)
    assert tr == [(0, 3)] and rej == 0 and obs[:3].tolist() == [0, 1, 2]


def _cam(f=500.0, k=0.0):
    return np.array([2, f, f, 320.0, 240.0, k, 0.0, 0.0])


def _rec(R, C):
    t = -R @ C
    return np.concatenate([R.reshape(-1), t, C])


def _view(rec, cam, X):
    p = rec[:9].reshape(3, 3) @ X + rec[9:12]
    return O.distort_px(cam, np.array([p[0] / p[2]]), np.array([p[1] / p[2]]))


def test_chain_of_two_surfaces_gives_two_points():
    # image 0 sees X1 and X2 at one keypoint (a wrong match chains them); images 1, 2 see X1, images 3, 4 see X2
    cam = _cam()
    recs = np.stack([_rec(np.eye(3), np.array([dx, 0.0, 0.0])) for dx in (0.0, 0.5, 1.0, -0.5, -1.0)])
    X1, X2 = np.array([0.2, 0.1, 8.0]), np.array([-0.3, 0.2, 9.0])
    xy = [_view(recs[0], cam, X1), _view(recs[1], cam, X1), _view(recs[2], cam, X1), _view(recs[3], cam, X2),
          _view(recs[4], cam, X2)]
    kp_xy = np.array([[a[0], b[0]] for a, b in xy])
    kp_key = np.arange(5, dtype=np.uint64) << np.uint64(44)
    kp_n = O.undistort_keypoints(kp_xy, kp_key, np.zeros(5, int), cam[None])
    pts, plen, perr, kp_point = O.triangulate(np.arange(5), [(0, 5)], kp_xy, kp_n, kp_key, recs, np.zeros(5, int),
                                              cam[None])
    assert len(pts) == 2
    np.testing.assert_allclose(pts[0], X1, rtol=1e-9)
    np.testing.assert_allclose(pts[1], X2, rtol=1e-9)
    assert kp_point.tolist() == [0, 0, 0, 1, 1]


def test_angle_rejection():
    cam = _cam()
    X = np.array([0.0, 0.0, 10.0])
    for base, n_pts in ((0.1, 0), (1.0, 1)):               # 0.57 degrees is rejected, 5.7 degrees accepted
        recs = np.stack([_rec(np.eye(3), np.array([dx, 0.0, 0.0])) for dx in (0.0, base)])
        kp_xy = np.array([[v[0] for v in _view(r, cam, X)] for r in recs])
        kp_key = np.arange(2, dtype=np.uint64) << np.uint64(44)
        kp_n = O.undistort_keypoints(kp_xy, kp_key, np.zeros(2, int), cam[None])
        pts, *_ = O.triangulate(np.arange(2), [(0, 2)], kp_xy, kp_n, kp_key, recs, np.zeros(2, int), cam[None])
        assert len(pts) == n_pts


@pytest.mark.parametrize('k', [(-0.08, 0.0), (0.05, 0.0), (-0.05, 0.01)])
def test_distortion_round_trip(k):
    c = np.array([3, 600.0, 600.0, 512.0, 384.0, k[0], k[1], 0.0])
    v, u = np.mgrid[0:768:16, 0:1024:16].astype(np.float64)
    xn, yn = O.undistort(c, u.reshape(-1), v.reshape(-1))
    px, py = O.distort_px(c, xn, yn)
    assert np.abs(px - u.reshape(-1)).max() < 1e-9 and np.abs(py - v.reshape(-1)).max() < 1e-9


def test_readers(tmp_path):
    p = tmp_path / 'pairs.txt'
    p.write_text('a b\n\nc d\n')
    assert S.read_pairs(str(p)) == [('a', 'b'), ('c', 'd')]
    p.write_text('a b\nc\n')
    with pytest.raises(ValueError, match='pairs.txt:2'):
        S.read_pairs(str(p))
    q = tmp_path / 'q.txt'
    q.write_text('q0.jpg SIMPLE_RADIAL 640 480 500 320 240 -0.01\nq1.jpg PINHOLE 640 480 500 510 320 240\n')
    qs = S.read_queries_with_intrinsics(str(q))
    assert list(qs) == ['q0.jpg', 'q1.jpg'] and qs['q1.jpg'].params.tolist() == [500, 510, 320, 240]
    q.write_text('q0.jpg OPENCV 640 480 1 2 3 4 5 6 7 8\n')
    with pytest.raises(ValueError, match='q.txt:1.*OPENCV'):
        S.read_queries_with_intrinsics(str(q))
    q.write_text('q0.jpg SIMPLE_RADIAL 640 480 500 320\n')
    with pytest.raises(ValueError, match='q.txt:1'):
        S.read_queries_with_intrinsics(str(q))
    with pytest.raises(ValueError, match='camera 7.*FOV'):
        S.camera_record('FOV', [1, 2, 3, 4, 5], 'camera 7')


def test_model_round_trip(tmp_path):
    from argparse import Namespace
    cams = {3: Namespace(id=3, model='SIMPLE_RADIAL', width=320, height=240, params=np.array([300, 160, 120, -0.05]))}
    ims = [Namespace(id=5, qvec=np.array([1.0, 0, 0, 0]), tvec=np.array([0.0, 0, 1]), camera_id=3, name='a.png'),
           Namespace(id=9, qvec=np.array([0.0, 1, 0, 0]), tvec=np.array([1.0, 0, 0]), camera_id=3, name='b.png')]
    kp_xy = np.array([[1.5, 2.5], [10.25, 3.0], [4.0, 4.5]])
    kp_key = np.array([0, 2, (1 << 44) | (1 << 22) | 1], dtype=np.uint64)     # the cells of kp_xy
    kp_point = np.array([0, -1, 0])
    m = S.SfmModel(cams, ims, 4.0, kp_xy, kp_key, kp_point, np.array([[1.0, 2, 3]]), np.array([2]),
                   np.array([0.25]), {})
    m.write(str(tmp_path))
    c = read_cameras_binary(str(tmp_path / 'cameras.bin'))
    assert c[3].model == 'SIMPLE_RADIAL' and c[3].params.tolist() == [300, 160, 120, -0.05]
    im = read_images_binary(str(tmp_path / 'images.bin'), points2D=True)
    assert [i.name for i in im.values()] == ['a.png', 'b.png']
    assert im[5].xys.tolist() == kp_xy[:2].tolist() and im[5].point3D_ids.tolist() == [0, -1]
    assert im[9].point3D_ids.tolist() == [0]
    pts = S.read_points3D_binary(str(tmp_path / 'points3D.bin'))
    assert pts[0].track == [(5, 0), (9, 0)] and pts[0].xyz.tolist() == [1, 2, 3] and pts[0].error == 0.25
    back = S.load_sfm_model(str(tmp_path))
    np.testing.assert_array_equal(back.kp_xy, kp_xy)
    np.testing.assert_array_equal(back.kp_key, kp_key)
    np.testing.assert_array_equal(back.kp_point, kp_point)
    assert back.points.tolist() == [[1, 2, 3]] and back.point_len.tolist() == [2]


def test_cli_argument_errors(tmp_path, capsys):
    f = tmp_path / 'f.txt'
    f.write_text('')
    base = ['--ckpt', str(f), '--images', str(tmp_path), '--model', str(tmp_path), '--db_pairs', str(f),
            '--query_pairs', str(f), '--queries', str(f), '--results', str(tmp_path / 'r.txt')]
    for bad, msg in ((['--images', str(f)], 'not a directory'), (['--db_pairs', str(tmp_path / 'x')], 'not a file'),
                     (['--queries', str(f), str(tmp_path / 'y')], 'not a file'),
                     (['--ransac_thres', '0'], 'must be positive'), (['--chunk_pairs', '0'], 'at least 1')):
        args = list(base)
        i = args.index(bad[0]) if bad[0] in args else len(args)
        args = args[:i] + bad + args[i + 2:] if bad[0] in base else args + bad
        with pytest.raises(SystemExit):
            S.main(args)
        assert msg in capsys.readouterr().err


def host_localize(tree, rows_fn, ransac_thres=12.0):
    """The oracle's query rows and cv2.solvePnPRansac per query -> {name: (R, t)}."""
    import cv2
    out = {}
    for q, R_t in rows_fn():
        rows, cam = R_t
        if len(rows) < 4:
            continue
        K = np.array([[cam[1], 0, cam[3]], [0, cam[2], cam[4]], [0, 0, 1]])
        ok, rv, tv, _ = cv2.solvePnPRansac(rows[:, 2:], rows[:, :2], K, None, reprojectionError=ransac_thres,
                                           iterationsCount=10000, confidence=0.99999, flags=cv2.SOLVEPNP_P3P)
        if ok:
            out[os.path.basename(q)] = (cv2.Rodrigues(rv)[0], tv.reshape(3))
    return out


def test_oracle_protocol_end_to_end(tmp_path):
    from patch2pix_b200 import localize as L
    from patch2pix_b200.synth import aachen_gt_matcher, synthetic_aachen_tree
    tree = synthetic_aachen_tree(str(tmp_path), 4, 6, 4)
    match = aachen_gt_matcher(tree, step=6)
    pairs = S.read_pairs(tree['db_pairs'])
    cameras, images, cams, img_cam, recs = S._model_tables(tree['model'])
    pt = S._pair_tables(images, cams, img_cam, recs, pairs, 4.0)
    mt = [match(os.path.join(tree['images'], a), os.path.join(tree['images'], b)) for a, b in pairs]
    r = O.triangulate_host((cams, img_cam, recs), pt, mt)
    assert len(r['points']) > 100 and r['point_err'].mean() < 2.0
    qs = S.read_queries_with_intrinsics(tree['queries'])
    index = {im.name: i for i, im in enumerate(images)}

    def rows_fn():
        for q, dbs in L.read_retrieval(tree['query_pairs']):
            qm = [match(os.path.join(tree['images'], q), os.path.join(tree['images'], d)) for d in dbs]
            cam = S.camera_record(qs[q].model, qs[q].params)
            rows, _ = O.query_rows(qm, [(0, index[d]) for d in dbs], [cam], r['kp_xy'], r['kp_key'],
                                   r['kp_point'], r['points'], 4.0)
            yield q, (rows, cam)
    est = host_localize(tree, rows_fn)
    ev = L.eval_localization(est, tree['gt'], thresholds=S.AACHEN_THRESHOLDS)
    assert ev['recall'][(0.25, 2.0)] == 1.0, ev['errors']
