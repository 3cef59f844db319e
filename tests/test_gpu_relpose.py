"""p2p_relpose_errors_batch against the numpy oracle (oracle/relpose_oracle.py), the per-pair-threshold E RANSAC
(p2p_find_essential_batch_th) against the single-pair and uniform-threshold calls, and eval_relpose end to end: exact
synthetic_two_view matches through a callable, and Patch2Pix on a synthetic pair tree against a host recomputation
through estimate_matches_from_files, find_essential_matrices, recover_poses and the oracle."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import relpose_oracle as O
from patch2pix_b200 import _lib
from patch2pix_b200 import pose as P
from patch2pix_b200 import relpose as RP
from patch2pix_b200.synth import _rotation, synthetic_relpose_tree, synthetic_two_view

pytestmark = pytest.mark.gpu
THR1 = [5e-4]
THR16 = np.geomspace(1e-7, 1e-1, 16).tolist()


def _intr(K0, K1):
    return np.array([K0[0, 0], K0[1, 1], K0[0, 2], K0[1, 2], K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]])


def _scene(seed, n, stride=4):
    """A synthetic_two_view pair with noise and outliers as [n, stride] rows (columns past 4 unrelated), its intrinsics,
    ground truth [12], a perturbed estimate [12] and an inlier count (0 for every fifth seed: no model)."""
    s = synthetic_two_view(seed, n, 0.3, 0.5, focal2=400.0 + 10 * (seed % 7))
    rng = np.random.default_rng([seed, 77])
    rows = np.concatenate([s['pts1'], s['pts2'], rng.normal(0, 100, (n, stride - 4))], 1)
    gt = np.concatenate([s['R'].reshape(9), s['t']])
    R = _rotation(rng.normal(0, 0.02, 3)) @ s['R']
    t = s['t'] / np.linalg.norm(s['t']) + rng.normal(0, 0.05, 3)
    est = np.concatenate([R.reshape(9), t])
    return rows, _intr(s['K1'], s['K2']), gt, est, 0 if seed % 5 == 4 else int(rng.integers(5, 500))


def _batch(seeds, sizes, stride=4):
    sc = [_scene(s, n, stride) for s, n in zip(seeds, sizes)]
    return ([r for r, *_ in sc], np.stack([x[1] for x in sc]), np.stack([x[2] for x in sc]),
            np.stack([x[3] for x in sc]), np.array([x[4] for x in sc], dtype=np.int32))


def _oracle(rows_list, intr, gt, est, cnt, thr, n_eff=None):
    cos, counts = [], []
    for k, rows in enumerate(rows_list):
        m = len(rows) if n_eff is None else n_eff[k]
        cos.append(O.pose_cosines(gt[k], est[k], cnt[k]))
        counts.append(O.counts(O.epipolar_errors(rows[:m], intr[k], gt[k]), thr))
    return np.array(cos), np.stack(counts)


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize('thr', [THR1, THR16], ids=['thr1', 'thr16'])
@pytest.mark.parametrize('stride', [4, 9])
def test_kernel_against_oracle(thr, stride):
    seeds = list(range(12))
    sizes = [300, 0, 1, 5000, 70, 0, 2000, 257, 1024, 3, 900, 40000]
    rows, intr, gt, est, cnt = _batch(seeds, sizes, stride)
    rows[6][5, 2] = np.nan                                      # a non-finite row never counts
    rows_d = [torch.from_numpy(r.reshape(-1, stride)).cuda() for r in rows]
    cos, counts = RP.relpose_errors(rows_d, intr, gt, est, cnt, thr)
    exp_cos, exp_counts = _oracle(rows, intr, gt, est, cnt, thr)
    assert _same(cos.cpu().numpy(), exp_cos)                    # bit for bit, NaN where there is no model
    assert np.array_equal(counts.cpu().numpy(), exp_counts)
    assert np.isnan(exp_cos[4]).all() and np.isfinite(exp_cos[0]).all()
    assert exp_counts[3, 0] > 0 and exp_counts[3, -2] < exp_counts[3, -1]      # the thresholds split the rows
    # K single-pair calls give the batch's records
    for k in range(len(rows)):
        c1, n1 = RP.relpose_errors(rows_d[k:k + 1], intr[k:k + 1], gt[k:k + 1], est[k:k + 1], cnt[k:k + 1], thr)
        assert _same(c1.cpu().numpy()[0], exp_cos[k]) and np.array_equal(n1.cpu().numpy()[0], exp_counts[k])


def _launch(h, rows, stride, offsets, n_dev, intr, gt, est, cnt, thr, L, out_off=0):
    dev = torch.device('cuda')
    offs = torch.from_numpy(offsets).to(dev)
    ex = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev) for a in (intr, gt, est)]
    cnt_d = torch.from_numpy(cnt).to(dev)
    K = offsets.size - 1
    out = torch.full((K + out_off, L), -7.0, dtype=torch.float64, device=dev)
    RP.relpose_errors_batch_into(h, rows, stride, offs, offsets, n_dev, ex[0].data_ptr(), ex[1].data_ptr(),
                                 ex[2].data_ptr(), cnt_d.data_ptr(), np.asarray(thr), out.data_ptr() + 8 * out_off * L,
                                 L)
    return out.cpu().numpy()


def test_kernel_n_dev_offsets_and_grid_schedules():
    sizes = [500, 0, 1300, 64, 7]
    rows, intr, gt, est, cnt = _batch(range(20, 25), sizes, 9)
    pre = np.full((3, 9), 1e6)                                  # rows before offsets[0] belong to no pair
    allrows = np.concatenate([pre] + rows)
    offsets = (3 + np.concatenate([[0], np.cumsum(sizes)])).astype(np.int64)
    n_eff = [250, 0, 1300, 64, 0]
    n_dev = torch.tensor([250.0, 3.0, 1e9, -1.0, 0.0], dtype=torch.float64, device='cuda')
    rows_d = torch.from_numpy(allrows).cuda()
    h = _lib.default_handle('cuda')
    L = 2 + (16 + 2) // 2 + 1                                   # a record wider than the kernel's output
    outs = []
    for sms in (0, 1, 7, 132):
        h.set_option('num_sms', sms)
        try:
            outs.append(_launch(h, rows_d, 9, offsets, C.c_void_p(n_dev.data_ptr()), intr, gt, est, cnt, THR16, L,
                                out_off=1))
        finally:
            h.set_option('num_sms', 0)
    exp_cos, exp_counts = _oracle(rows, intr, gt, est, cnt, THR16, n_eff)
    for out in outs:
        assert np.array_equal(out, outs[0], equal_nan=True)
        assert np.all(out[0] == -7.0) and np.all(out[1:, -1] == -7.0)     # nothing outside the records is written
        assert _same(out[1:, :2], exp_cos)
        assert np.array_equal(out[1:, 2:2 + 9].copy().view(np.int32)[:, :17], exp_counts)


def test_bad_arguments_raise():
    h = _lib.default_handle('cuda')
    rows = torch.zeros(4, 4, dtype=torch.float64, device='cuda')
    offs_h = np.array([0, 4], dtype=np.int64)
    offs = torch.from_numpy(offs_h).cuda()
    buf = torch.zeros(64, dtype=torch.float64, device='cuda')
    cnt = torch.ones(1, dtype=torch.int32, device='cuda')
    out = torch.zeros(16, dtype=torch.float64, device='cuda')
    Pv = C.c_void_p
    t = (C.c_double * 17)(*np.geomspace(1e-6, 1e-2, 17))

    def call(**kw):
        a = dict(rows=Pv(rows.data_ptr()), stride=4, offsets=Pv(offs.data_ptr()),
                 offsets_host=offs_h.ctypes.data_as(C.POINTER(C.c_int64)), K=1, intr=Pv(buf.data_ptr()),
                 gt=Pv(buf.data_ptr()), est=Pv(buf.data_ptr()), cnt=Pv(cnt.data_ptr()), thr=t, n_thr=1,
                 out=Pv(out.data_ptr()), out_stride=3)
        a.update(kw)
        return h.lib.p2p_relpose_errors_batch(h.h, a['rows'], a['stride'], a['offsets'], a['offsets_host'], a['K'],
                                              None, a['intr'], a['gt'], a['est'], a['cnt'], a['thr'], a['n_thr'],
                                              a['out'], a['out_stride'], h.stream())
    assert call() == 0
    for kw in [dict(n_thr=0), dict(n_thr=17), dict(out_stride=2), dict(n_thr=16, out_stride=10), dict(intr=None),
               dict(gt=None), dict(est=None), dict(cnt=None), dict(out=None), dict(stride=3), dict(thr=None),
               dict(thr=(C.c_double * 2)(1e-3, 1e-3), n_thr=2), dict(thr=(C.c_double * 1)(-1.0))]:
        assert call(**kw) == -1, kw
    with pytest.raises(ValueError):
        RP.relpose_errors([rows], np.zeros((1, 8)), np.zeros((1, 12)), np.zeros((1, 12)), [1], [2e-3, 1e-3])
    torch.cuda.synchronize()


# ---- per-pair thresholds ----------------------------------------------------------------------------------------------
def _essential_scenes():
    sc = [synthetic_two_view(40 + k, n, 0.35, 0.8, focal2=380.0 + 25 * k)
          for k, n in enumerate([400, 4, 0, 1200, 90, 2500, 5, 700])]
    return ([s['pts1'] for s in sc], [s['pts2'] for s in sc], [s['K1'] for s in sc], [s['K2'] for s in sc])


def test_per_pair_thresholds_match_single_pair_calls():
    p1, p2, K1, K2 = _essential_scenes()
    px = [0.3, 0.5, 1.0, 0.45, 2.0, 0.7, 1.0, 0.25]
    got = P.find_essential_matrices(p1, p2, K1, K2, px, conf=0.99999, max_iters=1000)
    n_model = 0
    for k in range(len(p1)):
        E, m = P.find_essential_matrix(p1[k], p2[k], K1[k], K2[k], px[k], conf=0.99999, max_iters=1000)
        assert (E is None) == (got[k][0] is None), k
        if E is not None:
            n_model += 1
            assert np.array_equal(E, got[k][0]), k
        assert np.array_equal(m, got[k][1]), k
    assert n_model >= 5
    # all thresholds equal: p2p_find_essential_batch's results
    same = P.find_essential_matrices(p1, p2, K1, K2, [0.6] * len(p1), conf=0.99999)
    ref = P.find_essential_matrices(p1, p2, K1, K2, 0.6, conf=0.99999)
    for (Ea, ma), (Eb, mb) in zip(same, ref):
        assert (Ea is None and Eb is None) or np.array_equal(Ea, Eb)
        assert np.array_equal(ma, mb)
    with pytest.raises(ValueError):
        P.find_essential_matrices(p1, p2, K1, K2, px[:-1])
    with pytest.raises(ValueError):
        P.find_essential_matrices(p1, p2, K1, K2, [0.0] + px[1:])


def test_per_pair_thresholds_select_different_models():
    """One scene at two thresholds in one batch: each pair gets its own threshold's inliers."""
    s = synthetic_two_view(9, 1500, 0.2, 1.5)
    got = P.find_essential_matrices([s['pts1']] * 2, [s['pts2']] * 2, [s['K1']] * 2, [s['K2']] * 2, [0.2, 3.0])
    assert got[0][1].sum() < got[1][1].sum()


# ---- eval_relpose ----------------------------------------------------------------------------------------------------
def _two_view_pairs(root, n_pairs, noise):
    """SuperGlue-format pair list of synthetic_two_view scenes (no image files) and a callable matcher returning each
    scene's correspondences."""
    scenes, lines = {}, []
    for k in range(n_pairs):
        s = synthetic_two_view(100 + k, 400, 0.0, noise, focal2=420.0 + 20 * k)
        n0, n1 = f'v{k}_0.png', f'v{k}_1.png'
        scenes[os.path.join(root, n0)] = np.concatenate([s['pts1'], s['pts2']], 1)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = s['R'], s['t']
        vals = np.concatenate([s['K1'].reshape(-1), s['K2'].reshape(-1), T.reshape(-1)])
        lines.append(' '.join([n0, n1, '0', '0'] + ['%.17g' % v for v in vals]))
    path = os.path.join(root, 'pairs.txt')
    with open(path, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    return path, lambda a, b: scenes[a]


def test_noise_free_matches_recover_the_pose(tmp_path):
    path, matcher = _two_view_pairs(str(tmp_path), 6, 0.0)
    lines = []
    res = RP.eval_relpose(matcher, path, str(tmp_path), lprint_=lines.append)
    assert res['n_pairs'] == 6 and not res['failed'] and res['n_matches'] == 400
    for r in res['records']:
        assert r.R_err < 0.1 and r.t_err < 0.1 and r.n_inliers == 400 and r.N == 400
    assert res['auc'][5.0] > 0.9 and res['prec'][5e-4] == 1.0
    assert len(lines) == 2 and 'failed=0' in lines[1]


def test_failed_and_short_pairs(tmp_path):
    path, base = _two_view_pairs(str(tmp_path), 5, 0.3)

    def matcher(a, b):
        if 'v1_' in a:
            raise RuntimeError('no matches for you')
        if 'v2_' in a:
            return base(a, b)[:3]                               # fewer than 5 rows: no model
        if 'v3_' in a:
            return torch.from_numpy(base(a, b)).cuda(), 'extra'
        return base(a, b)

    res = RP.eval_relpose(matcher, path, str(tmp_path), epi_thresholds=[1e-6, 5e-4], chunk_pairs=2,
                          lprint_=lambda s: None)
    recs = res['records']
    assert [f[0] for f in res['failed']] == [1] and 'no matches for you' in res['failed'][0][3]
    assert recs[1].match_failed and recs[1].N == 0 and recs[1].err == np.inf
    assert recs[2].N == 3 and recs[2].n_inliers == 0 and recs[2].err == np.inf and not recs[2].match_failed
    assert all(np.isfinite(recs[k].err) for k in (0, 3, 4))
    errs = [r.err for r in recs]
    assert res['auc'] == O.pose_auc(errs, [5.0, 10.0, 20.0])
    assert res['prec'] == O.precision([r.counts for r in recs], [1e-6, 5e-4])
    one = RP.eval_relpose(matcher, path, str(tmp_path), epi_thresholds=[1e-6, 5e-4], chunk_pairs=512,
                          lprint_=lambda s: None)
    for a, b in zip(recs, one['records']):                      # the chunking changes no record
        assert _same([a.cos_R, a.cos_t, a.N, a.n_inliers, a.n_good], [b.cos_R, b.cos_t, b.N, b.n_inliers, b.n_good])
        assert np.array_equal(a.counts, b.counts) and np.array_equal(a.R, b.R) and np.array_equal(a.t, b.t)
    empty = tmp_path / 'empty.txt'
    empty.write_text('')
    e = RP.eval_relpose(matcher, str(empty), str(tmp_path), lprint_=lambda s: None)
    assert e['n_pairs'] == 0 and all(np.isnan(v) for v in e['auc'].values())


@pytest.fixture(scope='module')
def net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


@pytest.mark.parametrize('fmt,eval_type,chunk', [('txt', 'fine', 512), ('npz', 'fine', 2), ('txt', 'coarse', 3)])
def test_patch2pix_matches_host(net, tmp_path, fmt, eval_type, chunk):
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    root = str(tmp_path)
    path, _ = synthetic_relpose_tree(root, 2, 5, fmt=fmt, size=(256, 192))
    pairs = RP.read_pairs(path, root)
    kw = dict(ksize=2, io_thres=0.25, ncn_thres=0.0, imsize=1024)
    thr = [1e-5, 5e-4, 1e-2]
    res = RP.eval_relpose(net, path, root, eval_type=eval_type, epi_thresholds=thr, chunk_pairs=chunk,
                          lprint_=lambda s: None, **kw)
    assert not res['failed'] and len(res['records']) == 5
    ms = [estimate_matches_from_files(net, p.path0, p.path1, kw['ksize'], kw['ncn_thres'], True, kw['io_thres'],
                                      eval_type, kw['imsize'])[0] for p in pairs]
    intr, Rt_gt, px = RP.pair_arrays(pairs, 0.5)
    Es = P.find_essential_matrices([m[:, :2] for m in ms], [m[:, 2:4] for m in ms], [p.K0 for p in pairs],
                                   [p.K1 for p in pairs], px, conf=0.99999, max_iters=1000)
    poses = P.recover_poses([np.zeros((3, 3)) if E is None else E for E, _ in Es], [m[:, :2] for m in ms],
                            [m[:, 2:4] for m in ms], [p.K0 for p in pairs], [p.K1 for p in pairs],
                            [m for _, m in Es], dist_th=1e9)
    n_model = 0
    for k, r in enumerate(res['records']):
        E, emask = Es[k]
        n_good, R, t, _ = poses[k]
        n_in = int(emask.sum()) if E is not None else 0
        n_model += E is not None
        assert r.N == len(ms[k]) and r.n_inliers == n_in and r.n_good == n_good, k
        assert np.array_equal(r.R, R) and np.array_equal(r.t, t.reshape(3)), k
        est = np.concatenate([R.reshape(9), t.reshape(3)])
        assert _same([r.cos_R, r.cos_t], O.pose_cosines(Rt_gt[k], est, n_in)), k
        assert (r.R_err, r.t_err) == O.pose_errors(r.cos_R, r.cos_t), k
        assert np.array_equal(r.counts, O.counts(O.epipolar_errors(ms[k], intr[k], Rt_gt[k]), thr)), k
    assert n_model >= 1
    assert res['auc'] == O.pose_auc([r.err for r in res['records']], [5.0, 10.0, 20.0])
