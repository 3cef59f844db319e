"""p2p_homography_errors against the numpy oracle (oracle/hpatches_oracle.py), and eval_hpatches end to end on
synthetic HPatches trees: ground-truth and displaced-rows matchers, and Patch2Pix against a host recomputation through
estimate_matches_from_files."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import hpatches_oracle as O
from patch2pix_b200 import _lib
from patch2pix_b200 import hpatches as HP
from patch2pix_b200.synth import synthetic_hpatches_tree

pytestmark = pytest.mark.gpu
EDGE_BAND = 1e-12
THR10 = list(range(1, 11))
THR16 = np.geomspace(0.05, 40.0, 16).tolist()
H_GT = np.array([[0.95, 0.08, 12.0], [-0.05, 1.03, -7.5], [1.2e-4, -0.8e-4, 1.0]])


def _rows(seed, n, stride):
    """[n, stride] float64: H_GT correspondences with sigma = 3 px noise, 30 % uniform outliers, ~1 % rows with a NaN;
    columns past 4 hold unrelated values."""
    rng = np.random.default_rng([seed, n, stride])
    x = rng.uniform([0, 0], [640, 480], (n, 2))
    px, py, _ = O.project(H_GT, x[:, 0], x[:, 1])
    y = np.stack([px, py], 1) + rng.normal(0, 3.0, (n, 2))
    out = rng.uniform(0, 1, n) < 0.3
    y[out] = rng.uniform([0, 0], [640, 480], (int(out.sum()), 2))
    rows = np.concatenate([x, y, rng.normal(0, 100, (n, stride - 4))], 1)
    nan = rng.uniform(0, 1, n) < 0.01
    rows[nan, rng.integers(0, 4, int(nan.sum()))] = np.nan
    return rows


def _pred_buf(H, count):
    buf = np.zeros(10, dtype=np.float64)
    buf[:9] = np.asarray(H, dtype=np.float64).reshape(9)
    buf[9:10].view(np.int32)[0] = count
    return torch.from_numpy(buf).cuda()


def _check_counts(got, d, thresholds):
    """Bit-exact counts, except rows within EDGE_BAND relative of a threshold, which may fall either way."""
    d = np.asarray(d)
    assert int(got[-1]) == len(d)
    for j, t in enumerate(thresholds):
        near = np.abs(d - t) <= EDGE_BAND * t
        with np.errstate(invalid='ignore'):
            lo = int(np.count_nonzero((d <= t) & ~near))
        assert lo <= int(got[j]) <= lo + int(near.sum()), (j, t, int(got[j]), lo, int(near.sum()))


def _check_corner(got, exp):
    if np.isinf(exp):
        assert got == np.inf
    else:
        assert np.isfinite(got) and abs(got - exp) <= 1e-12 * max(abs(exp), 1e-300), (got, exp)


H_PERT = H_GT + np.array([[1e-3, -2e-3, 0.7], [5e-4, 1e-3, -0.4], [1e-6, 2e-6, 0.0]])
PRED_CASES = {'exact': (H_GT, 57), 'perturbed': (H_PERT, 57), 'count0': (H_GT, 0),
              'nan': (np.full((3, 3), np.nan), -1)}


@pytest.mark.parametrize('thresholds', [THR10, THR16], ids=['thr10', 'thr16'])
@pytest.mark.parametrize('n_dev', ['none', 'n', 'half', 'zero'])
@pytest.mark.parametrize('stride', [4, 9])
@pytest.mark.parametrize('n', [0, 1, 1000, 70000])
def test_kernel_against_oracle(n, stride, n_dev, thresholds):
    rows = _rows(1, n, stride)
    m = {'none': n, 'n': n, 'half': n // 2, 'zero': 0}[n_dev]
    nd = None if n_dev == 'none' else torch.tensor([float(m)], dtype=torch.float64, device='cuda')
    d = O.reprojection_errors(rows[:m], H_GT)
    rows_d = torch.from_numpy(rows).cuda() if n else torch.zeros(0, stride, dtype=torch.float64, device='cuda')
    for name, (H, count) in PRED_CASES.items():
        counts, corner = HP.homography_errors(rows_d, H_GT, _pred_buf(H, count), 640, 480, thresholds, n_dev=nd)
        counts, corner = counts.cpu().numpy(), float(corner.cpu()[0])
        assert counts.shape == (len(thresholds) + 1,)
        _check_counts(counts, d, thresholds)
        _check_corner(corner, O.corner_error(H_GT, H, count, 640, 480))
        if name == 'exact':
            assert corner == 0.0


def test_kernel_bit_exact_and_deterministic():
    rows = torch.from_numpy(_rows(2, 50000, 9)).cuda()
    buf = _pred_buf(H_PERT, 10)
    outs = [HP.homography_errors(rows, H_GT, buf, 321, 207, THR16) for _ in range(3)]
    d = O.reprojection_errors(rows.cpu().numpy(), H_GT)
    exp = O.counts(d, THR16)
    for c, e in outs:
        assert np.array_equal(c.cpu().numpy(), exp)           # the kernel's arithmetic is the oracle's, bit for bit
        assert float(e.cpu()[0]) == O.corner_error(H_GT, H_PERT, 10, 321, 207)


def test_kernel_corner_at_w_zero():
    Hw = np.eye(3)
    Hw[2, 0] = -1.0 / 99.0                                    # corner (99, 0) of a 100 x 50 image has w = 0
    rows = torch.zeros(4, 4, dtype=torch.float64, device='cuda')
    _, e = HP.homography_errors(rows, np.eye(3), _pred_buf(Hw, 8), 100, 50, THR10)
    assert float(e.cpu()[0]) == np.inf
    _, e = HP.homography_errors(rows, Hw, _pred_buf(np.eye(3), 8), 100, 50, THR10)
    assert float(e.cpu()[0]) == np.inf


@pytest.mark.parametrize('bad', [[], [1, 1], [2, 1], [0, 1], [-1], [1, float('nan')], [1, float('inf')],
                                 list(range(1, 18))])
def test_bad_thresholds_raise(bad):
    rows = torch.zeros(4, 4, dtype=torch.float64, device='cuda')
    with pytest.raises(ValueError):
        HP.homography_errors(rows, H_GT, _pred_buf(H_GT, 4), 64, 48, bad)
    if 1 <= len(bad) <= 16:             # the C entry point checks them too
        h = _lib.default_handle('cuda')
        counts = torch.empty(len(bad) + 1, dtype=torch.int32, device='cuda')
        corner = torch.empty(1, dtype=torch.float64, device='cuda')
        with pytest.raises(RuntimeError, match='thresholds'):
            HP.homography_errors_into(h, rows, 4, 4, None, H_GT, C.c_void_p(_pred_buf(H_GT, 4).data_ptr()), 64, 48,
                                      np.array(bad, dtype=np.float64), C.c_void_p(counts.data_ptr()),
                                      C.c_void_p(corner.data_ptr()))


def test_null_pointers_and_bad_sizes_raise():
    h = _lib.default_handle('cuda')
    rows = torch.zeros(4, 4, dtype=torch.float64, device='cuda')
    buf = _pred_buf(H_GT, 4)
    counts = torch.empty(11, dtype=torch.int32, device='cuda')
    corner = torch.empty(1, dtype=torch.float64, device='cuda')
    t = (C.c_double * 10)(*THR10)
    H = (C.c_double * 9)(*H_GT.reshape(9))
    P = C.c_void_p
    good = [h.h, P(rows.data_ptr()), 4, 4, None, H, P(buf.data_ptr()), 64, 48, t, 10, P(counts.data_ptr()),
            P(corner.data_ptr()), h.stream()]
    assert h.lib.p2p_homography_errors(*good) == 0
    for i, v in [(1, None), (5, None), (6, None), (9, None), (11, None), (12, None), (2, 3), (7, 0), (8, 0), (10, 0),
                 (10, 17)]:
        args = list(good)
        args[i] = v
        assert h.lib.p2p_homography_errors(*args) == -1, i
    torch.cuda.synchronize()


# ---- eval_hpatches ------------------------------------------------------------------------------------------------
SEQS = [('i_a', (200, 150)), ('i_b', (257, 181)), ('v_c', (240, 176)), ('v_d', (224, 200)), ('v_e', (176, 144)),
        ('i_dc', (160, 128))]                        # i_dc: one of D2-Net's excluded sequences


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('hpatches'))
    return root, synthetic_hpatches_tree(root, 7, SEQS)


def _seq_k(p1, p2):
    seq = os.path.basename(os.path.dirname(p1))
    assert os.path.basename(p1) == '1.ppm' and os.path.dirname(p2) == os.path.dirname(p1)
    return seq, int(os.path.basename(p2).split('.')[0])


def _grid(w, h, step=9):
    ys, xs = np.mgrid[1:h - 1:step, 2:w - 1:step].astype(np.float64)
    return xs.reshape(-1) + 0.25, ys.reshape(-1) + 0.5


def _displaced(Hs, sizes, offsets):
    """Rows whose image-2 point is pi(H_gt x1) moved by offsets[r % len(offsets)] px along x."""
    def rows(p1, p2):
        seq, k = _seq_k(p1, p2)
        x, y = _grid(*sizes[seq])
        px, py, _ = O.project(Hs[seq][k - 2], x, y)
        off = np.asarray(offsets, dtype=np.float64)[np.arange(len(x)) % len(offsets)]
        return np.stack([x, y, px + off, py], 1)
    return rows


def test_ground_truth_matcher(tree):
    root, Hs = tree
    sizes = dict(SEQS)
    lines = []
    res = HP.eval_hpatches(_displaced(Hs, sizes, [0.0]), root, lprint_=lines.append)
    assert res['n_pairs'] == 25 and res['h_failed'] == 0
    assert [(r.seq, r.k) for r in res['records']] == [(s, k) for s in ('i_a', 'i_b', 'v_c', 'v_d', 'v_e')
                                                      for k in range(2, 7)]
    assert sum(r.seq.startswith('i_') for r in res['records']) == 10
    for split in ('all', 'i', 'v'):
        assert np.all(res['mma'][split] == 1.0) and res['mma'][split].shape == (10,)
        assert np.all(res['h_acc'][split] == 1.0) and res['h_acc'][split].shape == (4,)
    for r in res['records']:
        assert r.N == len(_grid(*sizes[r.seq])[0]) and r.n_inliers == r.N and r.corner_err < 1e-6
    assert len(lines) == 4 and 'failed=0' in lines[2]


def test_displaced_rows_and_short_matchers(tree):
    root, Hs = tree
    sizes = dict(SEQS)
    offsets = [0.5 + j for j in range(12)]           # clear of every threshold
    base = _displaced(Hs, sizes, offsets)

    def matcher(p1, p2, as_tensor=False):
        seq, k = _seq_k(p1, p2)
        if (seq, k) == ('v_d', 4):
            raise RuntimeError('no matches for you')
        rows = base(p1, p2)
        if (seq, k) == ('i_b', 3):
            rows = np.zeros((0, 4))
        elif (seq, k) == ('v_c', 5):
            rows = rows[:3] + [0, 0, 50.0, 0]
        rows = torch.from_numpy(rows).cuda() if as_tensor else rows
        return (rows, 'extra', 'outputs') if k == 6 else rows

    res = HP.eval_hpatches(matcher, root, lprint_=lambda s: None)
    res_t = HP.eval_hpatches(lambda a, b: matcher(a, b, True), root, lprint_=lambda s: None)
    short = {('v_d', 4), ('i_b', 3), ('v_c', 5)}
    for r in res['records']:
        mma = O.pair_mma(r.counts)
        if (r.seq, r.k) in short:
            assert np.all(mma == 0) and r.corner_err == np.inf
            assert r.match_failed == ((r.seq, r.k) == ('v_d', 4))
        else:
            n = len(_grid(*sizes[r.seq])[0])
            exp = np.array([sum(1 for i in range(n) if offsets[i % 12] <= t) / n for t in THR10])
            assert np.array_equal(mma, exp), (r.seq, r.k)
    assert res['h_failed'] >= 3
    for a, b in zip(res['records'], res_t['records']):
        assert (a.seq, a.k, a.N, a.n_inliers, a.match_failed) == (b.seq, b.k, b.N, b.n_inliers, b.match_failed)
        assert np.array_equal(a.counts, b.counts)
        assert a.corner_err == b.corner_err or (np.isnan(a.corner_err) and np.isnan(b.corner_err))
    for split in ('all', 'i', 'v'):
        assert np.array_equal(res['mma'][split], res_t['mma'][split])
        assert np.array_equal(res['h_acc'][split], res_t['h_acc'][split])


@pytest.fixture(scope='module')
def net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


@pytest.mark.parametrize('eval_type', ['fine', 'coarse'])
def test_patch2pix_matches_host(net, tree, eval_type):
    from patch2pix_b200.eval_helper import estimate_matches_from_files
    root, Hs = tree
    kw = dict(ksize=2, io_thres=0.25, ncn_thres=0.0, imsize=1024)
    res = HP.eval_hpatches(net, root, eval_type=eval_type, ransac_thres=2.0, lprint_=lambda s: None, **kw)
    seqs = {s.name: s for s in HP.read_hpatches(root)}
    n_model = 0
    for r in res['records']:
        s = seqs[r.seq]
        assert not r.match_failed
        m, _, _, inl, model = estimate_matches_from_files(net, s.paths[0], s.paths[r.k - 1], kw['ksize'],
                                                          kw['ncn_thres'], True, kw['io_thres'], eval_type,
                                                          kw['imsize'], verify=('H', 2.0))
        assert r.N == len(m)
        if model is None:
            assert r.n_inliers <= 0 and r.corner_err == np.inf
        else:
            n_model += 1
            assert r.n_inliers == int(inl.sum())
        _check_counts(r.counts, O.reprojection_errors(m, s.H_gt[r.k - 2]), THR10)
        _check_corner(r.corner_err, O.corner_error(s.H_gt[r.k - 2], model if model is not None else np.eye(3),
                                                   r.n_inliers, *s.size))
    assert n_model >= 1
