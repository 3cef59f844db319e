"""Many pairs per call: find_fundamental_matrices / find_homographies / find_essential_matrices / recover_poses and the
matches2relapose batches against the single-pair calls, pair by pair and bit for bit (include/p2p_b200.h,
p2p_*_batch)."""
import ctypes as C

import numpy as np
import pytest
import torch

from patch2pix_b200 import _lib
from patch2pix_b200 import pose as P
from patch2pix_b200 import verify as V
from patch2pix_b200.synth import synthetic_dominant_plane, synthetic_two_view

pytestmark = pytest.mark.gpu

SIZES = [0, 4, 6, 7, 5, 8, 100, 3200, 20000]       # empty, below the samples (4, 5, 6), the samples, large


def _scene(k, n):
    """Pair k of the mixed list: general, planar and dominant-plane scenes in turn, seeded by k."""
    kind = k % 3
    if kind == 2:
        sc = synthetic_dominant_plane(k, max(n, 1), 0.3, 0.1, 0.5)
    else:
        sc = synthetic_two_view(k, max(n, 1), 0.4, 0.5, planar=kind == 1, focal2=None if k % 4 else 560.0)
    return sc['pts1'][:n].copy(), sc['pts2'][:n].copy(), sc['K1'], sc['K2']


@pytest.fixture(scope='module')
def pairs():
    rng = np.random.default_rng(11)
    sizes = SIZES + [int(v) for v in rng.integers(9, 2500, 31)]
    return [_scene(k, n) for k, n in enumerate(sizes)]


def _same(a, b):
    """Bit equality of two results (None, arrays, ints, tuples)."""
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_same(got, want):
    assert len(got) == len(want)
    bad = [k for k, (g, w) in enumerate(zip(got, want)) if not _same(g, w)]
    assert not bad, f'pairs differing from the single-pair call: {bad}'


@pytest.mark.parametrize('which', ['F', 'H', 'DEGENSAC'])
def test_find_model_batch_matches_single(pairs, which):
    p1, p2 = [p[0] for p in pairs], [p[1] for p in pairs]
    if which == 'H':
        got = V.find_homographies(p1, p2, 2.0, seed=3)
        want = [V.find_homography(a, b, 2.0, seed=3) for a, b in zip(p1, p2)]
    else:
        dg = which == 'DEGENSAC'
        got = V.find_fundamental_matrices(p1, p2, 1.0, seed=3, degeneracy_check=dg)
        want = [V.find_fundamental_matrix(a, b, 1.0, seed=3, degeneracy_check=dg) for a, b in zip(p1, p2)]
    _assert_same(got, want)
    assert sum(F is not None for F, _ in got) >= len(pairs) - 5


def test_essential_and_pose_batch_match_single(pairs):
    p1, p2, K1, K2 = ([p[i] for p in pairs] for i in range(4))
    got = P.find_essential_matrices(p1, p2, K1, K2, 1.0, seed=5)
    want = [P.find_essential_matrix(*args, 1.0, seed=5) for args in zip(p1, p2, K1, K2)]
    _assert_same(got, want)
    E = [np.zeros((3, 3)) if e is None else e for e, _ in got]
    masks = [m for _, m in got]
    masks[3] = None                                      # all rows of that pair
    pg = P.recover_poses(E, p1, p2, K1, K2, masks)
    pw = [P.recover_pose(e, a, b, k1, k2, m) for e, a, b, k1, k2, m in zip(E, p1, p2, K1, K2, masks)]
    _assert_same(pg, pw)
    _assert_same(P.recover_poses(E, p1, p2, K1, K2), [P.recover_pose(*a) for a in zip(E, p1, p2, K1, K2)])


def test_matches2relapose_batches_match_single(pairs):
    ms = [np.concatenate((p[0], p[1]), 1) for p in pairs]
    K1, K2 = [p[2] for p in pairs], [p[3] for p in pairs]
    _assert_same(P.matches2relapose_batch(ms, K1, K2, rthres=1),
                 [P.matches2relapose(m[:, :2], m[:, 2:4], a, b, rthres=1) for m, a, b in zip(ms, K1, K2)])
    _assert_same(P.matches2relapose_degensac_batch(ms, K1, K2, rthres=1),
                 [P.matches2relapose_degensac(m[:, :2], m[:, 2:4], a, b, rthres=1) for m, a, b in zip(ms, K1, K2)])


def test_non_finite_pair_is_reported_and_isolated(pairs):
    sub = pairs[6:12]
    p1 = [p[0].copy() for p in sub]
    p2 = [p[1].copy() for p in sub]
    p1[2][17, 1] = np.nan
    with pytest.raises(ValueError, match='not finite'):
        V.find_fundamental_matrix(p1[2], p2[2], 1.0)
    with pytest.raises(ValueError, match='not finite'):
        V.find_fundamental_matrices(p1, p2, 1.0)
    with pytest.raises(ValueError, match='not finite'):
        P.find_essential_matrices(p1, p2, [p[2] for p in sub], [p[3] for p in sub], 1.0)
    dev = torch.device('cuda', torch.cuda.current_device())
    t1 = [torch.from_numpy(a).to(dev) for a in p1]
    t2 = [torch.from_numpy(b).to(dev) for b in p2]
    got = [(F.cpu().numpy(), m.cpu().numpy()) for F, m in V.find_fundamental_matrices(t1, t2, 1.0, degeneracy_check=True)]
    want = [tuple(x.cpu().numpy() for x in V.find_fundamental_matrix(a, b, 1.0, degeneracy_check=True))
            for a, b in zip(t1, t2)]
    _assert_same(got, want)
    assert np.isnan(got[2][0]).all() and not got[2][1].any()
    Kl1, Kl2 = [p[2] for p in sub], [p[3] for p in sub]
    got = [(E.cpu().numpy(), m.cpu().numpy()) for E, m in P.find_essential_matrices(t1, t2, Kl1, Kl2, 1.0)]
    want = [tuple(x.cpu().numpy() for x in P.find_essential_matrix(*a, 1.0)) for a in zip(t1, t2, Kl1, Kl2)]
    _assert_same(got, want)
    assert np.isnan(got[2][0]).all()


def test_n_dev_and_packed_rows(pairs):
    """row_stride 9 (p2p_finalize_matches' packed rows) and device row counts below the pairs' sizes."""
    sub = [p for p in pairs[4:20]]
    rng = np.random.default_rng(2)
    rows = [np.concatenate((a, b, rng.normal(size=(a.shape[0], 5))), 1) for a, b, _, _ in sub]
    n = np.array([r.shape[0] for r in rows])
    caps = np.where(np.arange(len(rows)) % 3 == 0, n, np.maximum(n - rng.integers(0, 50, len(rows)), 0)).astype(float)
    caps[1] = -1.0                                       # negative: all rows, as for a single pair
    offsets = np.concatenate(([0], np.cumsum(n))).astype(np.int64)
    dev = torch.device('cuda', torch.cuda.current_device())
    R = torch.from_numpy(np.concatenate(rows)).to(dev)
    offs = torch.from_numpy(offsets).to(dev)
    nd = torch.from_numpy(caps).to(dev)
    h = _lib.default_handle(dev)
    K, N = len(rows), int(offsets[-1])
    for model in (V.MODEL_F, V.MODEL_H, V.MODEL_F_DEGENSAC):
        out = torch.zeros(V.batch_out_size(K, N), dtype=torch.float64, device=dev)
        b = out.data_ptr()
        V.find_model_batch_into(h, model, R, 9, offs, offsets, C.c_void_p(nd.data_ptr()), 1.0, 0.999, 3000, 9, b,
                                b + 8 * (9 * K + (K + 1) // 2), b + 72 * K)
        got = V.parse_batch_host(out.cpu().numpy(), offsets)
        want = []
        for k in range(K):
            rk = R[offsets[k]:offsets[k + 1]].contiguous()
            o = torch.zeros(V.out_size(int(n[k])), dtype=torch.float64, device=dev)
            V.find_model_into(h, model, rk, 9, int(n[k]), C.c_void_p(nd.data_ptr() + 8 * k), 1.0, 0.999, 3000, 9, o)
            want.append(V.parse_host(o.cpu().numpy(), int(n[k])))
        _assert_same(got, want)
        for k in range(K):
            if 0 <= caps[k] < n[k]:
                assert not got[k][1][int(caps[k]):].any()
    # E and pose on the same packed rows
    intr = np.stack([np.asarray(P.intrinsics(a, b)) for _, _, a, b in sub])
    intr_d = torch.from_numpy(intr).to(dev)
    out = torch.zeros(P.batch_out_size(K, N), dtype=torch.float64, device=dev)
    pp = P._batch_ptrs(out, K, N)
    P.find_essential_batch_into(h, R, 9, offs, offsets, C.c_void_p(nd.data_ptr()), intr_d.data_ptr(), 1.0, 0.999, 1000, 4,
                                pp['E'], pp['emask'], pp['cnt'])
    P.recover_pose_batch_into(h, R, 9, offs, offsets, C.c_void_p(nd.data_ptr()), intr_d.data_ptr(), pp['E'], pp['emask'],
                              pp['Rt'], pp['pmask'], pp['good'])
    got = P._parse_batch(out.cpu().numpy(), offsets, K, N)
    want = []
    for k in range(K):
        rk = R[offsets[k]:offsets[k + 1]].contiguous()
        o = torch.zeros(P.out_size(int(n[k])), dtype=torch.float64, device=dev)
        ik = P.intrinsics(sub[k][2], sub[k][3])
        ndk = C.c_void_p(nd.data_ptr() + 8 * k)
        P.find_essential_into(h, rk, 9, int(n[k]), ndk, ik, 1.0, 0.999, 1000, 4, o)
        P.recover_pose_into(h, rk, 9, int(n[k]), ndk, ik, o.data_ptr(), o.data_ptr() + 184, o)
        want.append(P.parse_host(o.cpu().numpy(), int(n[k])))
    _assert_same(got, want)


def test_empty_batches():
    assert V.find_fundamental_matrices([], [], 1.0) == []
    assert V.find_homographies([], [], 2.0) == []
    assert P.find_essential_matrices([], [], [], [], 1.0) == []
    assert P.recover_poses([], [], [], [], []) == []
    assert P.matches2relapose_batch([], [], []) == []
    assert P.matches2relapose_degensac_batch([], [], []) == []


def _small_pairs(count, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        sc = synthetic_two_view(seed * 100000 + k, int(rng.integers(5, 40)), 0.3, 0.5, planar=k % 5 == 1)
        out.append((sc['pts1'], sc['pts2'], sc['K1'], sc['K2']))
    return out


def test_chunk_boundaries_change_nothing():
    """More pairs than one launch takes (the scratch budget's pair count), against the single-pair calls."""
    cf = V.batch_chunk_pairs(0)
    ce = V.batch_chunk_pairs(1)
    assert 1 < ce < cf <= 65535 and V.batch_chunk_pairs(2) <= 65535
    sub = _small_pairs(cf + 3, 1)
    p1, p2 = [p[0] for p in sub], [p[1] for p in sub]
    got = V.find_fundamental_matrices(p1, p2, 1.0, max_iters=1024, seed=2)
    want = [V.find_fundamental_matrix(a, b, 1.0, max_iters=1024, seed=2) for a, b in zip(p1, p2)]
    _assert_same(got, want)
    sub = sub[:ce + 3]
    p1, p2, K1, K2 = ([p[i] for p in sub] for i in range(4))
    got = P.find_essential_matrices(p1, p2, K1, K2, 1.0, max_iters=512, seed=2)
    want = [P.find_essential_matrix(*a, 1.0, max_iters=512, seed=2) for a in zip(p1, p2, K1, K2)]
    _assert_same(got, want)


def test_batches_are_deterministic_and_order_free(pairs):
    p1, p2 = [p[0] for p in pairs], [p[1] for p in pairs]
    K1, K2 = [p[2] for p in pairs], [p[3] for p in pairs]
    a = V.find_fundamental_matrices(p1, p2, 1.0, seed=8, degeneracy_check=True)
    _assert_same(V.find_fundamental_matrices(p1, p2, 1.0, seed=8, degeneracy_check=True), a)
    perm = np.random.default_rng(4).permutation(len(pairs))
    b = V.find_fundamental_matrices([p1[i] for i in perm], [p2[i] for i in perm], 1.0, seed=8, degeneracy_check=True)
    _assert_same(b, [a[i] for i in perm])
    e = P.matches2relapose_batch([np.concatenate(x, 1) for x in zip(p1, p2)], K1, K2)
    f = P.matches2relapose_batch([np.concatenate((p1[i], p2[i]), 1) for i in perm], [K1[i] for i in perm],
                                 [K2[i] for i in perm])
    _assert_same(f, [e[i] for i in perm])
