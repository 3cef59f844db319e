"""Edges of the two argmax kernels that take a user's score tensor, against float64 and the live reference:
  - SuperGlue's optimal transport and extraction (csrc/superglue.cu, p2p_sg_sinkhorn) against
    oracle/superglue_oracle.py at the kernel's tile and chunk boundaries (32-wide transpose tiles, 256-column row-pass
    chunks), with exact ties from duplicated keypoints, masked (-inf) keypoints and padded batches, NaN and +inf
    values, and large magnitudes.  Decisions follow np.argmax: NaN above +inf above every number, ties to the lowest
    index, so an all -inf line points at 0;
  - NCNet's proposals (csrc/coarse.cu, p2p_proposals) against the reference's corr_to_matches on volumes with NaN,
    +inf and -inf cells and slices (tests/golden/nonfinite_golden.npz, make_nonfinite_golden.py).
Every index a kernel returns must lie in range whatever the values: an index past the buffer is a device fault."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import superglue_oracle as O
from patch2pix_b200 import superglue as SG

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN, INF = float('nan'), float('inf')
GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _planted(seed, B, n, m, scale=20.0, d=64):
    """[B, n, m] fp32: scale x cosine similarities of seeded unit descriptors, 70% of the smaller side planted."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(B):
        def unit(k):
            x = torch.randn(k, d, generator=g, dtype=torch.float64)
            return x / x.norm(dim=1, keepdim=True)
        a, b = unit(n), unit(m)
        k = int(0.7 * min(n, m))
        pi, pj = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        b[pj] = a[pi] + 0.3 * unit(k)
        b = b / b.norm(dim=1, keepdim=True)
        out.append(a @ b.T * scale)
    return torch.stack(out).float()


def _run(scores, alpha, iters, thr):
    out = SG._sinkhorn(scores.to(DEV), torch.tensor(float(alpha), device=DEV), iters, thr, log_assign=True)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check(scores, alpha, iters, thr, valid=None):
    """Runs the kernel on scores [B, n, m] and checks every pair against the oracle: non-finite log_assign entries
    where the oracle's are, finite ones within sinkhorn_bound, and the decisions of every line that decidable_ties
    decides or that holds a NaN (those follow the first NaN exactly).  valid: per pair, (rows, cols) bool masks of the
    lines that are not finite padding; padded lines must come out unmatched with score 0 and are compared loosely
    (-1e9 + u + v rounds to multiples of 64 in fp32).  -> (outputs, per-pair decided (rows, cols), excluded fraction)"""
    B, n, m = scores.shape
    got = _run(scores, alpha, iters, thr)
    decided, excluded, total = [], 0, 0
    for b in range(B):
        s = scores[b].double().numpy()
        ref, vmax = O.log_optimal_transport(s, alpha, iters)
        la = got['log_assign'][b].astype(np.float64)
        for f in (np.isnan, np.isneginf, np.isposinf):
            assert np.array_equal(f(la), f(ref)), (b, f.__name__)
        vr, vc = valid[b] if valid is not None else (np.ones(n, bool), np.ones(m, bool))
        sv = s[np.ix_(vr, vc)]
        fin_s = sv[np.isfinite(sv)]
        amax = max(abs(alpha) if np.isfinite(alpha) else 0.0, float(np.abs(fin_s).max()) if fin_s.size else 0.0)
        bound = O.sinkhorn_bound(n, m, amax, vmax, iters)
        fin = np.isfinite(ref)
        inner = np.zeros_like(fin)
        inner[np.ix_(np.append(vr, True), np.append(vc, True))] = True
        if fin[inner].any():
            err = float(np.abs(la[fin & inner] - ref[fin & inner]).max())
            assert err <= bound, (b, err, bound)
        if (fin & ~inner).any():
            assert float(np.abs(la[fin & ~inner] - ref[fin & ~inner]).max()) <= 128 + bound, b
        e = O.extract(ref, thr)
        z = ref[:-1, :-1]
        rows, cols = O.decidable_ties(ref, thr, 2 * bound)
        rows = (rows & vr) | np.isnan(z).any(1)
        cols = (cols & vc) | np.isnan(z).any(0)
        ms_tol = np.expm1(bound) + 2.0 ** -21
        for k, sel in (('matches0', rows), ('matches1', cols)):
            assert np.array_equal(got[k][b][sel], e[k][sel]), (b, k, np.flatnonzero(got[k][b][sel] != e[k][sel]))
        for k, sel in (('mscores0', rows), ('mscores1', cols)):
            np.testing.assert_allclose(got[k][b][sel], e[k][sel], rtol=ms_tol, atol=1e-30, equal_nan=True,
                                       err_msg=f'{b} {k}')
        for k, sel in (('matches0', ~vr), ('matches1', ~vc)):
            assert (got[k][b][sel] == -1).all() and (e[k][sel] == -1).all(), (b, k)
        for k, sel in (('mscores0', ~vr), ('mscores1', ~vc)):
            assert (got[k][b][sel] == 0).all() and (e[k][sel] == 0).all(), (b, k)
        decided.append((rows, cols))
        excluded += int((~rows).sum() + (~cols).sum())
        total += n + m
    return got, decided, excluded / total


# ---- SuperGlue: sizes at the tile and chunk boundaries -----------------------------------------------------------------
@pytest.mark.parametrize('n, m, B', [(31, 256, 1), (32, 255, 3), (33, 257, 1), (255, 33, 1), (256, 31, 3),
                                     (257, 513, 1), (511, 32, 1), (513, 256, 1)])
def test_sinkhorn_boundary_sizes(n, m, B):
    _, _, frac = _check(_planted(n * 11 + m + B, B, n, m), 1.0, 100, 0.2)
    print(f'{n}x{m} B={B}: excluded {frac:.3f}')
    if min(n, m) >= 90:
        assert frac < 0.1, frac


# ---- exact ties from duplicated keypoints -------------------------------------------------------------------------------
TIE_PLACEMENTS = {     # (column pairs (src, dup), row pairs (src, dup)) on 300 x 600 scores
    'same_lane': ([(5, 37), (40, 136)], [(5, 37), (40, 104)]),
    'neighbour_lanes': ([(70, 71), (100, 99)], [(70, 71), (100, 99)]),
    'same_lane_next_chunk': ([(12, 268), (300, 556)], [(12, 268)]),
    'rows_in_other_warps': ([], [(3, 150), (200, 9), (60, 61)]),
}


@pytest.mark.parametrize('placement', sorted(TIE_PLACEMENTS))
def test_sinkhorn_exact_ties_go_to_the_lowest_index(placement):
    cpairs, rpairs = TIE_PLACEMENTS[placement]
    n, m = 300, 600
    g = torch.Generator().manual_seed(7)
    s = (3.0 * torch.randn(n, m, generator=g)).float()
    used_r = {i for p in rpairs for i in p}
    used_c = {j for p in cpairs for j in p}
    free_r = [i for i in range(n) if i not in used_r]
    free_c = [j for j in range(m) if j not in used_c]
    hot_r = []                       # the row that holds each duplicated column's maximum
    for k, (j, _) in enumerate(cpairs):
        s[free_r[k], j] = 15.0 + k
        hot_r.append(free_r[k])
    hot_c = []                       # the column that holds each duplicated row's maximum
    for k, (i, _) in enumerate(rpairs):
        s[i, free_c[k]] = 15.0 + k
        hot_c.append(free_c[k])
    for j, d in cpairs:
        s[:, d] = s[:, j]
    for i, d in rpairs:
        s[d, :] = s[i, :]
    got, decided, _ = _check(s[None], 1.0, 100, 0.2)
    la = got['log_assign'][0]
    rows, cols = decided[0]
    for j, d in cpairs:
        assert np.array_equal(la[:, j].view(np.int32), la[:, d].view(np.int32)), (j, d)
    for i, d in rpairs:
        assert np.array_equal(la[i].view(np.int32), la[d].view(np.int32)), (i, d)
    # the tied lines are decided, so _check compared them: each resolves to its lowest index
    for (j, d), r in zip(cpairs, hot_r):
        assert rows[r] and got['matches0'][0][r] == min(j, d), (j, d, got['matches0'][0][r])
        assert got['matches1'][0][max(j, d)] == -1
    for (i, d), c in zip(rpairs, hot_c):
        assert cols[c] and got['matches1'][0][c] == min(i, d), (i, d, got['matches1'][0][c])
        assert got['matches0'][0][max(i, d)] == -1


# ---- masked keypoints ----------------------------------------------------------------------------------------------------
def _masked_case(name):
    """-> (scores [B, n, m], threshold, valid per pair or None)"""
    if name == 'scattered':
        s = _planted(21, 1, 300, 280)
        s[0, [0, 31, 32, 100, 299]] = -INF
        s[0, :, [0, 5, 255, 256, 279]] = -INF
        return s, 0.2, None
    if name == 'padded_batch':
        sizes = [(300, 280), (150, 280), (233, 97)]
        s = torch.full((3, 300, 280), -INF)
        for b, (nb, mb) in enumerate(sizes):
            s[b, :nb, :mb] = _planted(30 + b, 1, nb, mb)[0]
        return s, 0.2, None
    if name == 'one_row_left':
        s = torch.full((1, 64, 300), -INF)
        s[0, 7] = _planted(40, 1, 1, 300)[0, 0]
        return s, 0.2, None
    if name == 'row0_col0_negative_threshold':
        s = _planted(50, 1, 120, 90)
        s[0, 0] = -INF
        s[0, :, 0] = -INF
        return s, -0.5, None
    if name == 'finite_padding':
        s = torch.full((2, 260, 200), -1e9)
        s[0, :260, :140] = _planted(60, 1, 260, 140)[0]
        s[1, :90, :200] = _planted(61, 1, 90, 200)[0]
        valid = [(np.arange(260) < 260, np.arange(200) < 140), (np.arange(260) < 90, np.arange(200) < 200)]
        return s, 0.2, valid
    raise ValueError(name)


MASKED = ['scattered', 'padded_batch', 'one_row_left', 'row0_col0_negative_threshold', 'finite_padding']


@pytest.mark.parametrize('name', MASKED)
def test_sinkhorn_masked_keypoints(name):
    s, thr, valid = _masked_case(name)
    got, decided, frac = _check(s, 1.0, 100, thr, valid)
    print(f'{name}: excluded {frac:.3f}')
    for b in range(s.shape[0]):
        z = s[b].numpy()
        rows, cols = decided[b]
        masked_r, masked_c = np.isneginf(z).all(1), np.isneginf(z).all(0)
        assert rows[masked_r].all() and cols[masked_c].all()      # a masked line is always compared
        assert (got['mscores0'][b][masked_r] == 0).all()
    if name == 'row0_col0_negative_threshold':
        # numpy's rule: row 0 and column 0 both point at index 0, a "mutual" pair of score exp(-inf) = 0 > -0.5
        assert got['matches0'][0][0] == 0 and got['matches1'][0][0] == 0 and got['mscores0'][0][0] == 0
    if name == 'one_row_left':
        assert (got['matches0'][0][np.arange(64) != 7] == -1).all()


# ---- NaN and +inf ---------------------------------------------------------------------------------------------------------
NONFINITE = {     # name: (n, m, iters, alpha, cells {(i, j): value} or a row index for a whole NaN row)
    'nan_first_chunk': (200, 600, 100, 1.0, {(17, 3): NAN}),
    'nan_middle_chunk': (200, 600, 100, 1.0, {(17, 300): NAN}),
    'nan_last_chunk': (200, 600, 100, 1.0, {(199, 590): NAN}),
    'nan_row_m255': (150, 255, 100, 1.0, 40),
    'nan_row_m256': (150, 256, 100, 1.0, 40),
    'nan_row_m256_one_iteration': (150, 256, 1, 1.0, 40),
    'nan_row_m257': (150, 257, 100, 1.0, 40),
    'nan_alpha': (120, 130, 100, NAN, {}),
    'pinf_cell': (120, 130, 100, 1.0, {(5, 6): INF}),
    'nan_and_inf_no_iterations': (100, 300, 0, 1.0, {(3, 4): NAN, (3, 290): NAN, (8, 290): INF, (9, 10): INF,
                                                      (9, 40): INF, (12, 7): -INF}),
}


def _nonfinite_scores(name):
    n, m, iters, alpha, cells = NONFINITE[name]
    s = _planted(len(name), 1, n, m)
    if isinstance(cells, int):
        s[0, cells] = NAN
    else:
        for (i, j), v in cells.items():
            s[0, i, j] = v
    return s, iters, alpha


@pytest.mark.parametrize('name', sorted(NONFINITE))
def test_sinkhorn_nan_and_inf(name):
    s, iters, alpha = _nonfinite_scores(name)
    got, _, _ = _check(s, alpha, iters, 0.2)
    if iters > 0:
        assert np.isnan(got['log_assign']).all()                   # NaN reaches every u and v, as in float64
        assert (got['matches0'] == -1).all() and (got['matches1'] == -1).all()
    for k, hi in (('matches0', s.shape[2]), ('matches1', s.shape[1])):
        assert (got[k] < hi).all()


# ---- large magnitudes -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('scale, alpha, iters', [(1e3, 1.0, 100), (1e4, 1.0, 100), (20.0, 1e4, 100),
                                                 (20.0, -1e4, 100), (20.0, 1.0, 1000)])
def test_sinkhorn_magnitudes(scale, alpha, iters):
    _, _, frac = _check(_planted(int(scale) % 97 + iters, 1, 220, 170, scale=scale), alpha, iters, 0.2)
    print(f'|C| <= {scale:g}, alpha {alpha:g}, iters {iters}: excluded {frac:.3f}')


# ---- determinism ----------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def test_masked_and_nan_results_are_grid_and_batch_invariant():
    s = torch.full((3, 300, 280), -INF)
    s[0, :300, :200] = _planted(70, 1, 300, 200)[0]
    s[1, :120, :280] = _planted(71, 1, 120, 280)[0]
    s[1, 50] = NAN
    s[2, :256, :256] = _planted(72, 1, 256, 256)[0]
    s[2, 3, 260] = NAN
    scores, alpha = s.to(DEV), torch.tensor(0.5, device=DEV)
    h = SG._lib.default_handle(DEV)
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    runs = []
    try:
        for v in (0, 1, 7, 131):
            h.set_option('num_sms', min(v, n_sm))
            runs.append(SG._sinkhorn(scores, alpha, 100, 0.2, log_assign=True))
    finally:
        h.set_option('num_sms', 0)
    for r in runs[1:]:
        for k in r:
            assert torch.equal(_bits(r[k]), _bits(runs[0][k])), k
    for b in range(3):
        single = SG._sinkhorn(scores[b:b + 1].contiguous(), alpha, 100, 0.2, log_assign=True)
        for k in single:
            assert torch.equal(_bits(single[k][0]), _bits(runs[0][k][b])), (b, k)
    assert torch.isnan(runs[0]['log_assign'][1]).all() and not torch.isnan(runs[0]['log_assign'][0]).any()


# ---- the whole module on a batch of two pairs of different sizes ----------------------------------------------------------
def test_superglue_forward_batch_of_two_against_float64():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = O.seeded_state_dict(3, proj_gain=16.0, bin_score=1.0)
    sg = SG.SuperGlue()
    sg.load_state_dict(sd)
    sg = sg.to(DEV)
    n, m, k = 110, 140, 80
    g = torch.Generator().manual_seed(8)

    def desc(c):
        d = torch.randn(2, 256, c, generator=g)
        return d / d.norm(dim=1, keepdim=True)
    d0, d1 = desc(n), desc(m)
    for b in range(2):
        pi, pj = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        d1[b][:, pj] = d0[b][:, pi]
    data = {'image0': torch.zeros(2, 1, 120, 160), 'image1': torch.zeros(2, 1, 96, 128),
            'keypoints0': torch.stack([torch.rand(2, n, generator=g) * 159, torch.rand(2, n, generator=g) * 119], 2),
            'keypoints1': torch.stack([torch.rand(2, m, generator=g) * 127, torch.rand(2, m, generator=g) * 95], 2),
            'scores0': torch.rand(2, n, generator=g), 'scores1': torch.rand(2, m, generator=g),
            'descriptors0': d0, 'descriptors1': d1}
    gdata = {kk: v.to(DEV) for kk, v in data.items()}
    out = sg(gdata)
    with torch.no_grad():
        s32 = sg.score_matrix(gdata).double().cpu().numpy()
    npd = O.to_numpy(sd)
    for b in range(2):
        ref_s = O.scores(npd, *[data[kk][b].double().numpy() for kk in ('keypoints0', 'keypoints1', 'scores0',
                                                                         'scores1', 'descriptors0', 'descriptors1')],
                         (120, 160), (96, 128), sg.config['GNN_layers'], 5)
        gnn_dev = float(np.abs(s32[b] - ref_s).max())
        assert gnn_dev < 1e-3, gnn_dev
        ref_la, vmax = O.log_optimal_transport(ref_s, float(sd['bin_score']), 100)
        tol = O.sinkhorn_bound(n, m, float(np.abs(ref_s).max()) + 1, vmax, 100) + 401 * gnn_dev
        e = O.extract(ref_la, 0.2)
        rows, cols = O.decidable(ref_la, 0.2, 2 * tol)
        assert (~rows).sum() + (~cols).sum() < 0.35 * (n + m)
        assert np.array_equal(out['matches0'][b].cpu().numpy()[rows], e['matches0'][rows])
        assert np.array_equal(out['matches1'][b].cpu().numpy()[cols], e['matches1'][cols])
        ms = out['matching_scores0'][b].cpu().numpy()[rows]
        assert (np.abs(ms - e['mscores0'][rows]) <= e['mscores0'][rows] * (np.expm1(tol) + 2.0 ** -21) + 1e-30).all()


# ---- NCNet proposals on non-finite volumes, against the reference ---------------------------------------------------------
@pytest.fixture(scope='module')
def nonfinite_gold():
    spec = importlib.util.spec_from_file_location('make_nonfinite_golden',
                                                  os.path.join(GOLD_DIR, 'make_nonfinite_golden.py'))
    K = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(K)
    return K, dict(np.load(os.path.join(GOLD_DIR, 'nonfinite_golden.npz')))


def _volume(gold, case, ks):
    v = torch.from_numpy(gold[f'vol_{case}']).to(DEV)
    d = tuple(torch.from_numpy(gold[f'delta_{case}_{n}']).to(DEV) for n in 'ijkl') if ks > 1 else None
    return v, d


def test_corr_to_matches_on_nonfinite_volumes_vs_reference(nonfinite_gold):
    from patch2pix_b200.ncnet import corr_to_matches
    K, gold = nonfinite_gold
    for case in K.CASES:
        for inv, sm, ks, ri in K.ARGS:
            key = K.nonfinite_key(case, inv, sm, ks, ri)
            v, d = _volume(gold, case, ks)
            got = corr_to_matches(v, d, ksize=ks, do_softmax=sm, scale='positive', invert_matching_direction=inv,
                                  return_indices=ri)
            for n, t in zip(('a0', 'a1', 'a2', 'a3'), got[:4]):
                t, e = t.cpu().numpy(), gold[f'{key}_{n}']
                if ri:
                    assert np.array_equal(t, e), (key, n, np.argwhere(t != e)[:4])
                else:
                    np.testing.assert_allclose(t, e, rtol=0, atol=1e-7, err_msg=f'{key} {n}')
            sc, e = got[4].cpu().numpy(), gold[f'{key}_score']
            if sm:
                np.testing.assert_allclose(sc, e, rtol=1e-5, atol=1e-7, equal_nan=True, err_msg=key)
            else:
                np.testing.assert_array_equal(sc, e, err_msg=key)       # the raw maximum, NaN as NaN


def test_cal_coarse_matches_on_nonfinite_volumes(nonfinite_gold):
    from patch2pix_b200.model import cal_coarse_matches
    from patch2pix_b200.ncnet import corr_to_matches
    K, gold = nonfinite_gold
    b, _, hA, wA, hB, wB = K.SHAPE
    for case in K.CASES:
        for ks in (1, 2):
            for sm in (True, False):
                v, d = _volume(gold, case, ks)
                m, sc = cal_coarse_matches(v, d, ks, sm, upsample=16, center=True)
                m = m.cpu()
                for c, hi in enumerate((wA, hA, wB, hB)):
                    assert (m[..., c] >= 8).all() and (m[..., c] < hi * ks * 16).all(), (case, ks, sm, c)
                fwd = torch.stack(corr_to_matches(v, d, ksize=ks, do_softmax=sm)[:4], -1).cpu()
                inv = torch.stack(corr_to_matches(v, d, ksize=ks, do_softmax=sm,
                                                  invert_matching_direction=True)[:4], -1).cpu()
                assert torch.equal(m, torch.cat([fwd, inv], 1) * 16 + 8), (case, ks, sm)


def test_corr_to_matches_topk_indices_stay_in_range(nonfinite_gold):
    from patch2pix_b200.ncnet import corr_to_matches_topk
    K, gold = nonfinite_gold
    _, _, hA, wA, hB, wB = K.SHAPE
    for case in K.CASES:
        for ks in (1, 2):
            for sm in (True, False):
                for inv in (False, True):
                    v, d = _volume(gold, case, ks)
                    got = corr_to_matches_topk(v, d, topk=2, ksize=ks, do_softmax=sm, invert_matching_direction=inv)
                    for t, hi in zip(got[:4], (wA, hA, wB, hB)):
                        t = t.cpu()
                        assert (t >= 0).all() and (t < hi * ks).all(), (case, ks, sm, inv)
