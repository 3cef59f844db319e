"""Host side of the non-finite and tie contract of SuperGlue's optimal transport and NCNet's proposals
(tests/test_gpu_argmax_edges.py runs the kernels against it):
  - oracle/superglue_oracle.py's log_optimal_transport and extract equal a float64 torch restatement of SuperGlue's
    published form (torch.logsumexp iterations, max(2) / max(1) / gather) on masked and NaN scores, so np.argmax's
    order (first NaN, first maximum, an all -inf line at 0) is the one the kernel has to follow;
  - the reference's corr_to_matches outputs on non-finite volumes (tests/golden/nonfinite_golden.npz);
  - the tie-aware decision rule (oracle.decidable_ties) on a hand-made matrix."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import superglue_oracle as O

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NAN, INF = float('nan'), float('inf')


def _published_ot(scores, alpha, iters):
    """SuperGlue's log_optimal_transport, [n, m] float64 -> log_assign [n+1, m+1]."""
    s = torch.as_tensor(scores, dtype=torch.float64)[None]
    a = torch.tensor(float(alpha), dtype=torch.float64)
    b, n, m = s.shape
    ms, ns = s.new_tensor(n), s.new_tensor(m)
    couplings = torch.cat([torch.cat([s, a.expand(b, n, 1)], -1),
                           torch.cat([a.expand(b, 1, m), a.expand(b, 1, 1)], -1)], 1)
    norm = -(ms + ns).log()
    log_mu = torch.cat([norm.expand(n), ns.log()[None] + norm])
    log_nu = torch.cat([norm.expand(m), ms.log()[None] + norm])
    u, v = torch.zeros_like(log_mu)[None], torch.zeros_like(log_nu)[None]
    for _ in range(iters):
        u = log_mu[None] - torch.logsumexp(couplings + v.unsqueeze(1), dim=2)
        v = log_nu[None] - torch.logsumexp(couplings + u.unsqueeze(2), dim=1)
    return (couplings + u.unsqueeze(2) + v.unsqueeze(1) - norm)[0].numpy()


def _published_extract(la, threshold):
    z = torch.as_tensor(la, dtype=torch.float64)[None, :-1, :-1]
    max0, max1 = z.max(2), z.max(1)
    i0, i1 = max0.indices, max1.indices
    mutual0 = torch.arange(z.shape[1])[None] == i1.gather(1, i0)
    mutual1 = torch.arange(z.shape[2])[None] == i0.gather(1, i1)
    zero = z.new_tensor(0)
    ms0 = torch.where(mutual0, max0.values.exp(), zero)
    ms1 = torch.where(mutual1, ms0.gather(1, i1), zero)
    valid0 = mutual0 & (ms0 > threshold)
    valid1 = mutual1 & valid0.gather(1, i1)
    return {'matches0': torch.where(valid0, i0, i0.new_tensor(-1))[0].numpy(),
            'matches1': torch.where(valid1, i1, i1.new_tensor(-1))[0].numpy(),
            'mscores0': ms0[0].numpy(), 'mscores1': ms1[0].numpy()}


def _scores(seed, n, m):
    return np.random.default_rng(seed).normal(0.0, 3.0, (n, m))


def _case(name):
    """(scores [n, m] float64, alpha, iters, threshold)"""
    s = _scores(len(name), 37, 45)
    alpha, iters, thr = 1.0, 20, 0.2
    if name == 'scattered_masks':
        s[[3, 17, 30]] = -INF
        s[:, [0, 8, 44]] = -INF
    elif name == 'padded':
        s[29:] = -INF
        s[:, 40:] = -INF
    elif name == 'one_row_left':
        s[:] = -INF
        s[5] = _scores(1, 1, 45)
    elif name == 'row0_col0_negative_threshold':
        s[0] = -INF
        s[:, 0] = -INF
        thr = -0.5
    elif name == 'finite_padding':
        s[29:] = -1e9
        s[:, 40:] = -1e9
    elif name == 'nan_cell':
        s[11, 13] = NAN
    elif name == 'nan_cell_no_iterations':
        s[11, 13] = NAN
        s[4, 7] = NAN
        iters = 0
    elif name == 'nan_row':
        s[9] = NAN
    elif name == 'nan_alpha':
        alpha = NAN
    else:
        raise ValueError(name)
    return s, alpha, iters, thr


CASES = ['scattered_masks', 'padded', 'one_row_left', 'row0_col0_negative_threshold', 'finite_padding', 'nan_cell',
         'nan_cell_no_iterations', 'nan_row', 'nan_alpha']


@pytest.mark.parametrize('name', CASES)
def test_oracle_equals_the_published_form_on_masked_and_nan_scores(name):
    s, alpha, iters, thr = _case(name)
    la, _ = O.log_optimal_transport(s, alpha, iters)
    ref = _published_ot(s, alpha, iters)
    np.testing.assert_array_equal(np.isnan(la), np.isnan(ref))
    np.testing.assert_array_equal(np.isneginf(la), np.isneginf(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(la[fin], ref[fin], rtol=1e-12, atol=1e-9)
    e, p = O.extract(la, thr), _published_extract(la, thr)
    for k in ('matches0', 'matches1', 'mscores0', 'mscores1'):
        np.testing.assert_array_equal(e[k], p[k], err_msg=k)       # NaN compares equal to NaN here
    if name == 'row0_col0_negative_threshold':
        assert e['matches0'][0] == 0 and e['matches1'][0] == 0 and e['mscores0'][0] == 0.0
    if name.startswith('nan') and iters > 0:
        assert np.isnan(la).all() and (e['matches0'] == -1).all() and e['i0'].max() == 0


def test_extraction_order_is_first_nan_then_first_maximum():
    la = np.full((5, 6), -1.0)
    la[0, :5] = [1.0, NAN, 3.0, NAN, 3.0]
    la[1, :5] = -INF
    la[2, :5] = [2.0, 5.0, 5.0, INF, INF]
    e = O.extract(la, 0.1)
    assert list(e['i0']) == [1, 0, 3, 0]
    t = torch.as_tensor(la[:-1, :-1]).max(1).indices.numpy()
    assert list(t) == list(e['i0'])


def _gold():
    spec = importlib.util.spec_from_file_location('make_nonfinite_golden',
                                                  os.path.join(GOLD_DIR, 'make_nonfinite_golden.py'))
    K = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(K)
    return K, dict(np.load(os.path.join(GOLD_DIR, 'nonfinite_golden.npz')))


def test_nonfinite_golden_holds_every_case():
    K, gold = _gold()
    b, _, hA, wA, hB, wB = K.SHAPE
    for ci, case in enumerate(K.CASES):
        v = gold[f'vol_{case}']
        assert v.dtype == np.float32 and v.shape == K.SHAPE
        assert np.array_equal(v, K.volume(case, 900 + ci).numpy(), equal_nan=True)
        for n, d in zip('ijkl', K.deltas(950 + ci, 2)):
            assert np.array_equal(gold[f'delta_{case}_{n}'], d.numpy())
        for inv, sm, ks, ri in K.ARGS:
            key = K.nonfinite_key(case, inv, sm, ks, ri)
            rows = hA * wA if inv else hB * wB
            for n in ('a0', 'a1', 'a2', 'a3', 'score'):
                assert gold[f'{key}_{n}'].shape == (b, rows), (key, n)
            assert gold[f'{key}_score'].dtype == np.float32
            assert gold[f'{key}_a0'].dtype == (np.int64 if ri else np.float32)
    # the reference's rules on these volumes: a NaN-softmax slice gives index 0 / NaN, an all -inf raw slice 0 / -inf
    key = K.nonfinite_key('nan_slice', False, True, 1, True)
    s = 1 * wB + 4
    assert np.isnan(gold[f'{key}_score'][0, s]) and gold[f'{key}_a0'][0, s] == 0 and gold[f'{key}_a1'][0, s] == 0
    key = K.nonfinite_key('ninf_slice', True, False, 1, True)
    s = 3 * wA
    assert (gold[f'{key}_score'][0, s:s + wA] == -np.inf).all() and (gold[f'{key}_a2'][0, s:s + wA] == 0).all()
    key = K.nonfinite_key('nan_cell', True, False, 1, True)
    assert np.isnan(gold[f'{key}_score'][0, 1 * wA + 2]) and gold[f'{key}_a2'][0, 1 * wA + 2] == 3


def test_tie_aware_decision_rule():
    # columns 1 and 3 are duplicates; row 2 is masked; row 3 duplicates row 0
    z = np.array([[0.0, 5.0, 1.0, 5.0],
                  [4.0, 0.5, 0.0, 0.5],
                  [-INF, -INF, -INF, -INF],
                  [0.0, 5.0, 1.0, 5.0]])
    la = np.full((5, 5), -3.0)
    la[:4, :4] = z
    rows, cols = O.decidable(la, 0.0, 0.1)
    assert not rows[0] and not rows[3]                # plain decidable(): a duplicate's gap is 0
    rows, cols = O.decidable_ties(la, 0.0, 0.1)
    e = O.extract(la, 0.0)
    assert list(e['i0']) == [1, 0, 0, 1] and list(e['i1']) == [1, 0, 0, 0]
    # row 0 -> column 1 (lowest of the tie 1 / 3), column 1 -> row 0 (lowest of the tie 0 / 3): decided, mutual
    assert rows[0] and cols[1] and e['matches0'][0] == 1 and e['matches1'][1] == 0
    assert rows[1] and cols[0] and e['matches0'][1] == 0
    # the masked row ties everywhere: decided, points at column 0 whose argmax is row 1: not mutual
    assert rows[2] and e['matches0'][2] == -1
    assert rows[3] and e['matches0'][3] == -1 and cols[3] and e['matches1'][3] == -1
    # a gap inside the tolerance is still undecided, ties or not
    rows, cols = O.decidable_ties(la, 0.0, 3.8)
    assert not rows[1] and not cols[2] and rows[0]
    la2 = la.copy()
    la2[1, 1] = NAN
    rows, cols = O.decidable_ties(la2, 0.0, 0.1)
    assert not rows[1] and not cols[1] and not rows[0]
