"""corr_to_matches_topk on the GPU (topk.cu): bit-exact indices against the float64 oracle at every rank, agreement
with the live reference's fixtures outside near-ties, topk = 1 against corr_to_matches, batch / repeat consistency,
and the argument checks that run before any launch."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import ncnet_topk_oracle as T

pytestmark = pytest.mark.gpu

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
_spec = importlib.util.spec_from_file_location('ncnet_topk_cases', os.path.join(GOLD_DIR, 'ncnet_topk_cases.py'))
K = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(K)


def _topk(*a, **kw):
    from patch2pix_b200.ncnet import corr_to_matches_topk
    return corr_to_matches_topk(*a, **kw)


def _volume(b, shape, kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 1, *shape, generator=g)
    if kind == 'zeros':         # a NeighConsensus stack ends in a ReLU: most entries are exact zeros
        x = torch.relu(x - 1.0)
    elif kind == 'dups':        # few distinct values, negative ones included
        x = torch.randint(-2, 3, x.shape, generator=g).float() * 0.25
    return x


def _deltas(shape, ks, fmt, seed):
    g = torch.Generator().manual_seed(seed)
    d = [torch.randint(0, ks, shape, generator=g) for _ in range(4)]
    return tuple(t.float() for t in d[:3]) + (d[3],) if fmt == 'mixed' else tuple(d)


def _oracle(x, d, k, ks, sm, inv):
    outs = [T.corr_to_matches_topk(x[i, 0], None if d is None else [t[i, 0] for t in d], k, ks, sm, inv)
            for i in range(x.shape[0])]
    return [torch.stack([o[c] for o in outs]) for c in range(5)]


def _check_exact(got, ref):
    assert [t.dtype for t in got] == [torch.int64] * 4 + [torch.float32]
    for c in range(4):
        assert got[c].shape == ref[c].shape
        assert torch.equal(got[c].cpu(), ref[c]), c
    np.testing.assert_allclose(got[4].cpu().double().numpy(), ref[4].numpy(), rtol=1e-5, atol=1e-30)


# (b, (hA, wA, hB, wB), kind): slices of length 1, a single-row grid and a 150-wide B grid, b = 3, many zeros, many
# duplicates, a slice above 8192 cells (two slices per CTA, ranks in three chunks), and 2000-cell slices whose
# 2000 ranks take two chunks
SHAPES = [(1, (1, 1, 2, 3), 'rand'), (2, (3, 2, 1, 1), 'rand'), (1, (1, 7, 1, 150), 'rand'), (3, (4, 5, 3, 6), 'rand'),
          (2, (6, 8, 5, 7), 'zeros'), (2, (5, 6, 7, 4), 'dups'), (1, (96, 90, 2, 3), 'zeros'),
          (1, (40, 50, 3, 4), 'rand')]


@pytest.mark.parametrize('inv', [False, True])
@pytest.mark.parametrize('b, shape, kind', SHAPES)
def test_topk_vs_oracle(b, shape, kind, inv):
    x = _volume(b, shape, kind, sum(shape) + b)
    hA, wA, hB, wB = shape
    n_slice = hB * wB if inv else hA * wA
    for k in sorted({1, min(3, n_slice), min(64, n_slice), n_slice}):
        for sm in (True, False):
            got = _topk(x.cuda(), topk=k, do_softmax=sm, invert_matching_direction=inv)
            _check_exact(got, _oracle(x, None, k, 1, sm, inv))


@pytest.mark.parametrize('fmt', ['mixed', 'int64'])
@pytest.mark.parametrize('ks', [1, 2, 3])
def test_topk_relocalised_vs_oracle(ks, fmt):
    for b, shape, kind in ((2, (4, 3, 5, 6), 'zeros'), (1, (3, 5, 2, 4), 'rand')):
        x = _volume(b, shape, kind, 7 * ks + b)
        d = _deltas(x.shape, ks, fmt, 11 * ks)
        for inv in (False, True):
            for k in (1, 4):
                for sm in (True, False):
                    got = _topk(x.cuda(), tuple(t.cuda() for t in d), topk=k, ksize=ks, do_softmax=sm,
                                invert_matching_direction=inv)
                    _check_exact(got, _oracle(x, d, k, ks, sm, inv))


def _separated(corr, topk, do_softmax, invert, rel=1e-6):
    hA, wA, hB, wB = corr.shape
    v = corr.double().reshape(hA * wA, hB * wB)
    if invert:
        v = v.t()
    s = torch.sort(torch.softmax(v, 0) if do_softmax else v, dim=0, descending=True).values
    gap = s[:-1] - s[1:]
    ok = torch.ones(s.shape, dtype=torch.bool)
    ok[:-1] &= gap > rel * s[:-1].abs()
    ok[1:] &= gap > rel * s[1:].abs()
    ok = ok[:topk]
    return (ok.t() if invert else ok).reshape(-1)


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD_DIR, 'ncnet_topk_golden.npz')))


def test_topk_vs_reference_fixtures(gold):
    for reloc in K.RELOCS:
        ks = max(reloc, 1)
        corr = torch.from_numpy(gold[f'r{reloc}_corr'])
        for key, inv, sm, k, fmt in K.cases(reloc):
            b, _, hA, wA, hB, wB = corr.shape
            n_slice, n = (hB * wB, hA * wA) if inv else (hA * wA, hB * wB)
            kk = n_slice if k == 'all' else k
            d = None
            if fmt is not None:
                d = [torch.from_numpy(gold[f'r{reloc}_d{c}']) for c in 'ijkl']
                d = tuple(t.long() for t in d) if fmt == 'int64' else tuple(d)
                d = tuple(t.cuda() for t in d)
            got = _topk(corr.cuda(), d, topk=kk, ksize=ks, do_softmax=sm, invert_matching_direction=inv)
            assert [str(t.dtype) for t in got] == list(gold[f'{key}_dtypes']), key
            for i in range(b):
                sep = _separated(corr[i, 0], kk, sm, inv)
                pos = torch.arange(kk * n)
                rank = pos % kk if inv else pos // n
                assert sep[rank == 0].double().mean() >= 0.9, key
                assert kk == 1 or sep[rank > 0].any(), key
                for c, name in enumerate(('jA', 'iA', 'jB', 'iB')):
                    ref = torch.from_numpy(gold[f'{key}_{name}'][i])
                    assert got[c][i].shape == ref.shape, key
                    assert torch.equal(got[c][i].cpu()[sep], ref[sep]), (key, i, name)
                np.testing.assert_allclose(got[4][i].cpu().numpy(), gold[f'{key}_score'][i], rtol=1e-5, atol=1e-7,
                                           err_msg=key)


def test_topk1_equals_corr_to_matches(gold):
    from patch2pix_b200.ncnet import corr_to_matches
    cases = [(torch.from_numpy(gold['r0_corr']), None, 1),
             (torch.from_numpy(gold['r2_corr']), tuple(torch.from_numpy(gold[f'r2_d{c}']) for c in 'ijkl'), 2),
             (_volume(2, (6, 8, 5, 7), 'zeros', 3), None, 1), (_volume(1, (5, 6, 7, 4), 'dups', 4), None, 1)]
    for x, d, ks in cases:
        d = None if d is None else tuple(t.cuda() for t in d)
        for inv in (False, True):
            for sm in (True, False):
                got = _topk(x.cuda(), d, topk=1, ksize=ks, do_softmax=sm, invert_matching_direction=inv)
                ref = corr_to_matches(x.cuda(), d, ksize=ks, do_softmax=sm, invert_matching_direction=inv)
                for c in range(4):
                    assert torch.equal(got[c], ref[c])
                torch.testing.assert_close(got[4], ref[4], rtol=1e-6, atol=0)


def test_topk_batch_equals_single_calls_and_repeats():
    x = _volume(3, (7, 9, 8, 6), 'zeros', 21).cuda()
    d = tuple(t.cuda() for t in _deltas(x.shape, 2, 'mixed', 22))
    for inv in (False, True):
        for k in (1, 5, 48):
            batch = _topk(x, d, topk=k, ksize=2, invert_matching_direction=inv)
            again = _topk(x, d, topk=k, ksize=2, invert_matching_direction=inv)
            for c in range(5):
                assert torch.equal(batch[c], again[c])
            for i in range(3):
                one = _topk(x[i:i + 1], tuple(t[i:i + 1] for t in d), topk=k, ksize=2, invert_matching_direction=inv)
                for c in range(5):
                    assert torch.equal(batch[c][i:i + 1], one[c])


def test_topk_rejections_before_any_launch():
    from patch2pix_b200 import _lib
    x = _volume(1, (2, 3, 4, 2), 'rand', 1).cuda()
    d = tuple(torch.zeros(x.shape, dtype=torch.int64, device='cuda') for _ in range(4))
    h = _lib.default_handle(x.device)
    torch.cuda.synchronize()
    n0 = h.launch_count()
    bad = [dict(corr4d=x, topk=0), dict(corr4d=x, topk=7), dict(corr4d=x, topk=9, invert_matching_direction=True),
           dict(corr4d=x.cpu(), topk=1), dict(corr4d=x.double(), topk=1), dict(corr4d=x, delta4d=d, ksize=4, topk=1),
           dict(corr4d=x[:, :, :, :, :, :1].expand(1, 1, 2, 3, 4, 2), delta4d=d[:3], ksize=2, topk=1)]
    for kw in bad:
        with pytest.raises(ValueError):
            _topk(**kw)
    assert h.launch_count() == n0
    _topk(x, topk=6)
    _topk(x, topk=8, invert_matching_direction=True)
