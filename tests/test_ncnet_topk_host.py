"""CPU checks of corr_to_matches_topk: the float64 oracle against the live reference's outputs
(tests/golden/ncnet_topk_golden.npz, make_ncnet_topk_golden.py), its agreement with the oracle's corr_to_matches at
topk = 1, the argument checks that run before any launch, and a ptxas guard for topk.cu."""
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import ncnet_oracle as O
from oracle import ncnet_topk_oracle as T

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
_spec = importlib.util.spec_from_file_location('ncnet_topk_cases', os.path.join(GOLD_DIR, 'ncnet_topk_cases.py'))
K = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(K)


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD_DIR, 'ncnet_topk_golden.npz')))


def separated(corr, topk, do_softmax, invert, rel=1e-6):
    """[topk * N] bool in the output layout: ranks whose float64 value (softmax or raw) differs from both neighbouring
    ranks of the slice's full order by more than rel (relative).  Elsewhere the reference's order is torch.topk's."""
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


def gold_inputs(gold, reloc, fmt):
    corr = torch.from_numpy(gold[f'r{reloc}_corr'])
    if fmt is None:
        return corr, None
    d = [torch.from_numpy(gold[f'r{reloc}_d{n}']) for n in 'ijkl']
    if fmt == 'int64':
        d = [t.long() for t in d]
    return corr, tuple(d)


def test_oracle_topk_vs_reference(gold):
    for reloc in K.RELOCS:
        ks = max(reloc, 1)
        for key, inv, sm, k, fmt in K.cases(reloc):
            corr, d = gold_inputs(gold, reloc, fmt)
            b, _, hA, wA, hB, wB = corr.shape
            n_slice, n = (hB * wB, hA * wA) if inv else (hA * wA, hB * wB)
            kk = n_slice if k == 'all' else k
            assert list(gold[f'{key}_dtypes']) == ['torch.int64'] * 4 + ['torch.float32'], key
            for i in range(b):
                got = T.corr_to_matches_topk(corr[i, 0], None if d is None else [t[i, 0] for t in d], kk, ks, sm, inv)
                ref = [gold[f'{key}_{c}'][i] for c in ('jA', 'iA', 'jB', 'iB', 'score')]
                assert all(r.shape == (kk * n,) for r in ref), key
                # layout: rank-major forward (position r * N + s is B cell s), cell-major inverted (s * k + r)
                pos = np.arange(kk * n)
                cell = pos // kk if inv else pos % n
                own = (ref[1], ref[0], hA, wA) if inv else (ref[3], ref[2], hB, wB)
                assert np.array_equal(own[0] // ks, cell // own[3]) and np.array_equal(own[1] // ks, cell % own[3])
                sep = separated(corr[i, 0], kk, sm, inv).numpy()
                assert sep.any(), key
                for c in range(4):
                    assert np.array_equal(got[c].numpy()[sep], ref[c][sep]), (key, i, c)
                np.testing.assert_allclose(got[4].numpy(), ref[4], rtol=1e-5, err_msg=key)


def test_oracle_topk1_equals_corr_to_matches(gold):
    g = torch.Generator().manual_seed(5)
    vols = [torch.from_numpy(gold['r0_corr'][1, 0]), torch.relu(torch.randn(3, 4, 5, 2, generator=g))]
    d2 = [torch.from_numpy(gold[f'r2_d{n}'][0, 0]) for n in 'ijkl']
    cases = [(v, None, 1) for v in vols] + [(torch.from_numpy(gold['r2_corr'][0, 0]), d2, 2)]
    for corr, d, ks in cases:
        for inv in (False, True):
            for sm in (True, False):
                got = T.corr_to_matches_topk(corr, d, 1, ks, sm, inv)
                ref = O.corr_to_matches(corr, d, ks, sm, 'positive', inv, True)
                for c in range(4):
                    assert torch.equal(got[c], ref[c])
                torch.testing.assert_close(got[4], ref[4], rtol=1e-12, atol=0)


def test_topk_rejects_bad_arguments_before_any_launch():
    from patch2pix_b200.ncnet import corr_to_matches_topk
    for x in (torch.zeros(1, 1, 2, 3, 2, 2), torch.zeros(1, 1, 2, 3, 2, 2, dtype=torch.float64),
              torch.zeros(1, 2, 2, 3, 2, 2), torch.zeros(1, 2, 3, 2, 2)):
        with pytest.raises(ValueError):
            corr_to_matches_topk(x, topk=1)


def test_topk_kernels_compile_without_spills(tmp_path):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'topk.cu'), '-o', str(tmp_path / 't.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-2000:]
    spills = [int(a) + int(c) for a, c in re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)]
    assert len(spills) == 2 and not any(spills), log       # corr_topk_kernel<forward / inverted>
