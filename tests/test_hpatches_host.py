"""The HPatches evaluation's host side (patch2pix_b200.hpatches, oracle/hpatches_oracle.py): the sequence reader, the
synthetic tree, the numpy restatement of the statistics and the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import hpatches_oracle as O
from patch2pix_b200.hpatches import D2NET_EXCLUDED, read_hpatches, summarize
from patch2pix_b200.synth import synthetic_hpatches_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('hpatches'))
    names = ['v_zz', ('i_b', (97, 65)), 'v_a', 'i_dc', ('v_m', (120, 90))]
    return root, synthetic_hpatches_tree(root, 3, names)


def test_reader_order_and_exclude(tree):
    root, Hs = tree
    seqs = read_hpatches(root)
    assert [s.name for s in seqs] == ['i_b', 'v_a', 'v_m', 'v_zz']           # sorted, i_dc excluded by default
    assert 'i_dc' in D2NET_EXCLUDED and len(D2NET_EXCLUDED) == 8
    assert [s.split for s in seqs] == ['i', 'v', 'v', 'v']
    s = seqs[0]
    assert s.size == (97, 65)
    assert [os.path.basename(p) for p in s.paths] == [f'{k}.ppm' for k in range(1, 7)]
    assert len(s.H_gt) == 5
    assert [s.name for s in read_hpatches(root, exclude=())] == ['i_b', 'i_dc', 'v_a', 'v_m', 'v_zz']
    assert [s.name for s in read_hpatches(root, exclude=('v_a', 'i_b'))] == ['i_dc', 'v_m', 'v_zz']


def test_reader_rejects_bad_name_and_missing_file(tmp_path):
    root = str(tmp_path)
    synthetic_hpatches_tree(root, 0, [('i_ok', (64, 48)), ('x_bad', (64, 48))])
    with pytest.raises(ValueError, match='x_bad'):
        read_hpatches(root)
    assert [s.name for s in read_hpatches(root, exclude=('x_bad',))] == ['i_ok']
    os.remove(os.path.join(root, 'i_ok', 'H_1_4'))
    with pytest.raises(FileNotFoundError, match=r'i_ok.H_1_4'):
        read_hpatches(root, exclude=('x_bad',))
    with pytest.raises(FileNotFoundError):
        read_hpatches(os.path.join(root, 'nowhere'))


def test_synthetic_tree_round_trip(tree):
    root, Hs = tree
    for name, H_list in Hs.items():
        for k, H in zip(range(2, 7), H_list):
            back = np.loadtxt(os.path.join(root, name, f'H_1_{k}'))
            assert back.dtype == np.float64 and np.array_equal(back.view(np.int64), H.view(np.int64)), (name, k)
            assert H[2, 2] == 1.0
    again = synthetic_hpatches_tree(os.path.join(root, 'again'), 3, ['v_zz', ('i_b', (97, 65))])
    assert all(np.array_equal(a, b) for a, b in zip(again['v_zz'], Hs['v_zz']))


def test_oracle_identity_and_offsets():
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 500, (200, 2))
    d = O.reprojection_errors(np.concatenate([p, p], 1), np.eye(3))
    assert np.all(d == 0)
    assert O.counts(d, [1, 2]).tolist() == [200, 200, 200]
    # translated rows at known offsets: offset j + 0.5 px along x for rows of group j
    off = np.repeat(np.arange(10) + 0.5, 20)
    rows = np.concatenate([p, p + np.stack([off, np.zeros_like(off)], 1)], 1)
    d = O.reprojection_errors(rows, np.eye(3))
    np.testing.assert_allclose(d, off, rtol=0, atol=1e-9)
    c = O.counts(d, range(1, 11))
    assert c.tolist() == [20 * t for t in range(1, 11)] + [200]
    np.testing.assert_array_equal(O.pair_mma(c), np.arange(1, 11) / 10)
    # a translation H: the error is the distance to the translated point
    T = np.array([[1.0, 0, 3.0], [0, 1.0, -4.0], [0, 0, 1.0]])
    np.testing.assert_allclose(O.reprojection_errors(np.concatenate([p, p], 1), T), 5.0, rtol=0, atol=1e-9)
    # NaN and inf are never correct
    bad = np.array([[np.nan, 1, 1, 1], [1, 1, np.inf, 1], [1, 1, 1, 1]])
    assert O.counts(O.reprojection_errors(bad, np.eye(3)), [1, 1e300]).tolist() == [1, 1, 3]


def test_oracle_empty_pair():
    c = O.counts(O.reprojection_errors(np.zeros((0, 4)), np.eye(3)), range(1, 11))
    assert c.tolist() == [0] * 11
    assert np.all(O.pair_mma(c) == 0)


def test_oracle_corner_error():
    H = np.array([[1.0, 0.1, 5.0], [0.02, 0.9, -3.0], [1e-4, 2e-4, 1.0]])
    assert O.corner_error(H, H, 10, 640, 480) == 0.0
    T = np.eye(3)
    T[0, 2] = 2.0
    assert O.corner_error(np.eye(3), T, 10, 640, 480) == 2.0
    assert O.corner_error(np.eye(3), np.eye(3), 0, 640, 480) == np.inf       # no model
    assert O.corner_error(np.eye(3), np.eye(3), -1, 640, 480) == np.inf
    # a corner mapped to w = 0: corner (w-1, 0) = (99, 0) under a predicted H with w = 1 - x / 99
    Hw = np.eye(3)
    Hw[2, 0] = -1.0 / 99.0
    assert O.project(Hw, 99.0, 0.0)[2] == 0.0
    assert O.corner_error(np.eye(3), Hw, 10, 100, 50) == np.inf
    assert O.corner_error(Hw, np.eye(3), 10, 100, 50) == np.inf
    assert O.corner_error(np.eye(3), np.full((3, 3), np.nan), 10, 100, 50) == np.inf


def _rec(seq, counts, corner):
    from argparse import Namespace
    return Namespace(seq=seq, k=2, N=int(counts[-1]), n_inliers=0, corner_err=corner,
                     counts=np.asarray(counts, dtype=np.int32), match_failed=False)


def test_split_summary_with_empty_split():
    recs = [_rec('v_a', [1, 2, 4], 0.5), _rec('v_a', [0, 0, 0], np.inf), _rec('v_b', [3, 3, 3], 2.0)]
    mma, hacc = summarize(recs, [1, 3])
    np.testing.assert_allclose(mma['v'], [(0.25 + 0 + 1) / 3, (0.5 + 0 + 1) / 3])
    np.testing.assert_array_equal(mma['all'], mma['v'])
    assert np.all(np.isnan(mma['i'])) and mma['i'].shape == (2,)
    np.testing.assert_allclose(hacc['v'], [1 / 3, 2 / 3])
    assert np.all(np.isnan(hacc['i'])) and hacc['i'].shape == (2,)
    om, oh = O.split_summary([r.seq for r in recs], [O.pair_mma(r.counts) for r in recs],
                             [r.corner_err for r in recs], [1, 3])
    for s in ('all', 'i', 'v'):
        np.testing.assert_array_equal(om[s], mma[s])
        np.testing.assert_array_equal(oh[s], hacc[s])


def test_cli_help():
    r = subprocess.run([sys.executable, '-m', 'patch2pix_b200.hpatches', '--help'], cwd=ROOT, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for opt in ('--ckpt', '--data_root', '--method', '--ksize', '--io_thres', '--ncn_thres', '--imsize',
                '--ransac_thres'):
        assert opt in r.stdout


def test_kernel_compiles_without_spills(tmp_path):
    import re
    import shutil
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'hpatches.cu'), '-o',
                                   str(tmp_path / 'h.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    found = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', r.stdout + r.stderr)
    assert [int(st) + int(ld) for st, ld in found] == [0]          # one kernel, no spills
