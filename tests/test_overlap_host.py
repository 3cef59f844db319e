"""Host side of the overlap precompute: the COLMAP reader's 2D points and the numpy oracle against the reference's own
outputs (tests/golden/make_ovs_golden.py), the synthetic model writer, and the build of overlap.cu."""
import json
import os
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest

from oracle import overlap_oracle as O
from patch2pix_b200 import evaluation as E
from patch2pix_b200.synth import write_colmap_model

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
MODELS = os.path.join(GOLDEN, 'ovs_colmap')
CASES = ('edge', 'random40', 'two_empty', 'one', 'zero')


@pytest.fixture(scope='module')
def golden():
    z = np.load(os.path.join(GOLDEN, 'ovs_golden.npz'))
    return z, json.loads(str(z['results_json']))


def _images(case, **kw):
    return E.read_images_binary(os.path.join(MODELS, case, 'images.bin'), **kw)


@pytest.mark.parametrize('case', CASES)
def test_reader_points2D_matches_reference(golden, case):
    z, res = golden
    ims = _images(case, points2D=True)
    assert list(ims) == res[case]['image_ids'] and [im.name for im in ims.values()] == res[case]['names']
    assert len(ims) == int(z[f'{case}_n'])
    for k, im in enumerate(ims.values()):
        ids, xys = z[f'{case}_ids_{k}'], z[f'{case}_xys_{k}']
        assert im.point3D_ids.dtype == np.int64 and im.point3D_ids.shape == (len(ids),)
        assert im.xys.dtype == np.float64 and im.xys.shape == (len(ids), 2)
        if len(ids):                              # the reference's empty lists are float64 [0] / [0, 2]: values only
            assert ids.dtype == np.int64 and xys.dtype == np.float64
        assert np.array_equal(im.point3D_ids, ids) and np.array_equal(im.xys, xys)
        assert im.point3D_ids.flags.writeable and im.xys.flags.c_contiguous


def test_default_reader_unchanged():
    for case in CASES:
        plain, full = _images(case), _images(case, points2D=True)
        assert list(plain) == list(full)
        for a, b in zip(plain.values(), full.values()):
            assert sorted(vars(a)) == ['camera_id', 'id', 'name', 'qvec', 'tvec']
            assert all(np.array_equal(getattr(a, f), getattr(b, f)) for f in vars(a))


def test_truncated_points_raise(tmp_path):
    src = os.path.join(MODELS, 'edge', 'images.bin')
    buf = open(src, 'rb').read()
    for cut in (len(buf) - 1, len(buf) - 24, len(buf) - 30):
        p = tmp_path / f'images_{cut}.bin'
        p.write_bytes(buf[:cut])
        for kw in ({}, {'points2D': True}):
            with pytest.raises(ValueError, match='truncated'):
                E.read_images_binary(str(p), **kw)


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(golden, case):
    z, res = golden
    ids = [z[f'{case}_ids_{k}'] for k in range(int(z[f'{case}_n']))]
    if 'cal_overlap_scores' in res[case]:
        assert res[case]['cal_overlap_scores'] == {'raises': 'ZeroDivisionError'}
        with pytest.raises(ZeroDivisionError):
            O.cal_overlap_scores(ids)
        return
    ov, nums = O.cal_overlap_scores(ids)
    assert ov.dtype == z[f'{case}_ov'].dtype and np.array_equal(ov, z[f'{case}_ov'])
    assert nums.dtype == z[f'{case}_nums'].dtype and np.array_equal(nums, z[f'{case}_nums'])
    names = res[case]['names']
    for t, want in res[case]['pair_names'].items():
        assert [list(p) for p in O.pairs(ov, names, float(t))] == want, t
    if len(ids) > 1:
        ex, cnt = O.exact_scores(ids)
        assert np.array_equal(ex, ov) and np.array_equal(cnt, nums)


def test_oracle_quirks(golden):
    z, res = golden
    ov, nums = z['edge_ov'], z['edge_nums']
    assert nums[0] == 0 and np.count_nonzero(nums == 0) == 1
    assert ov[7, 8] == 1.0 and [7, 8] not in res['edge']['pairs']['0.1']     # identical sets are dropped
    assert ov[10, 11] == 0.3 and [10, 11] in res['edge']['pairs']['0.3']      # exactly 3 / 10 passes t = 0.3
    assert ov[12, 13] == 0.2 and [12, 13] in res['edge']['pairs']['0.2']
    n = len(nums)                                 # t <= 0 also takes every zero below the diagonal
    assert len(res['edge']['pairs']['0']) == np.count_nonzero((ov >= 0) & (ov < 1)) > n * (n - 1) // 2
    assert res['edge']['pairs']['nan'] == []


def test_write_colmap_model_points(tmp_path):
    q, t = [1.0, 0.0, 0.0, 0.0], [0.5, -1.0, 2.0]
    write_colmap_model(str(tmp_path / 'a'), [(1, 0, 64, 48, [50.0, 32.0, 24.0])], [(3, q, t, 1, 'x.jpg')])
    want = struct.pack('<Q', 1) + struct.pack('<i7di', 3, *q, *t, 1) + b'x.jpg\x00' + struct.pack('<Q', 0)
    assert (tmp_path / 'a' / 'images.bin').read_bytes() == want              # without ids: the same bytes as before
    ids = np.array([-1, 0, 5, 2 ** 40, 7])
    write_colmap_model(str(tmp_path / 'b'), [(1, 0, 64, 48, [50.0, 32.0, 24.0])],
                       [(3, q, t, 1, 'x.jpg', ids), (4, q, t, 1, 'y.jpg')])
    ims = E.read_images_binary(str(tmp_path / 'b' / 'images.bin'), points2D=True)
    assert np.array_equal(ims[3].point3D_ids, ids) and np.array_equal(ims[3].xys[:, 0], np.arange(5))
    assert len(ims[4].point3D_ids) == 0 and ims[4].xys.shape == (0, 2)


def test_overlap_kernels_compile_without_spills(tmp_path):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'overlap.cu'), '-o', str(tmp_path / 'o.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    found = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', r.stdout + r.stderr)
    assert [int(st) + int(ld) for st, ld in found] == [0, 0]                  # pack and count kernels
