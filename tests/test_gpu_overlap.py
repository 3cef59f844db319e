"""GPU side of the overlap precompute: p2p_overlap_scores and the pair lists against the reference's own outputs
(tests/golden/make_ovs_golden.py) and an exact int64 Gram matrix, the ov_pairs.npy cache semantics, the device-to-host
copies per scene and the precompute script over a two-scene tree."""
import contextlib
import ctypes as C
import io
import json
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import overlap_oracle as O
from patch2pix_b200 import _lib
from patch2pix_b200 import evaluation as E
from patch2pix_b200.synth import synthetic_overlap_images, write_colmap_model

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
MODELS = os.path.join(GOLDEN, 'ovs_colmap')
CASES = ('edge', 'random40', 'two_empty', 'one', 'zero')
THRESHOLDS = [-0.5, 0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.8, 1.0, float('nan')]
CAMERA = [(1, 0, 640, 480, [500.0, 320.0, 240.0])]


@pytest.fixture(scope='module')
def golden():
    z = np.load(os.path.join(GOLDEN, 'ovs_golden.npz'))
    return z, json.loads(str(z['results_json']))


def _printed(fn, *a, **kw):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        res = fn(*a, **kw)
    return res, buf.getvalue().splitlines()


def _as_json(d):
    return [[repr(k), [list(p) for p in v]] for k, v in d.items()]


@pytest.mark.parametrize('case', CASES)
def test_scores_and_pairs_match_reference(golden, case, tmp_path):
    z, res = golden
    ims = E.read_images_binary(os.path.join(MODELS, case, 'images.bin'), points2D=True)
    model = tmp_path / 'sparse'
    model.mkdir()
    shutil.copy(os.path.join(MODELS, case, 'images.bin'), model)
    if 'cal_overlap_scores' in res[case]:
        with pytest.raises(ZeroDivisionError):
            E.cal_overlap_scores(list(ims), ims)
        with pytest.raises(ZeroDivisionError):
            E.sav_model_multi_ov_pairs(str(model), [0.1])
        with pytest.raises(ZeroDivisionError):
            E.load_model_ov_pairs(str(model), 0.3)
        return
    ov, nums = E.cal_overlap_scores(list(ims), ims)
    for got, want in ((ov, z[f'{case}_ov']), (nums, z[f'{case}_nums'])):
        assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want)
    names, scores = E._model_scores(str(model), 'cuda')
    got = E._pairs_by_threshold(names, scores, THRESHOLDS)                 # every threshold in one nonzero
    for t, pairs in zip(THRESHOLDS, got):
        assert [list(p) for p in pairs] == res[case]['pair_names'][repr(t)], t
        assert all(type(a) is str and type(b) is str for a, b in pairs)
    # ov_pairs.npy: fresh with a duplicated key, then a complete file, then an incomplete one
    for run in res[case]['sav_model_multi_ov_pairs']:
        d, lines = _printed(E.sav_model_multi_ov_pairs, str(model), run['overlaps'])
        assert lines == run['lines'] and _as_json(d) == run['dict']
        assert _as_json(np.load(model / 'ov_pairs.npy', allow_pickle=True).item()) == run['file']
    pairs, lines = _printed(E.load_model_ov_pairs, str(model), 0.3)
    assert lines == res[case]['load_model_ov_pairs']['lines']
    assert [list(p) for p in pairs] == res[case]['load_model_ov_pairs']['pairs']


def _seeded(n, seed):
    """Mixed densities and sizes up to 9000 keypoints (mostly not a multiple of 32), two pairs of identical sets, one
    image without a valid index and one with a single keypoint."""
    ims = synthetic_overlap_images(seed, n, n2d=9000, frac=(0.02, 0.98), vary_n2d=True, identical=[(1, n - 1), (5, 7)])
    ids = [im[5] for im in ims]
    for a in ids:
        if not np.any(a > 0):
            a[-1] = 1                             # a second empty image would raise ZeroDivisionError
    ids[3] = np.full(len(ids[3]), -1)
    ids[n // 2] = np.array([17])
    return ids


@pytest.mark.parametrize('n', [63, 64, 65, 129, 700])
def test_scores_bit_equal_exact_gram(n):
    ids = _seeded(n, n)
    want, cnt = O.exact_scores(ids)
    scores, counts = E.overlap_scores_device(ids)
    assert np.array_equal(counts.cpu().numpy(), cnt)
    got = scores.cpu().numpy()
    assert got.dtype == np.float64 and np.array_equal(got, want)
    assert np.count_nonzero(got == 1.0) == n + 2                              # the diagonal and the identical pairs


def _call(ids, offsets, words, scores):
    h = _lib.default_handle('cuda')
    flat = torch.from_numpy(ids).cuda()
    off = torch.from_numpy(offsets).cuda()
    n = len(offsets) - 1
    bits = torch.empty(max(n * words, 1), dtype=torch.int32, device='cuda')
    counts = torch.empty(max(n, 1), dtype=torch.int32, device='cuda')
    return h.lib.p2p_overlap_scores(h.h, _lib.ptr(flat), _lib.ptr(off), offsets.ctypes.data_as(C.POINTER(C.c_int64)),
                                    n, words, _lib.ptr(bits), _lib.ptr(counts), _lib.ptr(scores), h.stream())


def test_scores_independent_of_buffer_and_deterministic():
    ids = _seeded(129, 3)
    flat = np.concatenate(ids)
    offsets = np.concatenate([[0], np.cumsum([len(a) for a in ids])]).astype(np.int64)
    words = int((np.diff(offsets).max() + 31) // 32)
    outs = []
    for fill in (float('nan'), 7.0, None):
        scores = torch.full((129, 129), fill, dtype=torch.float64, device='cuda') if fill is not None else \
            torch.empty(129, 129, dtype=torch.float64, device='cuda')
        assert _call(flat, offsets, words, scores) == 0
        outs.append(scores.cpu().numpy())
    assert all(o.tobytes() == outs[0].tobytes() for o in outs[1:])
    assert np.array_equal(outs[0], O.exact_scores(ids)[0])


def test_invalid_arguments_raise():
    ids = np.array([1, 2, 3, -1, 5], dtype=np.int64)
    scores = torch.empty(2, 2, dtype=torch.float64, device='cuda')
    lib = _lib.load()
    assert _call(ids, np.array([0, 3, 2], dtype=np.int64), 1, scores) == -1          # decreasing offsets
    assert b'non-decreasing' in lib.p2p_last_error()
    assert _call(ids, np.array([0, 2, 5], dtype=np.int64), 0, scores) == -1          # words too small
    assert _call(ids, np.array([0, 2, 5], dtype=np.int64), 1, None) == -1            # null output
    h = _lib.default_handle('cuda')
    big = np.zeros((1 << 20) + 2, dtype=np.int64)
    assert h.lib.p2p_overlap_scores(h.h, None, None, big.ctypes.data_as(C.POINTER(C.c_int64)), (1 << 20) + 1, 0, None,
                                    None, None, h.stream()) == -1                   # more than 2^20 images
    assert _call(ids, np.array([0, 2, 5], dtype=np.int64), 1, scores) == 0


def test_sav_model_device_to_host_copies(tmp_path):
    from torch.profiler import ProfilerActivity, profile
    write_colmap_model(str(tmp_path), CAMERA, synthetic_overlap_images(1, 300, n2d=2000))

    def dtoh():
        if (tmp_path / 'ov_pairs.npy').exists():
            os.remove(tmp_path / 'ov_pairs.npy')
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            _printed(E.sav_model_multi_ov_pairs, str(tmp_path), [0.1, 0.2, 0.3, 0.4, 0.5])
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if 'Memcpy DtoH' in e.name)

    dtoh()                                                                   # warm-up
    n = dtoh()
    assert 1 <= n <= 2, n
    d = np.load(tmp_path / 'ov_pairs.npy', allow_pickle=True).item()
    assert sum(len(v) for v in d.values()) > 0


def test_precompute_two_scenes(tmp_path):
    overlaps = [0.1, 0.2, 0.3, 0.4, 0.5]
    scenes = {}
    for k, (scene, n) in enumerate((('s_a', 70), ('s_b', 33))):
        ims = synthetic_overlap_images(10 + k, n, n2d=600, vary_n2d=True, identical=[(0, 2)])
        write_colmap_model(str(tmp_path / scene / 'dense' / 'sparse'), CAMERA, ims)
        scenes[scene] = ims
    _, lines = _printed(E.precompute_immatch_val_ovs, str(tmp_path))
    listed = os.listdir(tmp_path)
    assert lines[0] == f'Target scenes: {listed}, ovs: {overlaps}' and lines[1] == ''
    for scene in listed:
        ims = scenes[scene]
        ov, _ = O.cal_overlap_scores([im[5] for im in ims])
        names = [im[4] for im in ims]
        d = np.load(tmp_path / scene / 'dense' / 'sparse' / 'ov_pairs.npy', allow_pickle=True).item()
        assert list(d) == overlaps
        for t in overlaps:
            assert d[t] == O.pairs(ov, names, t), (scene, t)
        i = lines.index(f'Start processing scene: {scene}')
        assert lines[i + 1:i + 6] == [f'ov>{t} pairs: {len(d[t])}' for t in overlaps]
        assert lines[i + 6].startswith('Finished, time ')
    np.random.seed(0)
    sel = E.select_pairs(str(tmp_path), sample_max=10 ** 6, min_overlap=0.3)
    assert [(s, len(p)) for s, _, p in sel] == [(s, len(np.load(tmp_path / s / 'dense' / 'sparse' / 'ov_pairs.npy',
                                                                allow_pickle=True).item()[0.3])) for s in listed]
    assert all(a in ims and b in ims for _, ims, p in sel for a, b in p)
