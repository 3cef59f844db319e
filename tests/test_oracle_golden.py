"""Pin the CPU oracle (oracle/p2p_oracle.py) against golden vectors produced by the
live reference (tests/golden/make_golden.py).  Integer outputs must be identical;
float outputs use a tolerance that only allows for CPU-ISA-dependent library
rounding (the authoring container reproduces them bit-for-bit)."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from patch2pix_b200.synth import synthetic_pair, synthetic_pair_shifted, synthetic_pair_sized

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
RTOL, ATOL = 2e-4, 2e-5


def _close(a, b, rtol=RTOL, atol=ATOL):
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=atol)


@pytest.mark.parametrize('name', ['stages_96x128', 'stages_128x96', 'stages_shift_128x160'])
def test_coarse_stages_and_predict_fine(name, seeded_sd, consensus_sd):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    gen = synthetic_pair_shifted if 'shift' in name else synthetic_pair
    seeded_sd = consensus_sd if 'shift' in name else seeded_sd
    im1, im2 = gen(int(g['pair_idx']), int(g['H']), int(g['W']))
    with torch.no_grad():
        f1 = O.backbone_forward_all(im1, seeded_sd)
        f2 = O.backbone_forward_all(im2, seeded_sd)
        for lvl in (1, 2, 3, 4):
            _close(f1[lvl][0, ::7, ::3, ::3], g[f'feat1_l{lvl}_sub'], rtol=1e-3, atol=1e-4)
        st = {}
        corr4d, delta4d = O.forward_coarse_match(f1[-1], f2[-1], seeded_sd, ksize=2, stages=st)
        _close(st['pooled'], g['pooled'])
        assert np.array_equal(np.stack([d.numpy() for d in delta4d]), g['delta'])
        _close(st['mutual1'], g['mutual1'])
        _close(st['ncn'], g['ncn'])
        _close(corr4d, g['corr4d'])
        cm, sc = O.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=8, center=True)
        assert cm.dtype == torch.int64
        assert np.array_equal(cm.numpy(), g['cand_matches'])
        _close(sc, g['cand_scores'])
        fm, fs = O.filter_coarse(cm, sc, 0.0, True)
        assert np.array_equal(fm[0].numpy(), g['mutual_matches'])
        _close(fs[0], g['mutual_scores'])
        fine, fine_p, mid, mid_p, coarse = O.predict_fine(im1, im2, seeded_sd, ksize=2, return_all=True)
        assert np.array_equal(coarse[0].numpy(), g['coarse'])
        _close(mid[0].reshape(-1, 4), g['mid'], atol=1e-3)
        _close(fine[0].reshape(-1, 4), g['fine'], atol=1e-3)
        _close(mid_p[0].reshape(-1), g['mid_p'], atol=1e-4)
        _close(fine_p[0].reshape(-1), g['fine_p'], atol=1e-4)
        pm, ps = O.predict_coarse(im1, im2, seeded_sd, ksize=2, ncn_thres=0.0, mutual=False)
        assert np.array_equal(pm[0].numpy(), g['predict_coarse_nomutual_matches'])
        _close(ps[0], g['predict_coarse_nomutual_scores'])


@pytest.mark.parametrize('name', ['trainseq_96x128', 'trainseq_shift_160x240'])
def test_train_forward_sequence(name, seeded_sd, consensus_sd):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    gen = synthetic_pair_shifted if 'shift' in name else synthetic_pair
    seeded_sd = consensus_sd if 'shift' in name else seeded_sd
    im1, im2 = gen(int(g['pair_idx']), int(g['H']), int(g['W']))
    with torch.no_grad():
        np.random.seed(int(g['np_seed']))
        fine, fine_p, mid, mid_p, anchors = O.train_forward_sequence(
            im1, im2, seeded_sd, ksize=2, ptmax=int(g['ptmax']), panc=8, return_all=True)
    assert np.array_equal(anchors[0].numpy(), g['anchors'])
    _close(mid[0], g['mid'], atol=1e-3)
    _close(fine[0], g['fine'], atol=1e-3)
    _close(mid_p[0], g['mid_p'], atol=1e-4)
    _close(fine_p[0], g['fine_p'], atol=1e-4)


@pytest.mark.parametrize('name', ['unequal_96x128_128x96', 'unequal_128x160_96x224'])
def test_unequal_sizes_predict_fine(name, consensus_sd):
    """Images of different sizes (transposed aspect; H1 > H2 with W1 < W2): every per-image size the reference uses --
    the 4D volume's two grids, the patch gathers' clamps, the regressor outputs' clamps -- must be the right image's."""
    g = np.load(os.path.join(GOLD, name + '.npz'))
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    assert im1.shape[2:] != im2.shape[2:]
    with torch.no_grad():
        f1 = O.backbone_forward_all(im1, consensus_sd)
        f2 = O.backbone_forward_all(im2, consensus_sd)
        st = {}
        corr4d, delta4d = O.forward_coarse_match(f1[-1], f2[-1], consensus_sd, ksize=2, stages=st)
        _close(st['pooled'], g['pooled'])
        assert np.array_equal(np.stack([d.numpy() for d in delta4d]), g['delta'])
        _close(st['ncn'], g['ncn'])
        _close(corr4d, g['corr4d'])
        cm, sc = O.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=8, center=True)
        assert np.array_equal(cm.numpy(), g['cand_matches'])
        _close(sc, g['cand_scores'])
        fine, fine_p, mid, mid_p, coarse = O.predict_fine(im1, im2, consensus_sd, ksize=2, return_all=True)
        assert np.array_equal(coarse[0].numpy(), g['coarse'])
        _close(mid[0].reshape(-1, 4), g['mid'], atol=1e-3)
        _close(fine[0].reshape(-1, 4), g['fine'], atol=1e-3)
        _close(mid_p[0].reshape(-1), g['mid_p'], atol=1e-4)
        _close(fine_p[0].reshape(-1), g['fine_p'], atol=1e-4)


def test_unequal_sizes_train_forward_sequence(consensus_sd):
    g = np.load(os.path.join(GOLD, 'unequal_trainseq_160x240_192x128.npz'))
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    with torch.no_grad():
        np.random.seed(int(g['np_seed']))
        fine, fine_p, mid, mid_p, anchors = O.train_forward_sequence(
            im1, im2, consensus_sd, ksize=2, ptmax=int(g['ptmax']), panc=8, return_all=True)
    assert np.array_equal(anchors[0].numpy(), g['anchors'])
    _close(mid[0], g['mid'], atol=1e-3)
    _close(fine[0], g['fine'], atol=1e-3)
    _close(mid_p[0], g['mid_p'], atol=1e-4)
    _close(fine_p[0], g['fine_p'], atol=1e-4)


def test_refine_matches(seeded_sd):
    g = np.load(os.path.join(GOLD, 'refine_128x160.npz'))
    im1, im2 = synthetic_pair(int(g['pair_idx']), int(g['H']), int(g['W']))
    cm = torch.from_numpy(g['coarse_in'])
    with torch.no_grad():
        r, s, c = O.refine_matches(im1, im2, cm.clone(), seeded_sd, io_thres=0.0)
        rt, st_, ct = O.refine_matches(im1, im2, cm.clone(), seeded_sd, io_thres=0.5)
    _close(r, g['refined'], atol=1e-3)
    _close(s, g['scores'], atol=1e-4)
    _close(c, g['coarse'])
    assert rt.shape == g['refined_t'].shape
    _close(rt, g['refined_t'], atol=1e-3)
    _close(ct, g['coarse_t'])


def test_shift_to_anchors_and_filter_quirks():
    m = [torch.tensor([[12, 20, 28, 36], [4, 4, 4, 4]])]
    a = O.shift_to_anchors(m, panc=8)[0]
    assert a.shape == (16, 4)
    assert a[0].tolist() == [4, 12, 28, 36] and a[7].tolist() == [12, 20, 36, 44]
    assert a[8].tolist() == [-4, -4, 4, 4]
    # no duplicate rows -> the mutual filter is skipped and every row survives unsorted (utils.py:48-50)
    cm = [torch.tensor([[9, 1, 1, 1], [3, 1, 1, 1], [5, 1, 1, 1]])]
    sc = [torch.tensor([0.3, 0.2, 0.1])]
    fm, fs = O.filter_coarse(cm, sc, 0.0, True)
    assert fm[0].tolist() == cm[0].tolist()
    # one mutual row -> first-occurrence score, lexicographic order
    cm = [torch.tensor([[9, 1, 1, 1], [3, 1, 1, 1], [9, 1, 1, 1], [3, 1, 1, 1]])]
    sc = [torch.tensor([0.3, 0.2, 0.9, 0.8])]
    fm, fs = O.filter_coarse(cm, sc, 0.0, True)
    assert fm[0].tolist() == [[3, 1, 1, 1], [9, 1, 1, 1]]
    assert fs[0].tolist() == pytest.approx([0.2, 0.3])


def test_filter_coarse_branches_vs_live_reference():
    """Every branch of networks/utils.py:38-72 (mutual skip, threshold skip, ptmax fill / cut / degenerate ids, numpy
    RNG order) on crafted candidate lists: fixtures written by the live reference (`make_golden.py filter`)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('filter_cases', os.path.join(GOLD, 'filter_cases.py'))
    fc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fc)
    g = np.load(os.path.join(GOLD, 'filter_quirks.npz'))
    for cname, kind, thres, mutual, ptmax, seed in fc.FILTER_CASES:
        rows, scores = fc.filter_case_inputs(kind)
        np.random.seed(seed)
        fm, fs = O.filter_coarse([rows.clone()], [scores.clone()], thres, mutual, ptmax=ptmax)
        assert np.array_equal(fm[0].numpy(), g[cname + '_matches']), cname
        assert np.array_equal(fs[0].numpy(), g[cname + '_scores']), cname
