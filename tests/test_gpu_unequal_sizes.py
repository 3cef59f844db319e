"""Image pairs of DIFFERENT sizes (H1 x W1 != H2 x W2) through the CUDA path, against the CPU oracle and against golden
vectors of the live reference.

This is how the reference's callers use it: load_im_flexible rescales each image on its own, so a portrait photo
matched against a landscape one gives two grids of different shapes.  Many places in the kernels pick a size by image
index (the two padded maps of the L2-normalise / permute launch, the GEMM's m- and n-tile counts, the window maps,
window-origin and output clamps, the window-sharing classifier, the scale factors of estimate_matches); with equal
images a mix-up between image 1 and image 2 is invisible.  Tolerances are those of test_gpu_parity.py.
"""
import json
import os

import numpy as np
import pytest
import torch

from test_gpu_parity import GOLD, OUT, _assert_e2e, _cfg, _delta_mismatch_report, _e2e_report, _tie_masks

pytestmark = pytest.mark.gpu

# name: (pair index, image 1 (H, W), image 2 (H, W)); the layer-3 map is /8, the pooled grid /16
CASES = {
    'transposed': (1, (96, 128), (128, 96)),        # H/W swaps between the images
    'crossed': (21, (128, 160), (96, 224)),         # H1 > H2 while W1 < W2: a swap of H alone or W alone shows
    'tiles': (5, (240, 320), (160, 192)),           # n1 = 1200 (10 m-tiles) against n2 = 480 (2 n-tiles); pooled 15x20 vs 10x12
    'reversed': (5, (160, 192), (240, 320)),        # the same with the GEMM roles swapped
    'tiny': (7, (64, 64), (480, 640)),              # nA = 16 (less than one tile) against 30x40
    'bench': (3, (480, 640), (640, 480)),           # portrait against landscape at the benchmark size
}
DEFAULTS = {'corr_passes': 3, 'nc_l2_mode': 0, 'gemm_impl': 0, 'mid_passes': 3, 'fine_passes': 1, 'mid_band': 26,
            'fuse_gather': 3, 'fc_impl': 1, 'share_windows': 1}


def _report(name, payload):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, f'unequal_{name}.json'), 'w') as f:
        json.dump(payload, f, indent=1)


def _restore(net):
    for k, v in DEFAULTS.items():
        net.set_option(k, v)


@pytest.fixture(scope='module')
def nets(seeded_sd, consensus_sd):
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    out = {}
    for weights, sd in (('consensus', consensus_sd), ('uniform', seeded_sd)):
        for panc in ((1, 8) if weights == 'consensus' else (1,)):
            cfg = _cfg(panc)
            cfg.weights_dict = sd
            out[weights, panc] = Patch2PixB200(cfg)
    return out


@pytest.fixture(scope='module')
def sds(seeded_sd, consensus_sd):
    return {'consensus': consensus_sd, 'uniform': seeded_sd}


_FEATS, _ORACLE = {}, {}


def _images(case):
    from patch2pix_b200.synth import synthetic_pair_sized
    idx, s1, s2 = CASES[case]
    return synthetic_pair_sized(idx, s1, s2)


def _feats(net, case):
    """fp32 pyramids of both images (each through the backbone on its own) on the GPU and on the host."""
    if case not in _FEATS:
        im1, im2 = _images(case)
        with torch.no_grad():
            f1 = net.extract.forward_all(im1.cuda(), [], early_feat=True)
            f2 = net.extract.forward_all(im2.cuda(), [], early_feat=True)
        assert f1[-1].shape[2:] != f2[-1].shape[2:]
        _FEATS[case] = (f1, f2, [t.cpu() for t in f1], [t.cpu() for t in f2])
    return _FEATS[case]


def _oracle_coarse(case, weights, sd, c1, c2, ksize=2):
    """The oracle's coarse stage (corr4d, delta4d, stages), computed once per case / weights / ksize."""
    from oracle import p2p_oracle as O
    key = (case, weights, ksize)
    if key not in _ORACLE:
        st = {}
        with torch.no_grad():
            o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], sd, ksize=ksize, stages=st)
        _ORACLE[key] = (o_corr, o_delta, st)
    return _ORACLE[key]


# ------------------------------------------------------------------------------------------------
# 1. coarse stages
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['transposed', 'crossed', 'tiles', 'reversed', 'tiny'])
@pytest.mark.parametrize('corr_passes,weights', [(0, 'consensus'), (3, 'consensus'), (3, 'uniform')],
                         ids=['simtcorr', 'tccorr', 'tccorr_uniform'])
def test_coarse_stages_vs_oracle(nets, sds, case, corr_passes, weights):
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    net, sd = nets[weights, 1], sds[weights]
    f1, f2, c1, c2 = _feats(net, case)
    o_corr, o_delta, st = _oracle_coarse(case, weights, sd, c1, c2)
    net.set_option('corr_passes', corr_passes)
    try:
        with torch.no_grad():
            corr4d, delta4d, stages = net.forward_coarse_match(f1[-1], f2[-1], ksize=2, return_stages=True)
            torch.cuda.synchronize()
    finally:
        _restore(net)
    assert corr4d.shape == o_corr.shape and len(delta4d) == 4
    # pooled correlation within 1e-6 of the oracle; an element further off must be nearer the exact (fp64) value than
    # the oracle's own fp32 sum is (both are fp32 dot products of 256 channels, ~1e-6 apart at the worst element)
    pooled = stages['pooled'].cpu()
    p64 = _pooled_fp64(c1[-1], c2[-1])
    err_oracle = (pooled - st['pooled']).abs()
    err_fp64, oracle_fp64 = (pooled.double() - p64).abs(), (st['pooled'].double() - p64).abs()
    far = err_oracle > 1e-6
    assert not (far & (err_fp64 > oracle_fp64)).any(), (err_oracle.max().item(), err_fp64.max().item())
    n_bad, n_unexplained = _delta_mismatch_report(delta4d, o_delta, c1[-1], c2[-1])
    assert n_unexplained == 0 and n_bad <= max(2, delta4d[0].numel() // 500), (n_bad, n_unexplained)
    scale = max(float(st['ncn'].abs().max()), 1e-30)
    np.testing.assert_allclose(stages['ncn'].cpu().numpy(), st['ncn'].numpy(), rtol=2e-4, atol=5e-6 * scale)
    np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=5e-6 * scale)
    with torch.no_grad():
        # proposal kernels on the ORACLE's volume: exact, except that where the reference's own fp32 softmax ties
        # several cells at its maximum, the row may name any one of them
        o_m, o_s = O.cal_coarse_matches(o_corr, o_delta, ksize=2, upsample=8, center=True)
        m2, s2 = net.cal_coarse_matches(o_corr.cuda(), tuple(d.cuda() for d in o_delta), ksize=2, upsample=8)
        assert m2.dtype == torch.int64
        sm_tie, in_tied_set = _softmax_ties(o_corr, m2.cpu())
        sm_diff = (m2.cpu() != o_m).any(-1)[0]
        assert not (sm_diff & ~sm_tie).any() and in_tied_set.all(), (int(sm_diff.sum()), int(sm_tie.sum()))
        np.testing.assert_allclose(s2.cpu().numpy(), o_s.numpy(), rtol=1e-4)
        # filter_coarse on the reference's candidate list
        fm, fs = filter_coarse([o_m[0].cuda()], [o_s[0].cuda()], 0.0, True)
        ofm, ofs = O.filter_coarse(o_m, o_s, 0.0, True)
        assert torch.equal(fm[0].cpu(), ofm[0])
        np.testing.assert_allclose(fs[0].cpu().numpy(), ofs[0].numpy(), rtol=1e-4)
        # our own volume: identical rows except on the reference's fp32 tie rows
        m, _ = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=8, center=True)
        diff = (m.cpu() != o_m).any(-1)[0]
        fragile = _tie_masks(o_corr, c1[-1], c2[-1], 2)
        assert int((diff & ~fragile).sum()) == 0 and int(diff.sum()) <= max(2, diff.numel() // 200), \
            (int(diff.sum()), int((diff & ~fragile).sum()))
    _report(f'coarse_{case}_{weights}_{"tc" if corr_passes else "simt"}',
            {'delta_cells_differing': n_bad, 'unexplained': n_unexplained, 'cells': int(delta4d[0].numel()),
             'pooled_err_vs_oracle': err_oracle.max().item(), 'pooled_err_vs_fp64': err_fp64.max().item(),
             'oracle_pooled_err_vs_fp64': oracle_fp64.max().item(), 'pooled_beyond_1e-6_of_oracle': int(far.sum()),
             'oracle_volume_rows_differing': int(sm_diff.sum()), 'reference_softmax_tie_rows': int(sm_tie.sum()),
             'own_volume_rows_differing': int(diff.sum()), 'reference_tie_rows': int(fragile.sum()),
             'mutual_matches': int(ofm[0].shape[0])})


def _pooled_fp64(feat1, feat2, k=2):
    """The 2^4-max-pooled correlation of the same features in fp64 (what the pooled stage approximates in fp32)."""
    from oracle import p2p_oracle as O
    corr = O.feat_correlation_4d(O.l2_normalize(feat1.double(), 1), O.l2_normalize(feat2.double(), 1))
    return O.maxpool4d(corr, k)[0]


def _softmax_ties(o_corr, m, cell=16):
    """Candidate rows whose softmax (computed as the reference computes it, in fp32) has its maximum at more than one
    cell -- the reference then takes the lowest index, while the kernels take the largest raw correlation: e.g. a row
    whose only non-zero entry is 1e-8 (exp(-1e-8) == 1 in fp32).  Also: does each row of m name a cell of that tied
    maximum (m's cells are pixel // cell for ksize 2, upsample 8)."""
    import torch.nn.functional as F
    _, _, hA, wA, hB, wB = o_corr.shape
    nA, nB = hA * wA, hB * wB
    p1 = F.softmax(o_corr.view(1, nA, hB, wB), dim=1).view(nA, nB)       # rows [0, nB): best A for every B cell
    p2 = F.softmax(o_corr.view(1, hA, wA, nB), dim=3).view(nA, nB)       # rows [nB, nB + nA): best B for every A cell
    mx1, mx2 = p1.max(0)[0], p2.max(1)[0]
    tie = torch.cat([(p1 == mx1).sum(0) > 1, (p2 == mx2[:, None]).sum(1) > 1])
    r = m[0]
    a = (r[:nB, 1] // cell) * wA + r[:nB, 0] // cell
    b = (r[nB:, 3] // cell) * wB + r[nB:, 2] // cell
    in_set = torch.cat([p1[a, torch.arange(nB)] == mx1, p2[torch.arange(nA), b] == mx2])
    return tie, in_set


def test_coarse_ksize1_vs_oracle(nets, sds):
    from oracle import p2p_oracle as O
    net = nets['consensus', 1]
    f1, f2, c1, c2 = _feats(net, 'crossed')
    o_corr, o_delta, _ = _oracle_coarse('crossed', 'consensus', sds['consensus'], c1, c2, ksize=1)
    with torch.no_grad():
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=1)
        assert delta4d is None and o_delta is None and corr4d.shape == o_corr.shape
        np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=5e-6 * float(o_corr.max()))
        o_m, _ = O.cal_coarse_matches(o_corr, None, ksize=1, upsample=8, center=True)
        m2, _ = net.cal_coarse_matches(o_corr.cuda(), None, ksize=1, upsample=8, center=True)
        assert torch.equal(m2.cpu(), o_m)
        m, _ = net.cal_coarse_matches(corr4d, None, ksize=1, upsample=8, center=True)
    diff = (m.cpu() != o_m).any(-1)[0]
    fragile = _tie_masks(o_corr, c1[-1], c2[-1], 1)
    assert int((diff & ~fragile).sum()) == 0 and int(diff.sum()) <= max(2, diff.numel() // 200), int(diff.sum())


def test_nc_layer2_modes_bit_identical(nets):
    """Both NC layer-2 block layouts issue the same MMAs in the same order: bit-identical on an unequal pair."""
    net = nets['consensus', 1]
    f1, f2, _, _ = _feats(net, 'tiles')
    outs = {}
    try:
        for mode in (1, 2):
            net.set_option('nc_l2_mode', mode)
            with torch.no_grad():
                corr4d, delta4d, st = net.forward_coarse_match(f1[-1], f2[-1], ksize=2, return_stages=True)
            torch.cuda.synchronize()
            outs[mode] = (corr4d.cpu(), st['ncn'].cpu(), delta4d.code.cpu())
    finally:
        _restore(net)
    for a, b in zip(outs[1], outs[2]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# 2. channels-last fp16 entries
# ------------------------------------------------------------------------------------------------
def test_fp16_channels_last_entries(nets, sds):
    """Each image's pyramid from the fp16 / channels_last backbone on its own, consumed by p2p_coarse_nhwc16 /
    p2p_refine_prepare_nhwc16; against the oracle and against the NCHW fp32 entries fed the same values."""
    net = nets['consensus', 8]
    im1, im2 = _images('tiles')
    with torch.no_grad():
        f1 = net._forward_all_fast(im1.cuda())
        f2 = net._forward_all_fast(im2.cuda())
        torch.cuda.synchronize()
        assert f1[1].dtype == torch.float16 and f1[-1].shape[2:] != f2[-1].shape[2:]
        u1 = [t.float().contiguous() for t in f1]
        u2 = [t.float().contiguous() for t in f2]
        c1, c2 = [t.cpu() for t in u1], [t.cpu() for t in u2]
        o, g, coarse = _e2e_u(net, sds['consensus'], (f1, f2, c1, c2), 100, 8, 3)
        rep = dict(_e2e_report(o, g), **coarse)
        np.random.seed(3)
        a = net.match_from_feats(f1, f2, 2, ptmax=100, return_all=True)
        np.random.seed(3)
        b = net.match_from_feats(u1, u2, 2, ptmax=100, return_all=True)
        torch.cuda.synchronize()
    assert torch.equal(a[4][0], b[4][0])
    rep['nhwc16_vs_nchw32_entry_max_px'] = (a[0][0] - b[0][0]).abs().max().item()
    _report('fp16_channels_last', rep)
    assert rep['nhwc16_vs_nchw32_entry_max_px'] < 0.05
    _assert_e2e(rep)


# ------------------------------------------------------------------------------------------------
# 3. refine against the oracle
# ------------------------------------------------------------------------------------------------
def _edge_rows(s1, s2):
    """Rows inside one image and outside the other on each axis (both ways round), on each image's own corner, at its
    own far clamp (size + 8) and beyond it, and at the near clamp."""
    (H1, W1), (H2, W2) = s1, s2
    xm, ym = min(W1, W2) + 3.0, min(H1, H2) + 3.0
    xM, yM = max(W1, W2) - 5.0, max(H1, H2) - 5.0
    return torch.tensor([[W1 - 1.0, H1 - 1.0, W2 - 1.0, H2 - 1.0],
                         [xm, 10.0, xm, 10.0], [10.0, ym, 10.0, ym], [xm, ym, xm, ym],
                         [xM, 12.0, xM, 12.0], [12.0, yM, 12.0, yM], [xM, yM, xM, yM],
                         [W1 + 8.0, H1 + 8.0, W2 + 8.0, H2 + 8.0], [W1 + 20.0, H1 + 21.0, W2 + 19.0, H2 + 22.0],
                         [W1 + 8.0, 5.0, 5.0, H2 + 8.0], [5.0, H1 + 8.0, W2 + 8.0, 5.0],
                         [-7.0, -8.0, -9.5, -7.5], [0.0, 0.0, 0.0, 0.0]])


def _random_matches(n, s1, s2, seed, integer):
    """n rows: the edge rows first, then uniform in each image's own range from -5 % to +105 %."""
    (H1, W1), (H2, W2) = s1, s2
    lim = torch.tensor([W1, H1, W2, H2], dtype=torch.float32)
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(n, 4, generator=g) * lim * 1.1 - 0.05 * lim
    e = _edge_rows(s1, s2)[:n]
    m[:e.shape[0]] = e + (0.0 if integer else 0.4)
    return m.long() if integer else m


def _refine_case(net, sd, case, matches, impl, mid_passes, fine_passes, mid_band=0):
    from oracle import p2p_oracle as O
    f1, f2, c1, c2 = _feats(net, case)
    net.set_option('gemm_impl', impl)
    net.set_option('mid_passes', mid_passes)
    net.set_option('fine_passes', fine_passes)
    net.set_option('mid_band', mid_band)
    try:
        with torch.no_grad():
            o_mid, o_midp = O.forward_fine_match(c1, c2, [matches], sd, 'regress_mid.')
            o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, sd, 'regress_fine.')
            mid, midp = net.forward_fine_match(f1, f2, [matches.cuda()], 16, 'center', net.regress_mid)
            fine_same, finep_same = net.forward_fine_match(f1, f2, [o_mid[0].cuda()], 16, 'center', net.regress_fine)
            fine_e2e, finep_e2e = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
            torch.cuda.synchronize()
    finally:
        _restore(net)
    om, of_ = o_mid[0].reshape(-1, 4), o_fine[0].reshape(-1, 4)
    mid_, fs_, fe_ = mid[0].cpu().reshape(-1, 4), fine_same[0].cpu().reshape(-1, 4), fine_e2e[0].cpu().reshape(-1, 4)
    strad = (mid_.long() != om.long()).any(1)
    e2e = (fe_ - of_).abs().max(1)[0]
    pe2e = (finep_e2e[0].cpu().reshape(-1) - o_finep[0].reshape(-1)).abs()
    return {
        'n': int(matches.shape[0]),
        'mid_err': (mid_ - om).abs().max().item(),
        'mid_p_err': (midp[0].cpu().reshape(-1) - o_midp[0].reshape(-1)).abs().max().item(),
        'fine_same_err': (fs_ - of_).abs().max().item(),
        'fine_same_p_err': (finep_same[0].cpu().reshape(-1) - o_finep[0].reshape(-1)).abs().max().item(),
        'straddle_rows': int(strad.sum()),
        'fine_e2e_err_nonstraddle': e2e[~strad].max().item() if (~strad).any() else 0.0,
        'fine_e2e_p_err_nonstraddle': pe2e[~strad].max().item() if (~strad).any() else 0.0,
        'fine_e2e_err': e2e.max().item(), 'fine_e2e_p_err': pe2e.max().item(),
    }


CONFIGS = {'simt33': (1, 3, 3, 0), 'tc33': (0, 3, 3, 0), 'tc31': (0, 3, 1, 0), 'tc11': (0, 1, 1, 0), 'band31': (0, 3, 1, 26)}


def _check_refine(r, mid_passes, fine_passes, band):
    mid_tol = 2e-4 if (mid_passes == 3 and band == 0) else 0.05
    fine_tol = 2e-4 if fine_passes == 3 else 0.05
    assert r['mid_err'] < mid_tol, r
    assert r['fine_same_err'] < fine_tol, r
    assert r['mid_p_err'] < 1e-3 and r['fine_same_p_err'] < 1e-3, r
    assert r['fine_e2e_err_nonstraddle'] < 0.5 and r['fine_e2e_p_err_nonstraddle'] < 1e-3, r
    if mid_passes == 3:      # the shipped configurations: EVERY row within tolerance, no window moved by a pixel
        assert r['straddle_rows'] == 0, r
        assert r['fine_e2e_err'] < 0.5 and r['fine_e2e_p_err'] < 1e-3, r


@pytest.mark.parametrize('case', ['transposed', 'crossed'])
@pytest.mark.parametrize('config', list(CONFIGS))
@pytest.mark.parametrize('integer', [True, False], ids=['int', 'float'])
def test_refine_vs_oracle(nets, sds, case, config, integer):
    impl, mp, fp, band = CONFIGS[config]
    _, s1, s2 = CASES[case]
    r = _refine_case(nets['consensus', 1], sds['consensus'], case, _random_matches(129, s1, s2, 3, integer),
                     impl, mp, fp, band)
    _report(f'refine_{case}_{config}_{"i" if integer else "f"}', r)
    _check_refine(r, mp, fp, band)


@pytest.mark.parametrize('n', [1, 1201])
@pytest.mark.parametrize('config,integer', [('tc31', True), ('band31', False), ('tc33', False)])
def test_refine_row_counts(nets, sds, n, config, integer):
    impl, mp, fp, band = CONFIGS[config]
    _, s1, s2 = CASES['crossed']
    r = _refine_case(nets['consensus', 1], sds['consensus'], 'crossed', _random_matches(n, s1, s2, n, integer),
                     impl, mp, fp, band)
    _report(f'refine_rows{n}_{config}_{"i" if integer else "f"}', r)
    _check_refine(r, mp, fp, band)


# ------------------------------------------------------------------------------------------------
# 4. paths that must agree bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['crossed', 'tiles'])
def test_fused_gather_generations(nets, case):
    """conv1 A operand through the window maps (fuse_gather 3), the fused gathers (1, 2) and the materialised patch
    tensor (0), 1-pass mid: 3 == 1 == 2 bit for bit, 0 within one fp16 rounding of the features."""
    net = nets['consensus', 1]
    _, s1, s2 = CASES[case]
    m = _random_matches(333, s1, s2, 11, False)
    f1, f2, _, _ = _feats(net, case)
    out = {}
    try:
        for fuse in (1, 2, 3, 0):
            net.set_option('fuse_gather', fuse)
            net.set_option('mid_band', 0)
            net.set_option('mid_passes', 1)
            with torch.no_grad():
                mid, midp = net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', net.regress_mid)
                fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
            torch.cuda.synchronize()
            out[fuse] = (mid[0].cpu(), midp[0].cpu(), fine[0].cpu(), finep[0].cpu())
    finally:
        _restore(net)
    rep = {}
    for fuse in (1, 2):
        same = (out[fuse][0].long() == out[0][0].long()).all(1)
        rep[f'gen{fuse}'] = {'mid_diff_px': (out[fuse][0] - out[0][0]).abs().max().item(),
                             'mid_conf_diff': (out[fuse][1] - out[0][1]).abs().max().item(),
                             'fine_diff_px_same_window': (out[fuse][2] - out[0][2]).abs().max(1)[0][same].max().item(),
                             'fine_conf_diff_same_window': (out[fuse][3] - out[0][3]).abs()[same].max().item(),
                             'rows_with_other_window': int((~same).sum())}
    _report(f'fused_gather_{case}', rep)
    for fuse in (1, 2):
        r = rep[f'gen{fuse}']
        assert r['mid_diff_px'] < 0.03 and r['mid_conf_diff'] < 5e-4, (fuse, rep)
        assert r['fine_diff_px_same_window'] < 0.05 and r['fine_conf_diff_same_window'] < 1e-3, (fuse, rep)
    for i in range(4):
        assert torch.equal(out[1][i], out[2][i]), ('fuse_gather 1 vs 2', i)
        assert torch.equal(out[3][i], out[1][i]), ('fuse_gather 3 vs 1', i, (out[3][i] - out[1][i]).abs().max().item())


def test_fc_tensor_core_vs_cuda_core(nets):
    net = nets['consensus', 1]
    _, s1, s2 = CASES['crossed']
    m = _random_matches(300, s1, s2, 5, True)
    f1, f2, _, _ = _feats(net, 'crossed')
    out = {}
    try:
        net.set_option('mid_band', 0)
        for impl in (1, 0):
            net.set_option('fc_impl', impl)
            with torch.no_grad():
                mid, midp = net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', net.regress_mid)
            torch.cuda.synchronize()
            out[impl] = (mid[0].cpu(), midp[0].cpu())
    finally:
        _restore(net)
    d = (out[1][0] - out[0][0]).abs().max().item()
    dp = (out[1][1] - out[0][1]).abs().max().item()
    _report('fc_tc_vs_simt', {'mid_diff_px': d, 'conf_diff': dp})
    assert d < 1e-4 and dp < 1e-5, (d, dp)


# ------------------------------------------------------------------------------------------------
# 5. window sharing
# ------------------------------------------------------------------------------------------------
SHIFTS = ((-8, -8), (8, -8), (-8, 8), (8, 8))


def _origins(m, s1, s2):
    """Window origins as the kernels compute them: trunc, then clamp each image's to [-7, its own size + 8]."""
    (H1, W1), (H2, W2) = s1, s2
    t = m.long() if m.is_floating_point() else m.clone()
    lim = torch.tensor([W1, H1, W2, H2])
    return torch.minimum(torch.maximum(t, torch.full_like(t, -7)), lim + 8)


def _shared_mask(m, s1, s2):
    """Per row: does it belong to a half-group with equal origins on the shared image (rows 0-3 share image 2's
    window, rows 4-7 image 1's)."""
    o = _origins(m, s1, s2)
    n = m.shape[0]
    mask = torch.zeros(n, dtype=torch.bool)
    for g in range(n // 8):
        a = o[8 * g:8 * g + 4, 2:]
        b = o[8 * g + 4:8 * g + 8, :2]
        mask[8 * g:8 * g + 4] = bool((a == a[0]).all())
        mask[8 * g + 4:8 * g + 8] = bool((b == b[0]).all())
    return mask


def _mixed_matches(s1, s2, n_groups=64):
    """shift_to_anchors-style groups (rows 0-3 move point 1 by (+-8, +-8), rows 4-7 point 2) over each image's own
    range, some half-groups broken by a pixel, and clamped windows at one image's far border that are not clamped at
    the other's: rows 0-3 on image 2 along the axis where image 2 is the smaller, rows 4-7 on image 1 along the axis
    where image 1 is the smaller (a limit taken from the wrong image leaves those windows distinct)."""
    (H1, W1), (H2, W2) = s1, s2
    g = torch.Generator().manual_seed(17)
    base = (torch.rand(n_groups, 4, generator=g) * torch.tensor([W1, H1, W2, H2], dtype=torch.float32)).floor()
    rows = []
    for k in range(n_groups):
        for h in range(2):
            for dx, dy in SHIFTS:
                r = base[k].clone()
                r[2 * h] += dx
                r[2 * h + 1] += dy
                rows.append(r)
    m = torch.stack(rows) + torch.rand(8 * n_groups, 4, generator=g) * 0.9
    for k in range(0, n_groups, 7):                 # break half-group A
        m[8 * k + 1 + k % 3, 2 + k % 2] += 1.0
    for k in range(3, n_groups, 11):                # break half-group B
        m[8 * k + 4 + k % 4, k % 2] -= 1.0
    far = torch.tensor([8.5, 9.9, 8.0, 9.25])
    ax2 = 3 if H2 < H1 else 2                       # image 2's smaller axis (y if H2 < H1, else x)
    ax1 = 0 if W1 < W2 else 1                       # image 1's smaller axis
    lim = [W1, H1, W2, H2]
    for k in range(5, n_groups, 6):
        m[8 * k:8 * k + 4, ax2] = lim[ax2] + far
        m[8 * k + 4:8 * k + 8, ax1] = lim[ax1] + far
    for k in range(2, n_groups, 9):                 # the near clamp
        m[8 * k:8 * k + 4, 2] = torch.tensor([-7.9, -9.0, -8.5, -7.0])
        m[8 * k + 4:8 * k + 8, 1] = torch.tensor([-7.5, -12.0, -8.0, -7.0])
    extra = torch.tensor([[3.5, 4.5, 100.2, 60.7], [3.5, 4.5, 100.2, 60.7], [W1 - 1.0, H1 - 1.0, W2 - 1.0, H2 - 1.0]])
    return torch.cat([m, extra])                    # partial last group


def _run_share(net, f1, f2, m, share, which='mid', mid_passes=3, mid_band=26):
    net.set_option('share_windows', share)
    net.set_option('mid_passes', mid_passes)
    net.set_option('mid_band', mid_band)
    try:
        with torch.no_grad():
            reg = net.regress_mid if which == 'mid' else net.regress_fine
            c, p = net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', reg)
        torch.cuda.synchronize()
        shared = net._handle.get_option('shared_rows')
    finally:
        _restore(net)
    return c[0].cpu(), p[0].cpu().reshape(-1), shared


@pytest.mark.parametrize('case', ['crossed', 'transposed'])
def test_window_sharing(nets, sds, case):
    from oracle import p2p_oracle as O
    net = nets['consensus', 8]
    _, s1, s2 = CASES[case]
    f1, f2, c1, c2 = _feats(net, case)
    m = _mixed_matches(s1, s2)
    rep = {}
    for integer in (False, True):
        mm = m.floor().long() if integer else m
        mask = _shared_mask(mm, s1, s2)
        assert 0 < int(mask.sum()) < mm.shape[0] - 3
        # 1-pass mid: unshared rows bit-identical to share_windows 0, shared ones within one reordering of the sum
        mid0, mp0, s0 = _run_share(net, f1, f2, mm, 0, mid_passes=1, mid_band=0)
        mid1, mp1, s1_ = _run_share(net, f1, f2, mm, 1, mid_passes=1, mid_band=0)
        assert s0 == 0 and s1_ == int(mask.sum()), (s1_, int(mask.sum()))
        assert torch.equal(mid1[~mask], mid0[~mask]) and torch.equal(mp1[~mask], mp0[~mask])
        assert (mid1 - mid0).abs().max().item() < 0.03 and (mp1 - mp0).abs().max().item() < 5e-4
        # the shipped configuration (risk band) with sharing, mid and fine against the ORACLE on every row
        mid, midp, sh = _run_share(net, f1, f2, mm, 1)
        assert sh == int(mask.sum())
        fine, finep, _ = _run_share(net, f1, f2, mid, 1, 'fine')
        with torch.no_grad():
            o_mid, o_midp = O.forward_fine_match(c1, c2, [mm], sds['consensus'], 'regress_mid.')
            o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, sds['consensus'], 'regress_fine.')
        strad = int((mid.long() != o_mid[0].long()).any(1).sum())
        r = {'shared_rows': sh, 'rows': int(mm.shape[0]), 'straddle_rows': strad,
             'mid_err': (mid - o_mid[0]).abs().max().item(), 'mid_p_err': (midp - o_midp[0]).abs().max().item(),
             'max_err_px': (fine - o_fine[0]).abs().max().item(), 'max_conf_err': (finep - o_finep[0]).abs().max().item()}
        rep['int' if integer else 'float'] = r
        assert strad == 0 and r['mid_err'] < 0.05 and r['mid_p_err'] < 1e-3, r
        assert r['max_err_px'] < 0.5 and r['max_conf_err'] < 1e-3, r
    _report(f'share_{case}', rep)


# ------------------------------------------------------------------------------------------------
# 6. end to end
# ------------------------------------------------------------------------------------------------
def _e2e_u(net, sd, feats, ptmax, panc, np_seed, case=None, weights='consensus'):
    """test_gpu_parity._e2e on an unequal pair, with the oracle's coarse stage shared between configurations."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    f1, f2, c1, c2 = feats
    with torch.no_grad():
        if case is not None:
            o_corr, o_delta, _ = _oracle_coarse(case, weights, sd, c1, c2)
        else:
            o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], sd, 2)
        o_m, o_s = O.cal_coarse_matches(o_corr, o_delta, 2, upsample=O.UPSAMPLE, center=True)
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=2)
        m, s = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
        diff = (m.cpu() != o_m).any(-1)[0]
        fragile = _tie_masks(o_corr, c1[-1], c2[-1], 2)
        coarse = {'candidate_rows': int(diff.numel()), 'rows_differing': int(diff.sum()),
                  'rows_differing_unexplained': int((diff & ~fragile).sum()), 'reference_tie_rows': int(fragile.sum())}
        assert coarse['rows_differing_unexplained'] == 0, coarse
        assert coarse['rows_differing'] <= max(2, diff.numel() // 200), coarse
        np.testing.assert_allclose(s.cpu().numpy()[0][~diff.numpy()], o_s.numpy()[0][~diff.numpy()], rtol=1e-3)
        np.random.seed(np_seed)
        if ptmax:
            o_cm, _ = O.filter_coarse(o_m, o_s, 0.0, True, ptmax=ptmax)
        else:
            o_cm, _ = O.filter_coarse(o_m, o_s, 0.0, True)
        o_cm = O.shift_to_anchors(o_cm, panc)
        o_mid, o_midp = O.forward_fine_match(c1, c2, o_cm, sd, 'regress_mid.')
        o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, sd, 'regress_fine.')
        np.random.seed(np_seed)
        cm, _ = filter_coarse([o_m[0].cuda()], [o_s[0].cuda()], 0.0, True, ptmax=ptmax if ptmax else None)
        cm = net.shift_to_anchors(cm)
        mid, midp = net.forward_fine_match(f1, f2, cm, 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
        torch.cuda.synchronize()
        # the fused production entry reproduces the staged path bit for bit; where our candidate list differs from the
        # reference's (on its fp32 tie rows), the staged path is re-run from our own candidates for that comparison
        own_cm, own_fine, own_finep = cm, fine, finep
        if coarse['rows_differing'] != 0:
            np.random.seed(np_seed)
            own_cm, _ = filter_coarse([m[0]], [s[0]], 0.0, True, ptmax=ptmax if ptmax else None)
            own_cm = net.shift_to_anchors(own_cm)
            own_mid, _ = net.forward_fine_match(f1, f2, own_cm, 16, 'center', net.regress_mid)
            own_fine, own_finep = net.forward_fine_match(f1, f2, own_mid, 16, 'center', net.regress_fine)
        np.random.seed(np_seed)
        g = net.match_from_feats(f1, f2, 2, 0.0, True, ptmax, return_all=True)
        torch.cuda.synchronize()
        assert torch.equal(g[4][0], own_cm[0]), 'fused entry: anchors differ from the staged path'
        assert torch.equal(g[0][0].reshape(-1, 4), own_fine[0].reshape(-1, 4)), 'fused entry differs from the staged path'
        assert torch.equal(g[1][0].reshape(-1), own_finep[0].reshape(-1))
    return (o_fine, o_finep, o_mid, o_midp, o_cm), (fine, finep, mid, midp, cm), coarse


@pytest.mark.parametrize('case,ptmax', [('crossed', None), ('crossed', 50), ('tiles', None), ('tiles', 100),
                                        ('bench', None), ('bench', 400)])
def test_end_to_end_vs_oracle(nets, sds, case, ptmax):
    panc = 8 if ptmax else 1
    net = nets['consensus', panc]
    feats = _feats(net, case)
    o, g, coarse = _e2e_u(net, sds['consensus'], feats, ptmax, panc, 11, case)
    rep = dict(_e2e_report(o, g), **coarse)
    _report(f'e2e_{case}_pt{ptmax}_pa{panc}', rep)
    _assert_e2e(rep)
    assert rep['n'] >= (0.9 * ptmax * panc if ptmax else 30), rep


# ------------------------------------------------------------------------------------------------
# 7. golden vectors of the live reference
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['unequal_96x128_128x96', 'unequal_128x160_96x224'])
def test_golden_reference_vectors(nets, name):
    from patch2pix_b200.synth import synthetic_pair_sized
    g = np.load(os.path.join(GOLD, name + '.npz'))
    net = nets['consensus', 1]
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    with torch.no_grad():
        fine, finep, mid, midp, coarse = net.predict_fine(im1.cuda(), im2.cuda(), ksize=2, return_all=True)
        corr4d, delta4d = net.forward(im1.cuda(), im2.cuda(), ksize=2)
    np.testing.assert_allclose(corr4d.cpu().numpy(), g['corr4d'], rtol=2e-3, atol=1e-6)
    differ = (torch.stack([d.cpu() for d in delta4d]).numpy().astype(np.int8) != g['delta']).any(0)
    assert not (differ & ~g['delta_fp32_tie']).any(), int(differ.sum())      # the fixtures hold no such ties today
    assert np.array_equal(coarse[0].cpu().numpy(), g['coarse'])
    assert np.abs(fine[0].cpu().numpy().reshape(-1, 4) - g['fine']).max() < 0.5
    assert np.abs(finep[0].cpu().numpy().reshape(-1) - g['fine_p']).max() < 1e-3


def test_golden_train_sequence(nets):
    from patch2pix_b200.model import filter_coarse
    from patch2pix_b200.synth import synthetic_pair_sized
    g = np.load(os.path.join(GOLD, 'unequal_trainseq_160x240_192x128.npz'))
    net = nets['consensus', 8]
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    with torch.no_grad():
        f1, f2 = net.extract_pair(im1.cuda(), im2.cuda())
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=2)
        cand, _ = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
        diff = (cand[0].cpu().numpy() != g['cand_matches'][0]).any(-1)
        assert not (diff & ~g['cand_fp32_tie']).any() and diff.sum() <= 4, int(diff.sum())
        np.random.seed(int(g['np_seed']))
        cm, _ = filter_coarse([torch.from_numpy(g['cand_matches'][0]).cuda()], [torch.from_numpy(g['cand_scores'][0]).cuda()],
                              0.0, True, ptmax=int(g['ptmax']))
        anchors = net.shift_to_anchors(cm)
        mid, midp = net.forward_fine_match(f1, f2, anchors, 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
        if diff.sum() == 0:
            np.random.seed(int(g['np_seed']))
            g2 = net.match_from_feats(f1, f2, 2, ptmax=int(g['ptmax']), return_all=True)
            assert torch.equal(g2[4][0], anchors[0]) and torch.equal(g2[0][0], fine[0])
    assert np.array_equal(anchors[0].cpu().numpy(), g['anchors'])
    assert np.abs(mid[0].cpu().numpy() - g['mid']).max() < 1e-2
    assert np.array_equal(np.trunc(mid[0].cpu().numpy()), np.trunc(g['mid']))
    assert np.abs(fine[0].cpu().numpy() - g['fine']).max() < 0.5
    assert np.abs(finep[0].cpu().numpy() - g['fine_p']).max() < 1e-3


# ------------------------------------------------------------------------------------------------
# 8. host glue
# ------------------------------------------------------------------------------------------------
def test_predict_fine_with_backbone_graphs_for_another_shape(nets, consensus_sd):
    """extract_pair's unequal branch: backbone graphs captured at image 1's shape must not be replayed for the pair."""
    from patch2pix_b200.model import Patch2PixB200
    cfg = _cfg(1)
    cfg.weights_dict = consensus_sd
    net = Patch2PixB200(cfg)
    im1, im2 = _images('transposed')
    with torch.no_grad():
        net.enable_backbone_graphs(im1.shape[2], im1.shape[3], instances=1)
        f1, f2 = net.extract_pair(im1.cuda(), im2.cuda())
        assert getattr(f1, 'graph_inst', None) is None and f1[-1].shape[2:] != f2[-1].shape[2:]
        a = net.predict_fine(im1.cuda(), im2.cuda(), ksize=2, return_all=True)
        b = nets['consensus', 1].predict_fine(im1.cuda(), im2.cuda(), ksize=2, return_all=True)
        torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x[0], y[0])
    assert a[4][0].shape[0] > 0


def test_estimate_matches_from_files_unequal(tmp_path, consensus_sd):
    """A portrait and a landscape PNG of different original sizes at imsize 320: the two images' (sx, sy) differ from
    each other and within each image."""
    pytest.importorskip('PIL')
    from PIL import Image
    from oracle import preprocess_oracle as PO
    from patch2pix_b200.eval_helper import estimate_matches, estimate_matches_from_files, load_model
    from patch2pix_b200.synth import synthetic_pair_sized
    net = load_model(consensus_sd)
    im1, im2 = synthetic_pair_sized(4, (410, 290), (300, 420))
    paths = []
    for i, im in enumerate((im1, im2)):
        u8 = ((im[0].permute(1, 2, 0) * 0.25 + 0.5).clamp(0, 1) * 255).byte().numpy()
        paths.append(str(tmp_path / f'im{i}.png'))
        Image.fromarray(u8).save(paths[-1])
    m, s, c = estimate_matches_from_files(net, paths[0], paths[1], io_thres=0.3, imsize=320)
    ts, scs = [], []
    for pth in paths:
        t, sc = PO.load_im_flexible_array(np.asarray(Image.open(pth).convert('RGB')), 2, net.upsample, 320)
        ts.append(torch.from_numpy(t).unsqueeze(0))
        scs.append(tuple(sc))
    assert ts[0].shape != ts[1].shape
    assert scs[0] != scs[1] and scs[0][0] != scs[0][1] and scs[1][0] != scs[1][1], scs
    m2, s2, c2 = estimate_matches(net, ts[0], ts[1], scs[0], scs[1], io_thres=0.3)
    assert np.array_equal(m, m2) and np.array_equal(s, s2) and np.array_equal(c, c2)
    with torch.no_grad():
        fine, fs, cm = net.predict_fine(ts[0].cuda(), ts[1].cuda(), ksize=2)
    fine, fs, cm = fine[0].cpu().numpy().reshape(-1, 4), fs[0].cpu().numpy().reshape(-1), cm[0].cpu().numpy()
    up = np.array([scs[0] + scs[1]])
    pos = np.where(fs > 0.3)[0]
    if len(pos) > 0:
        fine, fs, cm = fine[pos], fs[pos], cm[pos]
    assert np.array_equal(m, up * fine) and np.array_equal(s, fs) and np.array_equal(c, up * cm)
    assert len(m) > 0
    _report('estimate_from_files', {'matches': int(len(m)), 'scale1': list(scs[0]), 'scale2': list(scs[1])})


def test_eval_pairs_unequal_views(tmp_path):
    """eval_pairs on a validation scene whose pairs are views of different sizes, against the host flow of
    test_eval_end_to_end_matches_host run with each image's own K."""
    from PIL import Image
    from patch2pix_b200 import evaluation as E
    from patch2pix_b200 import pose as P
    from patch2pix_b200.eval_helper import estimate_matches_from_files, load_model
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_val_scene
    from test_gpu_eval import KW, _hist, _near_edge, _np_sampson, _pairs
    net = load_model(make_seeded_state_dict(0, nc_init='consensus'))
    root = str(tmp_path / 'val')
    synthetic_val_scene(root, 'sceneU', 3, [((320, 240), (240, 320)), ((288, 224), (256, 192)),
                                            ((320, 256), (224, 288))])
    pairs = _pairs(root, 10)
    assert len(pairs) == 3
    recs = E.eval_pairs(net, pairs, eval_type='fine', **KW)
    n_ok = 0
    for (p1, p2, im1, im2), r in zip(pairs, recs):
        assert Image.open(p1).size != Image.open(p2).size and not np.array_equal(im1.K, im2.K)
        t_gt, q_gt = P.abs2relapose(im1.c, im2.c, im1.q, im2.q)
        F = P.pose2fund(im1.K, im2.K, P.quat2mat(q_gt), t_gt)
        m, _, c, inl, Em, R, t = estimate_matches_from_files(net, p1, p2, KW['ksize'], KW['ncn_thres'], True,
                                                             KW['io_thres'], 'fine', KW['imsize'],
                                                             verify=('E', KW['rthres'], im1.K, im2.K))
        cdist, fdist = _np_sampson(np.asarray(c), F), _np_sampson(np.asarray(m), F)
        assert r.N == len(m) and len(m) > 0
        for k, d in ((0, cdist), (1, fdist)) + (((2, fdist[inl]),) if r.status == 'ok' else ()):
            exp = _hist(d, E.EVAL_BINS)
            assert r.counts[k, -1] == exp[-1]
            assert np.abs(r.counts[k, :-1] - exp[:-1]).sum() <= 2 * _near_edge(d, E.EVAL_BINS).sum(), (k, r.counts[k])
        if Em is None:
            assert r.status == 'geo_failed'
            continue
        assert r.status == 'ok' and r.n_inls == inl.sum()
        assert np.array_equal(r.R, R) and np.array_equal(r.t, t)
        terr = P.cal_vec_angle_error(t.squeeze(), t_gt)
        qerr = P.cal_quat_angle_error(P.mat2quat(R), q_gt)
        assert abs(r.terr - terr) <= 1e-9 and abs(r.qerr - qerr) <= 1e-9
        n_ok += 1
    assert n_ok >= 1
