"""GPU parity tests: the CUDA path (through the C ABI, via patch2pix_b200.model) against the CPU
oracle on identical seeded inputs, against the committed golden vectors of the live reference,
and -- at the benchmark size -- through size-independent properties.

Tolerances (BASELINE.json north_star): proposal rows bit-exact (int64, incl. order), refined
coordinates within 0.5 px, confidences within 1e-3.  The per-stage checks below are much tighter
than that wherever the arithmetic is fp32-grade.
"""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
OUT = os.path.join(os.path.dirname(os.path.dirname(__file__)), 'gpurun_out')


def _cfg(panc=1, regress=True):
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=panc, shared=False) if regress else None
    return Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                     weights_dict=None, change_stride=True, regressor_config=rc)


@pytest.fixture(scope='module')
def nets(seeded_sd):
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {}
    for panc in (1, 8):
        cfg = _cfg(panc)
        cfg.weights_dict = seeded_sd
        out[panc] = Patch2PixB200(cfg)
    return out


@pytest.fixture(scope='module')
def cnets(consensus_sd):
    """Benchmark-workload weights (trained-like NC filters): hundreds of distinct mutual matches per pair."""
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {}
    for panc in (1, 8):
        cfg = _cfg(panc)
        cfg.weights_dict = consensus_sd
        out[panc] = Patch2PixB200(cfg)
    return out


def _feats(net, pair_idx, H, W, shifted=False):
    from patch2pix_b200.synth import synthetic_pair, synthetic_pair_shifted
    im1, im2 = (synthetic_pair_shifted if shifted else synthetic_pair)(pair_idx, H, W)
    with torch.no_grad():
        f1 = net.extract.forward_all(im1.cuda(), [], early_feat=True)
        f2 = net.extract.forward_all(im2.cuda(), [], early_feat=True)
    return f1, f2, [t.cpu() for t in f1], [t.cpu() for t in f2]


def _report(name, payload):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, f'parity_{name}.json'), 'w') as f:
        json.dump(payload, f, indent=1)


# ------------------------------------------------------------------------------------------------
# tensor-core GEMM unit test + accumulation-accuracy probe
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,N,K', [(128, 256, 64), (200, 300, 256), (256, 512, 4672), (1000, 512, 1024)])
def test_umma_gemm_matches_fp64(M, N, K):
    """Tensor-core GEMM vs fp64.  Errors are normalised by mean |C|.  Expected levels: 1-pass ~3e-4 mean (fp16
    operand rounding); 3-pass with whole-K tensor-core accumulation drifts with K because the tensor core truncates
    (RZ) on every accumulate; 3-pass with short RN-accumulated segments is fp32-grade."""
    from patch2pix_b200 import _lib
    h = _lib.default_handle('cuda:0')
    g = torch.Generator().manual_seed(M * 7 + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g)
    ref = (a.double() @ b.double().t())
    scale = ref.abs().mean().item()
    ad, bd = a.cuda(), b.cuda()
    ref32 = (ad @ bd.t()).cpu().double()
    res = {'cublas_fp32': {'max': (ref32 - ref).abs().max().item() / scale, 'mean': (ref32 - ref).abs().mean().item() / scale}}
    limits = {(1, 0): (1e-3, 6e-3), (1, 2): (1e-3, 6e-3), (3, 0): (3e-7 + 4e-9 * K, 2e-5 + 3e-8 * K),
              (3, 1): (4e-7, 2e-5), (3, 4): (1.5e-6, 3e-5)}
    for (passes, seg), (mean_tol, max_tol) in limits.items():
        c = torch.full((M, N), float('nan'), device='cuda')
        _lib.check(h.lib.p2p_test_gemm(h.h, _lib.ptr(ad), _lib.ptr(bd), _lib.ptr(c), M, N, K, passes, seg, 64.0,
                                       h.stream()))
        torch.cuda.synchronize()
        err = (c.cpu().double() - ref).abs()
        res[f'p{passes}_s{seg}'] = {'max': err.max().item() / scale, 'mean': err.mean().item() / scale,
                                    'bias': ((c.cpu().double() - ref) * ref.sign()).mean().item() / scale}
        assert torch.isfinite(c).all()
        assert err.mean().item() / scale < mean_tol and err.max().item() / scale < max_tol, (passes, seg, res)
    _report(f'gemm_{M}x{N}x{K}', res)


def test_umma_gemm_positive_accumulation_drift():
    """All-positive operands expose accumulator rounding (RZ vs RN) as a systematic bias."""
    from patch2pix_b200 import _lib
    h = _lib.default_handle('cuda:0')
    M, N, K = 256, 256, 4608
    g = torch.Generator().manual_seed(5)
    a = torch.rand(M, K, generator=g) + 0.5
    b = torch.rand(N, K, generator=g) + 0.5
    ref = a.double() @ b.double().t()
    ref32 = (a.cuda() @ b.cuda().t()).cpu().double()
    ad, bd = a.cuda(), b.cuda()
    res = {'fp32_cublas_rel_bias': ((ref32 - ref) / ref).mean().item()}
    for passes, seg in ((3, 0), (3, 1), (3, 3), (3, 9)):
        c = torch.empty(M, N, device='cuda')
        _lib.check(h.lib.p2p_test_gemm(h.h, _lib.ptr(ad), _lib.ptr(bd), _lib.ptr(c), M, N, K, passes, seg, 64.0,
                                       h.stream()))
        rel = (c.cpu().double() - ref) / ref
        res[f'p{passes}_s{seg}'] = {'rel_bias': rel.mean().item(), 'rel_absmax': rel.abs().max().item()}
    _report('gemm_drift', res)
    assert abs(res['p3_s1']['rel_bias']) < 2e-6


# ------------------------------------------------------------------------------------------------
# coarse stage
# ------------------------------------------------------------------------------------------------
def _delta_mismatch_report(delta4d, o_delta, c1, c2, tie_eps=1e-6):
    """Cells where our pooling argmax differs from the oracle's are legitimate only where the
    oracle's own top-2 gap inside the 2^4 window is within fp32 rounding noise of a tie."""
    from oracle import p2p_oracle as O
    ours = torch.stack([d.cpu() for d in delta4d])
    ref = torch.stack(list(o_delta))
    bad = (ours != ref).any(0)
    if not bad.any():
        return 0, 0
    corr = O.feat_correlation_4d(O.l2_normalize(c1, 1), O.l2_normalize(c2, 1))
    sl = torch.cat([corr[:, :, i::2, j::2, k::2, l::2] for i in range(2) for j in range(2) for k in range(2) for l in range(2)], 1)
    top2 = sl.topk(2, dim=1)[0]
    gap = (top2[:, 0] - top2[:, 1]).unsqueeze(1)
    unexplained = bad & (gap > tie_eps)
    return int(bad.sum()), int(unexplained.sum())


@pytest.mark.parametrize('pair_idx,H,W', [(3, 96, 128), (5, 128, 96), (11, 160, 240)])
@pytest.mark.parametrize('corr_passes', [0, 3], ids=['simtcorr', 'tccorr'])
def test_coarse_stages_vs_oracle(nets, seeded_sd, pair_idx, H, W, corr_passes):
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    net = nets[1]
    net.set_option('corr_passes', corr_passes)
    try:
        f1, f2, c1, c2 = _feats(net, pair_idx, H, W)
        with torch.no_grad():
            st = {}
            o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], seeded_sd, ksize=2, stages=st)
            corr4d, delta4d, stages = net.forward_coarse_match(f1[-1], f2[-1], ksize=2, return_stages=True)
            torch.cuda.synchronize()
            assert corr4d.shape == o_corr.shape and len(delta4d) == 4 and delta4d[0].dtype == torch.int64
            np.testing.assert_allclose(stages['pooled'].cpu().numpy(), st['pooled'].numpy(), rtol=0, atol=1e-6)
            n_bad, n_unexplained = _delta_mismatch_report(delta4d, o_delta, c1[-1], c2[-1])
            assert n_unexplained == 0 and n_bad <= max(2, delta4d[0].numel() // 500), (n_bad, n_unexplained)
            np.testing.assert_allclose(stages['ncn'].cpu().numpy(), st['ncn'].numpy(), rtol=2e-4, atol=5e-6)
            np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=1e-7)
            # proposal kernels on reference-shaped inputs from outside (the ORACLE's corr4d/delta): exact
            o_m, o_s = O.cal_coarse_matches(o_corr, o_delta, ksize=2, upsample=8, center=True)
            m2, s2 = net.cal_coarse_matches(o_corr.cuda(), tuple(d.cuda() for d in o_delta), ksize=2, upsample=8)
            assert m2.dtype == torch.int64 and torch.equal(m2.cpu(), o_m)
            np.testing.assert_allclose(s2.cpu().numpy(), o_s.numpy(), rtol=1e-4)
            fm, fs = filter_coarse(m2, s2, 0.0, True)
            ofm, ofs = O.filter_coarse(o_m, o_s, 0.0, True)
            assert torch.equal(fm[0].cpu(), ofm[0])
            np.testing.assert_allclose(fs[0].cpu().numpy(), ofs[0].numpy(), rtol=1e-4)
            # our own corr4d/delta: identical rows except where a pooling-window tie was broken differently
            m, s = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
            diff_rows = int((m.cpu() != o_m).any(-1).sum())
            assert diff_rows <= 2 * n_bad, (diff_rows, n_bad)
            _report(f'coarse_{H}x{W}_{"tc" if corr_passes else "simt"}', {'delta_cells_differing': n_bad,
                    'unexplained': n_unexplained, 'proposal_rows_differing': diff_rows, 'cells': int(delta4d[0].numel())})
    finally:
        net.set_option('corr_passes', 3)


def test_coarse_ksize1_vs_oracle(nets, seeded_sd):
    from oracle import p2p_oracle as O
    net = nets[1]
    f1, f2, c1, c2 = _feats(net, 2, 64, 96)
    with torch.no_grad():
        o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], seeded_sd, ksize=1)
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=1)
        assert delta4d is None and o_delta is None
        np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=1e-7)
        o_m, o_s = O.cal_coarse_matches(o_corr, None, ksize=1, upsample=8, center=True)
        m, s = net.cal_coarse_matches(corr4d, None, ksize=1, upsample=8, center=True)
        assert torch.equal(m.cpu(), o_m)


@pytest.mark.parametrize('weights', ['uniform', 'consensus'])
def test_neigh_consensus_tensor_core_vs_oracle(nets, cnets, seeded_sd, consensus_sd, weights):
    """NeighConsensus on the tensor cores (fp16 hi/lo 3-pass, partial-map formulation, nc_umma.cu) against the oracle
    (conv3d loop of the reference) and against the fp32 CUDA-core kernels, on odd shapes, inputs of very different
    magnitude (device-side power-of-two scaling) and an all-zero input."""
    from oracle import p2p_oracle as O
    from patch2pix_b200 import _lib
    net, sd = (cnets[1], consensus_sd) if weights == 'consensus' else (nets[1], seeded_sd)
    h = net._ready()
    rep = {}
    for (hA, wA, hB, wB), amp in (((3, 4, 5, 6), 1.0), ((6, 5, 9, 11), 1e-3), ((8, 10, 8, 10), 37.0), ((15, 20, 15, 20), 1.0),
                                  ((2, 3, 17, 40), 1.0), ((4, 4, 4, 4), 0.0)):
        g = torch.Generator().manual_seed(hA * 100 + wB)
        x = (torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1) * amp
        ref = O.neigh_consensus(x, sd)
        xd = x.cuda()
        outs = {}
        for impl in (1, 0):
            net.set_option('nc_impl', impl)
            out = torch.full_like(xd, float('nan'))
            _lib.check(h.lib.p2p_neigh_consensus(h.h, _lib.ptr(xd), hA, wA, hB, wB, _lib.ptr(out), h.stream()))
            torch.cuda.synchronize()
            outs[impl] = out.cpu()
        net.set_option('nc_impl', 1)
        scale = max(ref.abs().max().item(), 1e-30)
        rep[f'{hA}x{wA}x{hB}x{wB}_amp{amp}'] = {'tc_vs_oracle': (outs[1] - ref).abs().max().item() / scale,
                                                'simt_vs_oracle': (outs[0] - ref).abs().max().item() / scale}
        assert torch.isfinite(outs[1]).all()
        np.testing.assert_allclose(outs[1].numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * scale)
        np.testing.assert_allclose(outs[0].numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * scale)
    _report(f'nc_tensor_core_{weights}', rep)


@pytest.mark.parametrize('mode', [1, 2])
def test_neigh_consensus_layer2_block_layouts(cnets, consensus_sd, mode):
    """NC layer 2 reads its A operand as SHIFTED windows of one block of hidden lines (nc_umma.cu): mode 1 = one
    haloed block per tile, mode 2 = one block per column tap; tap starts are 128-byte granular in both.
    Both layouts against the oracle on shapes with wB % 8 == 0, wB % 8 != 0, multi-row / single-row / split-row tiles;
    the two layouts issue the same MMAs in the same order, so they must agree bit for bit."""
    from oracle import p2p_oracle as O
    from patch2pix_b200 import _lib
    net = cnets[1]
    h = net._ready()
    rep = {}
    try:
        for hA, wA, hB, wB in ((3, 4, 5, 6), (6, 5, 9, 11), (3, 2, 30, 40), (2, 3, 12, 64), (2, 2, 7, 150), (3, 2, 45, 37),
                               (2, 3, 12, 30), (2, 2, 3, 200)):
            g = torch.Generator().manual_seed(hA * 1000 + wB)
            x = torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1
            ref = O.neigh_consensus(x, consensus_sd)
            xd = x.cuda()
            outs = {}
            for md in (mode, 3 - mode):
                net.set_option('nc_l2_mode', md)
                out = torch.full_like(xd, float('nan'))
                _lib.check(h.lib.p2p_neigh_consensus(h.h, _lib.ptr(xd), hA, wA, hB, wB, _lib.ptr(out), h.stream()))
                torch.cuda.synchronize()
                outs[md] = out.cpu()
            scale = float(ref.abs().max())
            rep[f'{hA}x{wA}x{hB}x{wB}'] = {'err': float((outs[mode] - ref).abs().max()) / scale,
                                           'modes_bit_identical': bool(torch.equal(outs[1], outs[2]))}
            np.testing.assert_allclose(outs[mode].numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * scale)
            assert torch.equal(outs[1], outs[2]), (hA, wA, hB, wB)
    finally:
        net.set_option('nc_l2_mode', 0)
        _report(f'nc_layer2_mode{mode}', rep)


def test_mutual_matching_and_unique_rows_ops():
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import mutual_matching, unique_rows
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 1, 5, 7, 6, 4, generator=g) - 0.2
    got = mutual_matching(x.cuda()).cpu()
    np.testing.assert_allclose(got.numpy(), O.mutual_matching(x).numpy(), rtol=1e-6, atol=1e-8)
    rows = torch.randint(0, 6, (5000, 4), generator=g) * 8 + 4
    for mutual in (True, False):
        ids = unique_rows(rows.cuda(), mutual).cpu().numpy()
        _, ref_ids, counts = np.unique(rows.numpy(), axis=0, return_index=True, return_counts=True)
        if mutual:
            ref_ids = ref_ids[counts > 1]
        assert np.array_equal(ids, ref_ids)
    assert len(unique_rows(torch.tensor([[1, 2, 3, 4], [4, 3, 2, 1]]).cuda(), True)) == 0
    with pytest.raises(RuntimeError):
        unique_rows(torch.tensor([[-1, 2, 3, 4]]).cuda(), True)


# ------------------------------------------------------------------------------------------------
# refine stage
# ------------------------------------------------------------------------------------------------
def _refine_case(net, sd, pair_idx, H, W, matches, impl, mid_passes, fine_passes, mid_band=0):
    from oracle import p2p_oracle as O
    f1, f2, c1, c2 = _feats(net, pair_idx, H, W)
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
        net.set_option('gemm_impl', 0)
        net.set_option('mid_passes', 3)
        net.set_option('fine_passes', 1)
        net.set_option('mid_band', 26)
    r = {
        'mid_err': (mid[0].cpu() - o_mid[0]).abs().max().item(),
        'mid_p_err': (midp[0].cpu() - o_midp[0]).abs().max().item(),
        'fine_same_err': (fine_same[0].cpu() - o_fine[0]).abs().max().item(),
        'fine_same_p_err': (finep_same[0].cpu() - o_finep[0]).abs().max().item(),
        'straddle_rows': int((mid[0].cpu().long() != o_mid[0].long()).any(1).sum()),
        'n': int(matches.shape[0]),
    }
    e2e = (fine_e2e[0].cpu() - o_fine[0]).abs().max(1)[0]
    strad = (mid[0].cpu().long() != o_mid[0].long()).any(1)
    r['fine_e2e_err_nonstraddle'] = e2e[~strad].max().item() if (~strad).any() else 0.0
    r['fine_e2e_p_err_nonstraddle'] = (finep_e2e[0].cpu() - o_finep[0]).abs()[~strad].max().item() if (~strad).any() else 0.0
    r['fine_e2e_err'] = e2e.max().item()
    r['fine_e2e_p_err'] = (finep_e2e[0].cpu() - o_finep[0]).abs().max().item()
    return r


def _random_matches(n, H, W, seed, integer):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(n, 4, generator=g) * torch.tensor([W, H, W, H]) * 1.1 - 0.05 * torch.tensor([W, H, W, H])
    m[0] = torch.tensor([0.0, 0.0, W - 1.0, H - 1.0])
    if n > 1:
        m[1] = torch.tensor([W + 3.0, -2.5, 7.999, 8.0])
    return m.long() if integer else m


@pytest.mark.parametrize('impl,mid_passes,fine_passes,band', [(1, 3, 3, 0), (0, 3, 3, 0), (0, 3, 1, 0), (0, 1, 1, 0), (0, 3, 1, 26)],
                         ids=['simt33', 'tc33', 'tc31', 'tc11', 'band31'])
@pytest.mark.parametrize('integer', [True, False])
def test_refine_vs_oracle(nets, seeded_sd, impl, mid_passes, fine_passes, band, integer):
    net = nets[1]
    H, W = 128, 160
    n = 77 if band == 0 else 777
    r = _refine_case(net, seeded_sd, 9, H, W, _random_matches(n, H, W, 3, integer), impl, mid_passes, fine_passes, band)
    _report(f'refine_impl{impl}_m{mid_passes}_f{fine_passes}_b{band}_{"i" if integer else "f"}', r)
    mid_tol = 2e-4 if (mid_passes == 3 and band == 0) else 0.05
    fine_tol = 2e-4 if fine_passes == 3 else 0.05
    assert r['mid_err'] < mid_tol, r
    assert r['fine_same_err'] < fine_tol, r
    assert r['mid_p_err'] < 1e-3 and r['fine_same_p_err'] < 1e-3, r
    assert r['fine_e2e_err_nonstraddle'] < 0.5 and r['fine_e2e_p_err_nonstraddle'] < 1e-3, r
    if mid_passes == 3:      # the shipped configurations: EVERY row within tolerance, no window moved by a pixel
        assert r['straddle_rows'] == 0, r
        assert r['fine_e2e_err'] < 0.5 and r['fine_e2e_p_err'] < 1e-3, r


@pytest.mark.parametrize('n', [1, 2, 3, 129, 1201])
def test_refine_ragged_sizes(nets, seeded_sd, n):
    net = nets[1]
    H, W = 96, 128
    r = _refine_case(net, seeded_sd, 4, H, W, _random_matches(n, H, W, n, True), 0, 3, 1)
    assert r['mid_err'] < 2e-4 and r['fine_same_err'] < 0.05 and r['fine_same_p_err'] < 1e-3, r
    r = _refine_case(net, seeded_sd, 4, H, W, _random_matches(n, H, W, n, True), 0, 3, 1, 26)
    assert r['mid_err'] < 0.05 and r['straddle_rows'] == 0 and r['fine_same_err'] < 0.05, r


def test_refine_empty_and_errors(nets):
    net = nets[1]
    f1, f2, _, _ = _feats(net, 4, 96, 128)
    out, pr = net.forward_fine_match(f1, f2, [torch.zeros(0, 4, dtype=torch.int64, device='cuda')], 16, 'center',
                                     net.regress_mid)
    assert out[0].shape == (0, 4) and pr[0].shape == (0,)
    with pytest.raises(RuntimeError):
        net.forward_fine_match(f1, f2, [torch.zeros(3, 4)], 16, 'center', net.regress_mid)      # CPU tensor
    with pytest.raises(RuntimeError):
        net.forward_fine_match(f1, f2, [torch.zeros(3, 4, device='cuda')], 8, 'center', net.regress_mid)  # psize
    with pytest.raises(RuntimeError):
        net.forward_coarse_match(f1[-1].cpu(), f2[-1].cpu(), ksize=2)


# ------------------------------------------------------------------------------------------------
# end to end sequences
# ------------------------------------------------------------------------------------------------
def _tie_masks(o_corr, c1, c2, ksize, tie_eps=1e-6, margin_eps=2e-5):
    """Rows of the reference's OWN candidate list that are ambiguous under fp32 rounding (any two correct fp32
    implementations may disagree there): the selected 4D cell's pooling window holds a top-2 gap <= tie_eps
    (-> a different relocalisation delta), or the argmax of its corr4d row/column has a top-2 margin
    <= margin_eps * max(corr4d) (-> a different partner).  Returns a bool mask over the [nB + nA] candidate rows."""
    from oracle import p2p_oracle as O
    mm = o_corr[0, 0].reshape(o_corr.shape[2] * o_corr.shape[3], -1)
    nA, nB = mm.shape
    scale = mm.max().clamp_min(1e-30)
    tA = mm.topk(2, dim=0)[0]
    tB = mm.topk(2, dim=1)[0]
    fragile = torch.cat([(tA[0] - tA[1]) <= margin_eps * scale, (tB[:, 0] - tB[:, 1]) <= margin_eps * scale])
    if ksize > 1:
        corr = O.feat_correlation_4d(O.l2_normalize(c1, 1), O.l2_normalize(c2, 1))
        k = ksize
        sl = torch.cat([corr[:, :, i::k, j::k, a::k, b::k] for i in range(k) for j in range(k) for a in range(k) for b in range(k)], 1)
        top2 = sl.topk(2, dim=1)[0]
        tie = ((top2[:, 0] - top2[:, 1]) <= tie_eps)[0].reshape(nA, nB)
        ia = mm.argmax(0)                       # best A per B cell (rows [0, nB))
        ib = mm.argmax(1)                       # best B per A cell (rows [nB, nB + nA))
        fragile = fragile | torch.cat([tie[ia, torch.arange(nB)], tie[torch.arange(nA), ib]])
    return fragile


def _e2e(net, sd, pair_idx, H, W, ptmax, panc, np_seed=7, shifted=False, feats=None):
    """Whole hot path against the oracle.  Stage 1 (coarse): the candidate lists must agree on every row that is not an
    fp32 tie of the reference itself (`_tie_masks`; such rows are counted and reported).  Stage 2 (everything
    downstream: unique/mutual filter, ptmax sampling, anchors, mid, fine) starts from the REFERENCE's candidate list on
    both sides and is compared strictly.  When the candidate lists agree completely -- the normal case -- the fused
    production entry (match_from_feats) must in addition reproduce the staged result bit for bit."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    f1, f2, c1, c2 = feats if feats is not None else _feats(net, pair_idx, H, W, shifted)
    with torch.no_grad():
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
        # downstream, from the reference's candidates on both sides
        thres_mutual = (0.0, True)
        np.random.seed(np_seed)
        if ptmax:
            o_cm, _ = O.filter_coarse(o_m, o_s, 0.0, True, ptmax=ptmax)
        else:
            o_cm, _ = O.filter_coarse(o_m, o_s, *thres_mutual)
        o_cm = O.shift_to_anchors(o_cm, panc)
        o_mid, o_midp = O.forward_fine_match(c1, c2, o_cm, sd, 'regress_mid.')
        o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, sd, 'regress_fine.')
        np.random.seed(np_seed)
        cm, _ = filter_coarse([o_m[0].cuda()], [o_s[0].cuda()], 0.0, True, ptmax=ptmax if ptmax else None)
        cm = net.shift_to_anchors(cm)
        mid, midp = net.forward_fine_match(f1, f2, cm, 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
        torch.cuda.synchronize()
        if coarse['rows_differing'] == 0:
            np.random.seed(np_seed)
            g = net.match_from_feats(f1, f2, 2, 0.0, True, ptmax, return_all=True)
            torch.cuda.synchronize()
            assert torch.equal(g[4][0], cm[0]), 'fused entry: anchors differ from the staged path'
            dfine = (g[0][0].reshape(-1, 4) - fine[0].reshape(-1, 4)).abs()
            assert torch.equal(g[0][0].reshape(-1, 4), fine[0].reshape(-1, 4)), \
                ('fused entry differs from the staged path', dfine.max().item(), int((dfine > 0).any(1).sum()),
                 (g[3][0].reshape(-1) - midp[0].reshape(-1)).abs().max().item(), (g[2][0].reshape(-1, 4) - mid[0].reshape(-1, 4)).abs().max().item())
            assert torch.equal(g[1][0].reshape(-1), finep[0].reshape(-1))
    o = (o_fine, o_finep, o_mid, o_midp, o_cm)
    g = (fine, finep, mid, midp, cm)
    return o, g, coarse


def _e2e_report(o, g):
    """north_star tolerances over EVERY row: no straddle (trunc(mid) equal to the reference's), coordinates within
    0.5 px, confidences within 1e-3.  A straddle is 'explained' only if the REFERENCE's own mid coordinate lies within
    2e-4 px of an integer (its trunc() is then an fp32 coin flip in any implementation); such rows are counted and
    excluded from the error maxima, everything else is strict."""
    o_fine, o_finep, o_mid, o_midp, o_cm = o
    fine, finep, mid, midp, cm = g
    assert cm[0].dtype == torch.int64 and torch.equal(cm[0].cpu(), o_cm[0]), 'proposals must be bit-exact'
    om = o_mid[0].reshape(-1, 4)
    strad = (mid[0].cpu().reshape(-1, 4).long() != om.long()).any(1)
    ref_tie = ((om - om.round()).abs() < 2e-4).any(1)
    explained = strad & ref_tie
    keep = ~explained
    err = (fine[0].cpu().reshape(-1, 4) - o_fine[0].reshape(-1, 4)).abs().max(1)[0]
    perr = (finep[0].cpu().reshape(-1) - o_finep[0].reshape(-1)).abs()
    detail = [{'row': int(r), 'ref_mid': [float(v) for v in om[r]], 'our_mid': [float(v) for v in mid[0].cpu().reshape(-1, 4)[r]]}
              for r in torch.nonzero(strad).flatten()[:4]]
    return {'n': int(err.numel()), 'distinct_proposals': int(torch.unique(o_cm[0], dim=0).shape[0]),
            'straddle_rows': int((strad & ~ref_tie).sum()), 'straddle_rows_reference_tie': int(explained.sum()),
            'straddle_detail': detail,
            'max_err_px': err[keep].max().item(), 'max_conf_err': perr[keep].max().item(),
            'mid_err': (mid[0].cpu().reshape(-1, 4) - om).abs().max().item()}


def _assert_e2e(rep):
    assert rep['straddle_rows'] == 0, rep
    assert rep['max_err_px'] < 0.5 and rep['max_conf_err'] < 1e-3, rep


@pytest.mark.parametrize('pair_idx,H,W,ptmax,panc', [(3, 96, 128, None, 1), (6, 240, 320, None, 1), (3, 96, 128, 12, 8),
                                                    (8, 240, 320, 50, 8)])
def test_end_to_end_vs_oracle(nets, seeded_sd, pair_idx, H, W, ptmax, panc):
    o, g, coarse = _e2e(nets[panc], seeded_sd, pair_idx, H, W, ptmax, panc)
    rep = dict(_e2e_report(o, g), **coarse)
    _report(f'e2e_{H}x{W}_pt{ptmax}_pa{panc}', rep)
    _assert_e2e(rep)


@pytest.mark.parametrize('pair_idx,H,W,ptmax,panc', [(1, 128, 160, None, 1), (4, 240, 320, None, 1), (6, 240, 320, 100, 8),
                                                    (10, 320, 480, 200, 8)])
def test_end_to_end_vs_oracle_benchmark_workload(cnets, consensus_sd, pair_idx, H, W, ptmax, panc):
    """Same, on the benchmark workload family (consensus NC weights, 16-px-shifted views): hundreds of DISTINCT
    mutual matches per pair, so every proposal / window is a different one (the last case is BASELINE configs[1]).
    "Bit-exact proposals" is only meaningful where the reference's own argmax is stable under fp32 rounding: with
    16-px-aligned views every pooling window holds four near-equal maxima, so at ~1e3 cells a few exact-tie flips per
    pair are expected in ANY fp32 implementation; `_e2e` explains and counts them."""
    o, g, coarse = _e2e(cnets[panc], consensus_sd, pair_idx, H, W, ptmax, panc, shifted=True)
    rep = dict(_e2e_report(o, g), **coarse)
    _report(f'e2e_shift_{H}x{W}_pt{ptmax}_pa{panc}', rep)
    _assert_e2e(rep)
    assert rep['distinct_proposals'] >= (0.9 * ptmax * panc if ptmax else 30), rep


@pytest.mark.parametrize('name', ['stages_96x128', 'stages_128x96', 'stages_shift_128x160'])
def test_golden_reference_vectors(nets, cnets, name):
    """CUDA path (incl. our cuDNN fp32 backbone) against outputs of the LIVE reference."""
    from patch2pix_b200.synth import synthetic_pair, synthetic_pair_shifted
    g = np.load(os.path.join(GOLD, name + '.npz'))
    net = cnets[1] if 'shift' in name else nets[1]
    im1, im2 = (synthetic_pair_shifted if 'shift' in name else synthetic_pair)(int(g['pair_idx']), int(g['H']), int(g['W']))
    with torch.no_grad():
        fine, finep, mid, midp, coarse = net.predict_fine(im1.cuda(), im2.cuda(), ksize=2, return_all=True)
        corr4d, delta4d = net.forward(im1.cuda(), im2.cuda(), ksize=2)
    np.testing.assert_allclose(corr4d.cpu().numpy(), g['corr4d'], rtol=2e-3, atol=1e-6)
    assert np.array_equal(torch.stack([d.cpu() for d in delta4d]).numpy().astype(np.int8), g['delta'])
    assert np.array_equal(coarse[0].cpu().numpy(), g['coarse'])
    assert np.abs(fine[0].cpu().numpy().reshape(-1, 4) - g['fine']).max() < 0.5
    assert np.abs(finep[0].cpu().numpy().reshape(-1) - g['fine_p']).max() < 1e-3


def test_golden_train_sequence_and_refine_only(nets, cnets):
    """Training-loop forward sequence (ptmax, panc 8) against fixtures written by the LIVE reference.  The candidate list
    must equal the reference's on every row the reference itself does not mark as an fp32 tie (`cand_fp32_tie`,
    computed by make_golden.py from the reference's tensors); everything downstream starts from the reference's
    candidates and is compared strictly."""
    from patch2pix_b200.model import filter_coarse
    from patch2pix_b200.synth import synthetic_pair, synthetic_pair_shifted
    for name in ('trainseq_96x128', 'trainseq_shift_160x240'):
        g = np.load(os.path.join(GOLD, name + '.npz'))
        net = cnets[8] if 'shift' in name else nets[8]
        im1, im2 = (synthetic_pair_shifted if 'shift' in name else synthetic_pair)(int(g['pair_idx']), int(g['H']), int(g['W']))
        with torch.no_grad():
            f1 = net.extract.forward_all(im1.cuda(), [], True)
            f2 = net.extract.forward_all(im2.cuda(), [], True)
            corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=2)
            cand, sc = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
            diff = (cand[0].cpu().numpy() != g['cand_matches'][0]).any(-1)
            assert not (diff & ~g['cand_fp32_tie']).any() and diff.sum() <= 4, (name, int(diff.sum()))
            np.random.seed(int(g['np_seed']))
            cm, _ = filter_coarse([torch.from_numpy(g['cand_matches'][0]).cuda()], [torch.from_numpy(g['cand_scores'][0]).cuda()],
                                  0.0, True, ptmax=int(g['ptmax']))
            anchors = net.shift_to_anchors(cm)
            mid, midp = net.forward_fine_match(f1, f2, anchors, 16, 'center', net.regress_mid)
            fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
            if diff.sum() == 0:                # the fused production entry reproduces the staged path
                np.random.seed(int(g['np_seed']))
                g2 = net.match_from_feats(f1, f2, 2, ptmax=int(g['ptmax']), return_all=True)
                assert torch.equal(g2[4][0], anchors[0]) and torch.equal(g2[0][0], fine[0])
        assert np.array_equal(anchors[0].cpu().numpy(), g['anchors']), name
        assert np.abs(mid[0].cpu().numpy() - g['mid']).max() < 1e-2, name
        assert np.array_equal(np.trunc(mid[0].cpu().numpy()), np.trunc(g['mid'])), name     # no fine window moved
        assert np.abs(fine[0].cpu().numpy() - g['fine']).max() < 0.5, name
        assert np.abs(finep[0].cpu().numpy() - g['fine_p']).max() < 1e-3, name
    g = np.load(os.path.join(GOLD, 'refine_128x160.npz'))
    net = nets[1]
    im1, im2 = synthetic_pair(int(g['pair_idx']), int(g['H']), int(g['W']))
    with torch.no_grad():
        r, s, c = net.refine_matches(im1.cuda(), im2.cuda(), torch.from_numpy(g['coarse_in']).cuda(), io_thres=0.0)
        rt, st, ct = net.refine_matches(im1.cuda(), im2.cuda(), g['coarse_in'], io_thres=0.5)
    assert np.abs(r - g['refined']).max() < 0.5 and np.abs(s - g['scores']).max() < 1e-3
    assert rt.shape == g['refined_t'].shape and np.abs(ct - g['coarse_t']).max() == 0


# ------------------------------------------------------------------------------------------------
# benchmark size (640x480, ptmax 400, panc 8): oracle for the coarse stage, properties for the rest
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('workload', ['legacy', 'benchmark'])
def test_full_size_640x480(nets, seeded_sd, cnets, consensus_sd, workload):
    """BASELINE configs[2] (the bench configuration): whole sequence against the oracle, EVERY one of the 3200 rows.
    'benchmark' = the workload bench.py times (consensus NC weights, shifted views: 400 distinct proposals);
    'legacy' = round-1's generator (13-17 mutual matches tiled 24x; exact zeros and ties in the NC output)."""
    bench = workload == 'benchmark'
    net, sd = (cnets[8], consensus_sd) if bench else (nets[8], seeded_sd)
    H, W = 480, 640
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    feats = _feats(net, 3 if bench else 0, H, W, shifted=bench)
    f1, f2 = feats[0], feats[1]
    o, g, coarse = _e2e(net, sd, 3 if bench else 0, H, W, 400, 8, np_seed=11, shifted=bench, feats=feats)
    with torch.no_grad():
        fine, finep, mid, midp, anch = g
        assert anch[0].shape == (3200, 4)
        rep = dict(_e2e_report(o, g), **coarse)
        _report(f'full_640x480_{workload}', rep)
        _assert_e2e(rep)
        if bench:
            assert rep['distinct_proposals'] >= 3000, rep       # 400 distinct mutual matches x 8 anchors (a few coincide)
        # properties of the refine outputs
        fm, pm = fine[0].cpu(), finep[0].cpu()
        assert fm.shape == (3200, 4) and pm.shape == (3200,)
        assert (fm[:, 0::2] >= 0).all() and (fm[:, 0::2] <= W).all() and (fm[:, 1::2] >= 0).all() and (fm[:, 1::2] <= H).all()
        assert (pm > 0).all() and (pm < 1).all()
        assert ((mid[0].cpu() - anch[0].cpu().float()).abs() <= 8.0 + 1e-4).all()   # offsets live in [-8, 8)
        # run-to-run determinism of the fused production entry (its own candidate list: it may differ from the staged
        # result above on the reference's fp32 tie rows, which _e2e starts from the reference's candidates)
        runs = []
        for _ in range(2):
            np.random.seed(11)
            runs.append(net.match_from_feats(f1, f2, 2, ptmax=400, return_all=True))
            torch.cuda.synchronize()
        assert all(torch.equal(a[0], b[0]) for a, b in zip(runs[0], runs[1]))
        if coarse['rows_differing'] == 0:
            assert torch.equal(runs[0][0][0], fine[0]) and torch.equal(runs[0][1][0], finep[0])


# ------------------------------------------------------------------------------------------------
# other BASELINE.json configurations
# ------------------------------------------------------------------------------------------------
def test_config1_480x320_ptmax200(nets, seeded_sd):
    """BASELINE configs[1]: single 480x320 pair, full coarse+mid+fine, ptmax=200 panc=8 (1600 patches/stage);
    the whole sequence is compared with the oracle (proposals exact, refine on every row)."""
    o, g, coarse = _e2e(nets[8], seeded_sd, 21, 320, 480, 200, 8)
    assert g[4][0].shape == (1600, 4)
    rep = dict(_e2e_report(o, g), **coarse)
    _report('config1_480x320', rep)
    _assert_e2e(rep)


def test_config3_1024x768_ptmax1000(cnets, consensus_sd):
    """BASELINE configs[3]: 1024x768, ptmax=1000 (x8 anchors = 8000 patches/stage), the 4D-volume memory path
    (V = 9.4 M cells, un-pooled volume 604 MB never materialised).  The WHOLE coarse stage is compared with the
    oracle at this size (pooled correlation, NC output, final corr4d, proposals, filter_coarse), the refine stage on a
    1-in-10 subsample of the rows, plus size-independent properties."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    net = cnets[8]
    H, W = 768, 1024
    f1, f2, c1, c2 = _feats(net, 1, H, W, shifted=True)
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    with torch.no_grad():
        st = {}
        o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], consensus_sd, ksize=2, stages=st)
        corr4d, delta4d, stages = net.forward_coarse_match(f1[-1], f2[-1], ksize=2, return_stages=True)
        assert corr4d.shape == (1, 1, 48, 64, 48, 64)
        np.testing.assert_allclose(stages['pooled'].cpu().numpy(), st['pooled'].numpy(), rtol=0, atol=3e-6)
        n_bad, n_unexplained = _delta_mismatch_report(delta4d, o_delta, c1[-1], c2[-1])
        assert n_unexplained == 0, (n_bad, n_unexplained)
        nc_scale = float(st['ncn'].abs().max())
        np.testing.assert_allclose(stages['ncn'].cpu().numpy(), st['ncn'].numpy(), rtol=2e-4, atol=5e-6 * nc_scale)
        np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=5e-6 * nc_scale)
        del st, stages
        # integer work at full size: proposals + unique/mutual filter
        o_m, o_s = O.cal_coarse_matches(o_corr, o_delta, ksize=2, upsample=8, center=True)
        m2, s2 = net.cal_coarse_matches(o_corr.cuda(), tuple(d.cuda() for d in o_delta), ksize=2, upsample=8)
        assert torch.equal(m2.cpu(), o_m)                                     # kernels on the oracle's volume: exact
        m, s = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=8, center=True)
        diff = (m.cpu() != o_m).any(-1)[0]                                   # on our own volume: exact up to reference ties
        fragile = _tie_masks(o_corr, c1[-1], c2[-1], 2)
        assert int((diff & ~fragile).sum()) == 0 and int(diff.sum()) <= 30, (int(diff.sum()), int((diff & ~fragile).sum()))
        fm, fs = filter_coarse(m2, s2, 0.0, True)
        ofm, ofs = O.filter_coarse(o_m, o_s, 0.0, True)
        assert torch.equal(fm[0].cpu(), ofm[0]) and fm[0].shape[0] >= 1000
        np.testing.assert_allclose(fs[0].cpu().numpy(), ofs[0].numpy(), rtol=1e-3)
        np.random.seed(5)
        o_cm, _ = O.filter_coarse(o_m, o_s, 0.0, True, ptmax=1000)
        o_anch = O.shift_to_anchors(o_cm, 8)
        np.random.seed(5)
        cm, _ = filter_coarse([o_m[0].cuda()], [o_s[0].cuda()], 0.0, True, ptmax=1000)
        anch = net.shift_to_anchors(cm)
        mid, midp = net.forward_fine_match(f1, f2, anch, 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
        torch.cuda.synchronize()
        assert anch[0].shape == (8000, 4) and torch.equal(anch[0].cpu(), o_anch[0])
        assert torch.unique(anch[0], dim=0).shape[0] >= 7500             # 1000 distinct matches x 8 anchors (a few coincide)
        np.random.seed(5)
        g2 = net.match_from_feats(f1, f2, 2, ptmax=1000, return_all=True)      # fused production entry at this size
        assert g2[4][0].shape == (8000, 4) and g2[0][0].shape == (8000, 4)
        if int(diff.sum()) == 0:
            assert torch.equal(g2[4][0], anch[0]) and torch.equal(g2[0][0], fine[0])
        fm_ = fine[0].cpu()
        assert (fm_[:, 0::2] >= 0).all() and (fm_[:, 0::2] <= W).all() and (fm_[:, 1::2] >= 0).all() and (fm_[:, 1::2] <= H).all()
        assert ((mid[0].cpu() - anch[0].cpu().float()).abs() <= 8.0 + 1e-4).all()
        idx = torch.arange(0, 8000, 10)
        o_mid, _ = O.forward_fine_match(c1, c2, [o_anch[0][idx]], consensus_sd, 'regress_mid.')
        o_fine, o_fp = O.forward_fine_match(c1, c2, o_mid, consensus_sd, 'regress_fine.')
        strad = (mid[0].cpu()[idx].long() != o_mid[0].long()).any(1)
        err = (fm_[idx] - o_fine[0]).abs().max(1)[0]
        rep = {'n_sub': int(idx.numel()), 'straddle_rows': int(strad.sum()), 'max_err_px': err.max().item(),
               'max_conf_err': (finep[0].cpu()[idx] - o_fp[0]).abs().max().item(), 'delta_cells_differing': n_bad,
               'candidate_rows_differing': int(diff.sum()), 'reference_tie_rows': int(fragile.sum())}
        _report('config3_1024x768', rep)
        _assert_e2e(rep)


def test_large_shapes_the_reference_accepts(cnets, consensus_sd):
    """Shapes beyond round 1's kernel limits (NC layer 2: hB*wB <= 3072; unique: <= 16384 candidates): ksize 1 at
    384x512 (3072 cells per image, 6144 candidates, un-pooled NC) and a 1280x960-shaped B grid at ksize 2."""
    from oracle import p2p_oracle as O
    net = cnets[1]
    f1, f2, c1, c2 = _feats(net, 5, 256, 320, shifted=True)
    with torch.no_grad():
        o_corr, _ = O.forward_coarse_match(c1[-1], c2[-1], consensus_sd, ksize=1)
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=1)
        assert delta4d is None
        np.testing.assert_allclose(corr4d.cpu().numpy(), o_corr.numpy(), rtol=5e-4, atol=5e-6 * float(o_corr.max()))
        o_m, _ = O.cal_coarse_matches(o_corr, None, ksize=1, upsample=8, center=True)
        m, _ = net.cal_coarse_matches(corr4d, None, ksize=1, upsample=8, center=True)
        diff = (m.cpu() != o_m).any(-1)[0]
        fragile = _tie_masks(o_corr, c1[-1], c2[-1], 1)
        assert int((diff & ~fragile).sum()) == 0 and int(diff.sum()) <= 12, (int(diff.sum()), int(fragile.sum()))
    # NeighConsensus alone on a wide, non-multiple-of-4 B grid and a tall one (tile logic, no shape cap)
    from patch2pix_b200 import _lib
    h = net._ready()
    for hA, wA, hB, wB in ((3, 5, 7, 150), (4, 3, 90, 37), (2, 2, 80, 60)):
        g = torch.Generator().manual_seed(hB)
        x = torch.rand(1, 1, hA, wA, hB, wB, generator=g)
        ref = O.neigh_consensus(x, consensus_sd)
        xd = x.cuda()
        out = torch.empty_like(xd)
        _lib.check(h.lib.p2p_neigh_consensus(h.h, _lib.ptr(xd), hA, wA, hB, wB, _lib.ptr(out), h.stream()))
        np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * float(ref.abs().max()))


def test_fused_gather_matches_materialised_gather(nets, seeded_sd):
    """1-pass conv1 with the gather fused into producer warps vs the TMA path over the materialised
    patch tensor: same math up to one extra fp16 rounding of the (level-normalised) features."""
    net = nets[1]
    H, W = 128, 160
    m = _random_matches(333, H, W, 11, False)
    f1, f2, _, _ = _feats(net, 9, H, W)
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
        net.set_option('fuse_gather', 3)
        net.set_option('mid_band', 26)
        net.set_option('mid_passes', 3)
    rep = {}
    for fuse in (1, 2):
        d_mid = (out[fuse][0] - out[0][0]).abs().max().item()
        d_p = (out[fuse][1] - out[0][1]).abs().max().item()
        same = (out[fuse][0].long() == out[0][0].long()).all(1)          # fine windows identical
        d_fine = (out[fuse][2] - out[0][2]).abs().max(1)[0][same].max().item()
        d_fp = (out[fuse][3] - out[0][3]).abs()[same].max().item()
        rep[f'gen{fuse}'] = {'mid_diff_px': d_mid, 'mid_conf_diff': d_p, 'fine_diff_px_same_window': d_fine,
                             'fine_conf_diff_same_window': d_fp, 'rows_with_other_window': int((~same).sum())}
        assert d_mid < 0.03 and d_p < 5e-4 and d_fine < 0.05 and d_fp < 1e-3, (fuse, rep)
    assert torch.equal(out[1][0], out[2][0]), 'both fused generations implement the same arithmetic'
    # window-map + strided-TMA conv1 (fuse_gather = 3): bit-identical A operand and MMA order -> bit-identical results
    for i in range(4):
        assert torch.equal(out[3][i], out[1][i]), ('fuse_gather 3 vs 1', i, (out[3][i] - out[1][i]).abs().max().item())
    _report('fused_vs_materialised', rep)


def test_estimate_matches_helper(seeded_sd):
    """The matcher glue of utils/eval/model_helper.py:64-109 (io_thres filter, rescaling) on top of the CUDA path."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.eval_helper import estimate_matches, load_model
    from patch2pix_b200.synth import synthetic_pair
    net = load_model(seeded_sd)
    im1, im2 = synthetic_pair(6, 240, 320)
    with torch.no_grad():
        f1, f2 = net.extract_pair(im1.cuda(), im2.cuda())         # the same (batched) backbone call predict_fine makes
        fine, fp, cm = O.hot_path_from_feats([t.cpu() for t in f1], [t.cpu() for t in f2], seeded_sd, 2, 0.0, True)
    fine, fp, cm = fine[0].reshape(-1, 4).numpy(), fp[0].reshape(-1).numpy(), cm[0].numpy()
    srt = np.sort(fp)
    gaps = srt[1:] - srt[:-1]
    g = int(np.argmax(gaps))
    thr = float(0.5 * (srt[g] + srt[g + 1]))          # threshold in the widest score gap: robust to 1e-4 differences
    m, s, c = estimate_matches(net, im1, im2, scale1=(2.0, 1.5), scale2=(1.25, 1.0), io_thres=thr)
    pos = np.where(fp > thr)[0]
    if len(pos) > 0:
        fine, fp, cm = fine[pos], fp[pos], cm[pos]
    up = np.array([[2.0, 1.5, 1.25, 1.0]])
    assert m.shape == fine.shape and np.abs(m - up * fine).max() < 0.5 * 2.0
    assert np.abs(s - fp).max() < 1e-3 and np.array_equal(c, up * cm)
    mc, sc, _ = estimate_matches(net, im1, im2, eval_type='coarse', mutual=False)
    assert mc.shape[1] == 4 and mc.shape[0] == sc.shape[0] > 0


def test_fc_tensor_core_vs_cuda_core(nets):
    """FeatRegressNet.fc on the tensor cores (3-pass, segmented) vs the fp32 CUDA-core FC kernel."""
    net = nets[1]
    H, W = 128, 160
    m = _random_matches(300, H, W, 5, True)
    f1, f2, _, _ = _feats(net, 9, H, W)
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
        net.set_option('fc_impl', 1)
        net.set_option('mid_band', 26)
    d = (out[1][0] - out[0][0]).abs().max().item()
    dp = (out[1][1] - out[0][1]).abs().max().item()
    _report('fc_tc_vs_simt', {'mid_diff_px': d, 'conf_diff': dp})
    assert d < 1e-4 and dp < 1e-5, (d, dp)


def test_batched_inputs(nets, seeded_sd):
    """The reference API is batched (b > 1 in forward_coarse_match / cal_coarse_matches, lists in
    forward_fine_match); the CUDA path loops over batch items and must give per-item identical results."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import filter_coarse
    net = nets[1]
    fa = _feats(net, 3, 96, 128)
    fb = _feats(net, 4, 96, 128)
    f1 = [torch.cat([x, y], 0) for x, y in zip(fa[0], fb[0])]
    f2 = [torch.cat([x, y], 0) for x, y in zip(fa[1], fb[1])]
    with torch.no_grad():
        corr4d, delta4d = net.forward_coarse_match(f1[-1], f2[-1], ksize=2)
        assert corr4d.shape[0] == 2 and delta4d[0].shape[0] == 2
        cm, sc = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
        fm, fs = filter_coarse(cm, sc, 0.0, True)
        assert len(fm) == 2
        mid, midp = net.forward_fine_match(f1, f2, fm, 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
        torch.cuda.synchronize()
        for i, (c1, c2) in enumerate(((fa[2], fa[3]), (fb[2], fb[3]))):
            o_fine, o_fp, o_cm = O.hot_path_from_feats(c1, c2, seeded_sd, 2, 0.0, True)
            assert torch.equal(fm[i].cpu(), o_cm[0])
            assert (fine[i].cpu().reshape(-1, 4) - o_fine[0].reshape(-1, 4)).abs().max() < 0.5
            assert (finep[i].cpu().reshape(-1) - o_fp[0].reshape(-1)).abs().max() < 1e-3


def test_load_checkpoint_file(tmp_path, nets, seeded_sd):
    """A checkpoint file in the released format (model_helper.py:28-62) gives the same network as the in-memory
    state_dict: panc is forced to 1 and predict_fine is bit-identical to a directly constructed model."""
    from argparse import Namespace
    from patch2pix_b200.eval_helper import load_checkpoint, load_model
    from patch2pix_b200.synth import synthetic_pair
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    path = tmp_path / 'p2p.pth'
    torch.save({'backbone': 'ResNet34', 'feat_idx': [0, 1, 2, 3], 'state_dict': seeded_sd, 'regressor_config': rc}, path)
    net_f = load_checkpoint(str(path), lprint=lambda s: None)
    net_m = load_model(seeded_sd)
    assert net_f.panc == 1
    im1, im2 = synthetic_pair(2, 96, 128)
    with torch.no_grad():
        a = net_f.predict_fine(im1.cuda(), im2.cuda(), ksize=2)
        b = net_m.predict_fine(im1.cuda(), im2.cuda(), ksize=2)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x[0], y[0])
    nc_path = tmp_path / 'nc.pth'
    torch.save({k: v for k, v in seeded_sd.items() if not k.startswith('regress')}, nc_path)
    net_nc = load_checkpoint(str(nc_path), method='nc', lprint=lambda s: None)
    with torch.no_grad():
        cm, sc = net_nc.predict_coarse(im1.cuda(), im2.cuda(), ksize=2)
        cm2, sc2 = net_m.predict_coarse(im1.cuda(), im2.cuda(), ksize=2)
    assert torch.equal(cm[0], cm2[0]) and torch.equal(sc[0], sc2[0])


def test_filter_coarse_branches_vs_golden():
    """Every branch of filter_coarse (networks/utils.py:38-72) with the np.unique step on the device, against the
    fixtures the live reference wrote for the crafted candidate lists of tests/golden/filter_cases.py."""
    import importlib.util
    import os
    from patch2pix_b200.model import filter_coarse
    gold = os.path.join(os.path.dirname(__file__), 'golden')
    spec = importlib.util.spec_from_file_location('filter_cases', os.path.join(gold, 'filter_cases.py'))
    fc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fc)
    g = np.load(os.path.join(gold, 'filter_quirks.npz'))
    for cname, kind, thres, mutual, ptmax, seed in fc.FILTER_CASES:
        rows, scores = fc.filter_case_inputs(kind)
        np.random.seed(seed)
        fm, fs = filter_coarse([rows.cuda()], [scores.cuda()], thres, mutual, ptmax=ptmax)
        assert np.array_equal(fm[0].cpu().numpy(), g[cname + '_matches']), cname
        assert np.array_equal(fs[0].cpu().numpy(), g[cname + '_scores']), cname


def test_unique_rows_large_lists_and_many_outstanding_tickets():
    """np.unique on the device beyond 16384 rows (global-scratch sort) and > 16 tickets in flight (every ticket owns
    its pinned counter buffer)."""
    from patch2pix_b200.model import unique_rows, unique_rows_submit
    g = torch.Generator().manual_seed(3)
    rows = torch.randint(0, 40, (40000, 4), generator=g) * 8 + 4
    rows[20000:30000] = rows[:10000]
    for mutual in (True, False):
        ids = unique_rows(rows.cuda(), mutual).cpu().numpy()
        _, ref_ids, counts = np.unique(rows.numpy(), axis=0, return_index=True, return_counts=True)
        if mutual:
            ref_ids = ref_ids[counts > 1]
        assert np.array_equal(ids, ref_ids)
    lists = [torch.randint(0, 5, (50 + 7 * i, 4), generator=g) * 16 + 4 for i in range(40)]
    tickets = [unique_rows_submit(r.cuda(), True) for r in lists]
    for r, tk in zip(lists, tickets):
        _, ref_ids, counts = np.unique(r.numpy(), axis=0, return_index=True, return_counts=True)
        assert np.array_equal(tk.wait().cpu().numpy(), ref_ids[counts > 1])
    # both implementations (rank sort over the whole GPU for lists <= 8192 rows, single-block bitonic network) at the
    # sizes around their block / chunk boundaries, with triple and double occurrences, and the out-of-range error
    from patch2pix_b200 import _lib
    h = _lib.default_handle(torch.device('cuda', 0))
    try:
        for n in (1, 2, 3, 255, 256, 257, 1000, 2400, 4097, 8192, 8193, 12000):
            r = torch.randint(0, 12, (n, 4), generator=g) * 16 + 4
            if n >= 9:
                r[n // 3:n // 3 + n // 9] = r[:n // 9]
                r[2 * (n // 3):2 * (n // 3) + n // 18] = r[:n // 18]
            _, ref_ids, counts = np.unique(r.numpy(), axis=0, return_index=True, return_counts=True)
            for impl in (1, 0):
                h.set_option('unique_impl', impl)
                for mutual in (True, False):
                    ids = unique_rows(r.cuda(), mutual, h).cpu().numpy()
                    assert np.array_equal(ids, ref_ids[counts > 1] if mutual else ref_ids), (n, impl, mutual)
        h.set_option('unique_impl', 1)
        bad = torch.full((300, 4), 70000, dtype=torch.int64)
        with pytest.raises(RuntimeError, match='65535'):
            unique_rows(bad.cuda(), True, h)
        ok = torch.randint(0, 12, (300, 4), generator=g) * 16 + 4            # the scratch is clean again after the error
        _, ref_ids, counts = np.unique(ok.numpy(), axis=0, return_index=True, return_counts=True)
        assert np.array_equal(unique_rows(ok.cuda(), False, h).cpu().numpy(), ref_ids)
    finally:
        h.set_option('unique_impl', 1)


def test_select_anchor_kernel_matches_reference_indexing(cnets):
    """filter_coarse's index arithmetic + shift_to_anchors in one launch vs the reference formulation in torch."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import _select_anchor
    g = torch.Generator().manual_seed(9)
    rows = torch.randint(0, 80, (700, 4), generator=g) * 8 + 4
    scores = torch.rand(700, generator=g)
    ids = torch.randperm(700, generator=g)[:300].int()
    sel = torch.randint(0, 300, (1000,), generator=g).int()
    m, s, a = _select_anchor(rows.cuda(), scores.cuda(), ids.cuda(), sel.cuda(), 1000, 8, 8)
    want = rows[ids.long()][sel.long()]
    assert torch.equal(m.cpu(), want) and torch.equal(s.cpu(), scores[ids.long()][sel.long()])
    assert torch.equal(a.cpu(), O.shift_to_anchors([want], 8)[0])
    assert torch.equal(cnets[8].shift_to_anchors([want.cuda()])[0].cpu(), O.shift_to_anchors([want], 8)[0])
    m, s, a = _select_anchor(rows.cuda(), scores.cuda(), None, None, 700, 1, 8)
    assert torch.equal(m.cpu(), rows) and a is None


def test_backbone_graph_tf32_path(cnets, consensus_sd):
    """The end-to-end path bench.py times: pinned host images -> H2D -> CUDA-graphed cuDNN backbone with TF32
    convolutions -> hot path.  (1) graph replay == eager under the same math mode; (2) the hot path on THOSE
    features equals the oracle on the same features (proposals exact, every row within tolerance) -- the backbone is
    not part of the path (SURVEY s8 f1), its TF32 deviation from the fp32 backbone is reported, not asserted away;
    (3) a graph instance that still backs a pending ticket refuses to be replayed."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.synth import synthetic_pair_shifted
    cfg = _cfg(8)
    cfg.weights_dict = consensus_sd
    net = Patch2PixB200(cfg)
    H, W = 240, 320
    im1, im2 = synthetic_pair_shifted(6, H, W)
    try:
        with torch.no_grad():
            f32 = net.extract_pair(im1.cuda(), im2.cuda())
            torch.backends.cudnn.allow_tf32 = True
            eager = net.extract_pair(im1.cuda(), im2.cuda())
            net.enable_backbone_graphs(H, W, instances=2)
            f1, f2 = net.extract_pair(im1.pin_memory(), im2.pin_memory())
            torch.cuda.synchronize()
            for a, b in zip(list(f1) + list(f2), list(eager[0]) + list(eager[1])):
                torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
            dev = max(((a - b).abs().max() / b.abs().max()).item() for a, b in zip(list(f1), list(f32[0])))
            c1, c2 = [t.cpu() for t in f1], [t.cpu() for t in f2]
            np.random.seed(2)
            o = O.hot_path_from_feats(c1, c2, consensus_sd, 2, 0.0, True, 100, 8, return_all=True)
            np.random.seed(2)
            tk = net.submit_coarse(f1, f2, 2, True)
            net.extract_pair(im1.pin_memory(), im2.pin_memory())          # the other instance: fine
            with pytest.raises(RuntimeError, match='pending'):
                net.extract_pair(im1.pin_memory(), im2.pin_memory())      # would overwrite the ticket's features
            g = net.finish_match(tk, 0.0, 100, return_all=True)
            torch.cuda.synchronize()
            rep = _e2e_report(o, g)
            rep['tf32_vs_fp32_backbone_rel_dev'] = dev
            # overlap mode (the backbone graph of the next pair replays on a side stream while the hot path of the pairs
            # in flight runs): a pipelined sequence over three different pairs equals the serial results bit for bit
            pairs = [synthetic_pair_shifted(k, H, W) for k in (6, 7, 8)]
            pinned = [(a.pin_memory(), b.pin_memory()) for a, b in pairs]
            net.enable_backbone_graphs(H, W, instances=3, overlap=True)
            serial = []
            for k, (a, b) in enumerate(pinned):          # same graph instance per pair as in the pipelined rounds below
                np.random.seed(10 + k)
                serial.append(net.match_from_feats(*net.extract_pair(a, b), 2, ptmax=100))
                torch.cuda.synchronize()
            tks = []
            for k, (a, b) in enumerate(pinned):
                tks.append(net.submit_coarse(*net.extract_pair(a, b), 2, True))
            for rnd in range(2):                     # second round re-uses the instances (inst['free'] protocol)
                outs = []
                for k, tk in enumerate(tks):
                    np.random.seed(10 + k)
                    outs.append(net.finish_match(tk, 0.0, 100))
                    if rnd == 0:                     # refill the instance that was just released
                        a, b = pinned[k]
                        tks[k] = net.submit_coarse(*net.extract_pair(a, b), 2, True)
                torch.cuda.synchronize()
                for sref, out in zip(serial, outs):
                    assert torch.equal(sref[0][0], out[0][0]) and torch.equal(sref[1][0], out[1][0]) and torch.equal(sref[2][0], out[2][0])
            _report('backbone_graph_tf32', rep)
            _assert_e2e(rep)
            assert dev < 2e-2, dev
    finally:
        torch.backends.cudnn.allow_tf32 = False


def test_gpu_preprocessing_is_bit_exact():
    """SURVEY s8 f4: load_im_flexible's resize + ToTensor + Normalize on the GPU (p2p_preprocess_image) against Pillow /
    torchvision's formulation (bit-exact: the resampling is integer arithmetic) and against the numpy oracle."""
    pytest.importorskip('PIL')
    from PIL import Image
    from oracle import preprocess_oracle as PO
    from patch2pix_b200.preprocess import preprocess_image
    rng = np.random.RandomState(1)
    for ho, wo, imsize in ((375, 500, 320), (480, 640, None), (200, 150, 1000), (768, 1024, 640), (97, 211, 160)):
        img = (rng.rand(ho, wo, 3) * 255).astype(np.uint8)
        out, scale, res = preprocess_image(img, 2, 16, imsize, return_resized=True)
        want, wscale = PO.load_im_flexible_array(img, 2, 16, imsize)
        assert scale == wscale and tuple(out.shape) == want.shape
        ht, wt = want.shape[1:]
        pil = np.array(Image.fromarray(img).resize((wt, ht), Image.BICUBIC))
        assert np.array_equal(res.cpu().numpy(), pil), (ho, wo, imsize)
        assert np.array_equal(out.cpu().numpy(), want), (ho, wo, imsize)
    with pytest.raises(RuntimeError):
        preprocess_image(np.zeros((10, 10, 4), np.uint8))


def test_estimate_matches_from_files(tmp_path, consensus_sd):
    """Image files in, matches out (utils/eval/model_helper.py:64-109): decode on the host, everything else on the GPU;
    equals the tensor-level entry fed with the oracle's (Pillow-exact) preprocessing, and the one-copy tail equals the
    reference's numpy formulation."""
    pytest.importorskip('PIL')
    from PIL import Image
    from oracle import preprocess_oracle as PO
    from patch2pix_b200.eval_helper import estimate_matches, estimate_matches_from_files, load_model
    from patch2pix_b200.synth import synthetic_pair_shifted
    net = load_model(consensus_sd)
    im1, im2 = synthetic_pair_shifted(4, 300, 400)
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
        scs.append(sc)
    m2, s2, c2 = estimate_matches(net, ts[0], ts[1], scs[0], scs[1], io_thres=0.3)
    assert m.dtype == np.float64 and s.dtype == np.float32 and c.dtype == np.float64
    assert np.array_equal(m, m2) and np.array_equal(s, s2) and np.array_equal(c, c2)
    # the device-side tail against the reference's numpy formulation on the raw predict_fine outputs
    with torch.no_grad():
        fine, fs, cm = net.predict_fine(ts[0].cuda(), ts[1].cuda(), ksize=2)
    fine, fs, cm = fine[0].cpu().numpy().reshape(-1, 4), fs[0].cpu().numpy().reshape(-1), cm[0].cpu().numpy()
    up = np.array([scs[0] + scs[1]])
    n_all = len(fs)
    pos = np.where(fs > 0.3)[0]
    if len(pos) > 0:
        fine, fs, cm = fine[pos], fs[pos], cm[pos]
    assert np.array_equal(m, up * fine) and np.array_equal(s, fs) and np.array_equal(c, up * cm)
    assert len(m) > 20
    # nothing passes -> everything is kept
    m3, s3, _ = estimate_matches(net, ts[0], ts[1], scs[0], scs[1], io_thres=2.0)
    assert len(m3) == n_all and len(s3) == n_all


def test_backbone_fp16_channels_last_path(consensus_sd):
    """The fp16 / channels_last backbone of the end-to-end path: pyramids come out channels-last fp16 and are consumed
    directly (p2p_coarse_nhwc16 / p2p_refine_prepare_nhwc16).  The hot path on THOSE features equals the oracle on the
    same values (up-cast to fp32 NCHW): proposals exact up to reference ties, every row within tolerance; and equals
    our own NCHW-fp32 entry points fed the same values (same arithmetic behind a different load)."""
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.synth import synthetic_pair_shifted
    cfg = _cfg(8)
    cfg.weights_dict = consensus_sd
    net = Patch2PixB200(cfg)
    H, W = 240, 320
    im1, im2 = synthetic_pair_shifted(6, H, W)
    with torch.no_grad():
        net.enable_backbone_graphs(H, W, instances=2, fast=True)
        f1, f2 = net.extract_pair(im1.pin_memory(), im2.pin_memory())
        torch.cuda.synchronize()
        assert f1[1].dtype == torch.float16 and f1[0].dtype == torch.float32
        u1 = [t.float().contiguous() for t in f1]
        u2 = [t.float().contiguous() for t in f2]
        c1, c2 = [t.cpu() for t in u1], [t.cpu() for t in u2]
        o, g, coarse = _e2e(net, consensus_sd, 6, H, W, 100, 8, np_seed=3, feats=(f1, f2, c1, c2))
        rep = dict(_e2e_report(o, g), **coarse)
        # the same values through the NCHW fp32 entry points
        np.random.seed(3)
        a = net.match_from_feats(f1, f2, 2, ptmax=100, return_all=True)
        np.random.seed(3)
        b = net.match_from_feats(u1, u2, 2, ptmax=100, return_all=True)
        torch.cuda.synchronize()
        assert torch.equal(a[4][0], b[4][0])
        rep['nhwc16_vs_nchw32_entry_max_px'] = (a[0][0] - b[0][0]).abs().max().item()
        assert rep['nhwc16_vs_nchw32_entry_max_px'] < 0.05
        # deviation of the fp16 backbone from the fp32 one (reported; the backbone is not part of the path)
        ref = net.extract.forward_all(torch.cat([im1, im2]).cuda(), [], True)
        rep['fp16_vs_fp32_backbone_rel_dev'] = max(((x[:1].float() - y[:1]).abs().max() / y.abs().max()).item() for x, y in zip(f1[1:], ref[1:]))
        _report('backbone_fp16_channels_last', rep)
        _assert_e2e(rep)
        assert rep['fp16_vs_fp32_backbone_rel_dev'] < 3e-2, rep
