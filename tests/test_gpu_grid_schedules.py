"""The persistent tensor-core kernels on grid schedules other than one CTA per SM of a 132-SM H100.

Every umma_gemm and NeighConsensus launch is persistent: CTA b runs tiles b, b + grid, b + 2 grid, ... and carries
pipeline stages, barrier parities, staged scale / bias, the shared-window class and double-buffered operands from one
tile to the next.  Each output tile is computed whole by one CTA in a fixed k order, and tiles meet only through
order-free maxima, so every result must be bit-identical for every grid size.  With 132 CTAs no CTA of a 2- or
4-column launch ever changes column tile (132 is a multiple of both); the grids here make CTAs run many tiles (1, 2),
alternate column tiles (3, 7, 131) and follow the H100 PCIe schedule (114 SMs).

Each case computes its reference once (float64 or the CPU oracle), runs the default grid and then every grid of
GRIDS: all outputs must equal the default grid's bit for bit, and the default, 1 and 131 grids must also meet the
tolerances the other GPU tests use against the same reference.
"""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GRIDS = (1, 2, 3, 7, 114, 131)
TOL_GRIDS = (0, 1, 131)        # grids also compared with the reference (0 = one CTA per SM)
DEFAULTS = {'num_sms': 0, 'nc_l2_mode': 0, 'mid_passes': 3, 'fine_passes': 1, 'mid_band': 26, 'fuse_gather': 3,
            'share_windows': 1, 'epi_async': 1, 'fc_impl': 1, 'tile_trace': 0}
SHIFTS = ((-8, -8), (8, -8), (-8, 8), (8, 8))


def _grids():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (0,) + tuple(g for g in GRIDS if g <= sms)


def _restore(h):
    for k, v in DEFAULTS.items():
        h.set_option(k, v)


def _over_grids(h, fn, grids=None):
    """{grid: fn()'s tensors on the host} for the default grid and then every grid of GRIDS."""
    out = {}
    try:
        for g in grids or _grids():
            h.set_option('num_sms', g)
            with torch.no_grad():
                r = fn()
            torch.cuda.synchronize()
            out[g] = [t.cpu() for t in r]
    finally:
        h.set_option('num_sms', 0)
    return out


def _assert_grid_independent(out, what):
    base = out[0]
    for g, r in out.items():
        assert len(r) == len(base)
        for i, (a, b) in enumerate(zip(base, r)):
            assert a.shape == b.shape and torch.equal(a, b), \
                (what, f'grid {g}', f'output {i}', int((a != b).sum()) if a.shape == b.shape else (a.shape, b.shape))


@pytest.fixture(scope='module')
def net(consensus_sd):
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    cfg = Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=consensus_sd, change_stride=True, regressor_config=rc)
    n = Patch2PixB200(cfg)
    n._ready()
    return n


def _feats(net, im1, im2):
    with torch.no_grad():
        f1 = net.extract.forward_all(im1.cuda(), [], early_feat=True)
        f2 = net.extract.forward_all(im2.cuda(), [], early_feat=True)
    return f1, f2, [t.cpu() for t in f1], [t.cpu() for t in f2]


# ------------------------------------------------------------------------------------------------
# 1. the GEMM itself (p2p_test_gemm) against float64
# ------------------------------------------------------------------------------------------------
# (passes, seg_len) -> (mean, max) error over mean |C|, as in test_gpu_parity.test_umma_gemm_matches_fp64
GEMM_LIMITS = {(1, 0): lambda K: (1e-3, 6e-3), (3, 0): lambda K: (3e-7 + 4e-9 * K, 2e-5 + 3e-8 * K),
               (3, 1): lambda K: (4e-7, 2e-5), (3, 4): lambda K: (1.5e-6, 3e-5)}


# tiles: ceil(M / 128) x ceil(N / 256) 256-wide ones (1-pass) and twice as many 128-wide ones (3-pass)
@pytest.mark.parametrize('M,N,K', [
    (1000, 300, 256),      # 16 / 32: many tiles per CTA at grids 1-7, both column tiles per CTA at 3 and 7
    (700, 4800, 128),      # 114 / 228: on one and two multiples of 114
    (600, 5800, 192),      # 115 / 230: just above them
    (1200, 3300, 128),     # 130 / 260: just below 131 and 2 x 131
    (1400, 3000, 320),     # 132 / 264: just above them
    (16700, 300, 320),     # 262 / 524: on 2 x 131 and 4 x 131
])
def test_gemm(M, N, K):
    from patch2pix_b200 import _lib
    h = _lib.default_handle('cuda:0')
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g)
    ref = a.double() @ b.double().t()
    scale = ref.abs().mean().item()
    ad, bd = a.cuda(), b.cuda()
    for (passes, seg), lim in GEMM_LIMITS.items():
        def run():
            c = torch.full((M, N), float('nan'), device='cuda')
            _lib.check(h.lib.p2p_test_gemm(h.h, _lib.ptr(ad), _lib.ptr(bd), _lib.ptr(c), M, N, K, passes, seg, 64.0,
                                           h.stream()))
            return [c]
        out = _over_grids(h, run)
        mean_tol, max_tol = lim(K)
        for grid in TOL_GRIDS:
            err = (out[grid][0].double() - ref).abs()
            assert torch.isfinite(out[grid][0]).all(), (passes, seg, grid)
            assert err.mean().item() / scale < mean_tol and err.max().item() / scale < max_tol, \
                (passes, seg, grid, err.mean().item() / scale, err.max().item() / scale)
        _assert_grid_independent(out, (M, N, K, passes, seg))


# ------------------------------------------------------------------------------------------------
# 2. coarse stage: correlation, NeighConsensus, mutual matching (p2p_coarse) against the oracle
# ------------------------------------------------------------------------------------------------
def _pooled_fp64(feat1, feat2, k=2):
    from oracle import p2p_oracle as O
    corr = O.feat_correlation_4d(O.l2_normalize(feat1.double(), 1), O.l2_normalize(feat2.double(), 1))
    return O.maxpool4d(corr, k)[0]


def _delta_mismatch_report(delta4d, o_delta, c1, c2, tie_eps=1e-6):
    """(cells whose pooling argmax differs from the oracle's, those of them not explained by an fp32 tie of the
    oracle's own top two values in the 2^4 window)."""
    from oracle import p2p_oracle as O
    bad = (torch.stack(list(delta4d)) != torch.stack(list(o_delta))).any(0)
    if not bad.any():
        return 0, 0
    corr = O.feat_correlation_4d(O.l2_normalize(c1, 1), O.l2_normalize(c2, 1))
    sl = torch.cat([corr[:, :, i::2, j::2, k::2, l::2] for i in range(2) for j in range(2) for k in range(2)
                    for l in range(2)], 1)
    top2 = sl.topk(2, dim=1)[0]
    gap = (top2[:, 0] - top2[:, 1]).unsqueeze(1)
    return int(bad.sum()), int((bad & (gap > tie_eps)).sum())


@pytest.mark.parametrize('pair_idx,size1,size2', [(11, (160, 240), (160, 240)), (5, (240, 320), (160, 192))],
                         ids=['160x240', '240x320_160x192'])
def test_coarse_stages(net, consensus_sd, pair_idx, size1, size2):
    from oracle import p2p_oracle as O
    from patch2pix_b200.synth import synthetic_pair_sized
    f1, f2, c1, c2 = _feats(net, *synthetic_pair_sized(pair_idx, size1, size2))
    st = {}
    with torch.no_grad():
        o_corr, o_delta = O.forward_coarse_match(c1[-1], c2[-1], consensus_sd, ksize=2, stages=st)
    p64 = _pooled_fp64(c1[-1], c2[-1])
    scale = max(float(st['ncn'].abs().max()), 1e-30)
    h = net._handle

    def run():
        corr4d, delta4d, stages = net.forward_coarse_match(f1[-1], f2[-1], ksize=2, return_stages=True)
        return [stages['pooled'], *delta4d, stages['ncn'], corr4d]
    out = _over_grids(h, run)
    for grid in TOL_GRIDS:
        pooled, delta, ncn, corr4d = out[grid][0], out[grid][1:5], out[grid][5], out[grid][6]
        # within 1e-6 of the oracle, or nearer the fp64 value than the oracle's own fp32 sum
        far = (pooled - st['pooled']).abs() > 1e-6
        assert not (far & ((pooled.double() - p64).abs() > (st['pooled'].double() - p64).abs())).any(), grid
        n_bad, n_unexplained = _delta_mismatch_report(delta, o_delta, c1[-1], c2[-1])
        assert n_unexplained == 0 and n_bad <= max(2, delta[0].numel() // 500), (grid, n_bad, n_unexplained)
        np.testing.assert_allclose(ncn.numpy(), st['ncn'].numpy(), rtol=2e-4, atol=5e-6 * scale, err_msg=str(grid))
        np.testing.assert_allclose(corr4d.numpy(), o_corr.numpy(), rtol=5e-4, atol=5e-6 * scale, err_msg=str(grid))
    _assert_grid_independent(out, ('coarse', size1, size2))


# the shapes of test_gpu_parity's NeighConsensus tests: (hA, wA, hB, wB), amplitude
NC_SHAPES = [((3, 4, 5, 6), 1.0), ((6, 5, 9, 11), 1e-3), ((8, 10, 8, 10), 37.0), ((15, 20, 15, 20), 1.0),
             ((2, 3, 17, 40), 1.0), ((4, 4, 4, 4), 0.0), ((3, 2, 30, 40), 1.0), ((2, 3, 12, 64), 1.0),
             ((2, 2, 7, 150), 1.0), ((3, 2, 45, 37), 1.0), ((2, 3, 12, 30), 1.0), ((2, 2, 3, 200), 1.0)]


@pytest.fixture(scope='module')
def nc_cases(consensus_sd):
    from oracle import p2p_oracle as O
    cases = []
    for (hA, wA, hB, wB), amp in NC_SHAPES:
        g = torch.Generator().manual_seed(hA * 100 + wB)
        x = (torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1) * amp
        cases.append((x, O.neigh_consensus(x, consensus_sd)))
    return cases


@pytest.mark.parametrize('l2_mode', [1, 2, 9, 10])
def test_neigh_consensus(net, nc_cases, l2_mode):
    """Layer 1's double-buffered x blocks and hidden-line stores are indexed by the CTA's own tile count; layer 2 runs
    one (mode + 8) or two CTAs per SM slot."""
    from patch2pix_b200 import _lib
    h = net._handle
    try:
        h.set_option('nc_l2_mode', l2_mode)
        for x, ref in nc_cases:
            _, _, hA, wA, hB, wB = x.shape
            xd = x.cuda()

            def run():
                o = torch.full_like(xd, float('nan'))
                _lib.check(h.lib.p2p_neigh_consensus(h.h, _lib.ptr(xd), hA, wA, hB, wB, _lib.ptr(o), h.stream()))
                return [o]
            out = _over_grids(h, run)
            scale = max(ref.abs().max().item(), 1e-30)
            for grid in TOL_GRIDS:
                assert torch.isfinite(out[grid][0]).all(), (x.shape, grid)
                np.testing.assert_allclose(out[grid][0].numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * scale,
                                           err_msg=str((x.shape, grid)))
            _assert_grid_independent(out, ('nc', tuple(x.shape), l2_mode))
    finally:
        _restore(h)


# ------------------------------------------------------------------------------------------------
# 3. refine stage: mid then fine, against the oracle
# ------------------------------------------------------------------------------------------------
H, W = 128, 160


def _random_rows(n, seed, integer):
    """n rows uniform over -5 % .. 105 % of the image, the first two on the corners and past the borders."""
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(n, 4, generator=g) * torch.tensor([W, H, W, H]) * 1.1 - 0.05 * torch.tensor([W, H, W, H])
    m[0] = torch.tensor([0.0, 0.0, W - 1.0, H - 1.0])
    if n > 1:
        m[1] = torch.tensor([W + 3.0, -2.5, 7.999, 8.0])
    return m.long() if integer else m


def _anchor_rows(n_groups, H, W, seed):
    """shift_to_anchors-style float matches: rows 0-3 of a group move point 1 by (+-8, +-8), rows 4-7 point 2; every
    seventh group has one row moved by a pixel, which leaves its half-group unshared."""
    g = torch.Generator().manual_seed(seed)
    base = (torch.rand(n_groups, 4, generator=g) * torch.tensor([W, H, W, H], dtype=torch.float32)).floor()
    rows = []
    for k in range(n_groups):
        for h in range(2):
            for dx, dy in SHIFTS:
                r = base[k].clone()
                r[2 * h] += dx
                r[2 * h + 1] += dy
                rows.append(r)
    m = torch.stack(rows) + torch.rand(8 * n_groups, 4, generator=g) * 0.9
    for k in range(0, n_groups, 7):
        m[8 * k + 1 + k % 3, 2 + k % 2] += 1.0
    return m


def _outside_rows(n, seed):
    """Every coordinate 9-30 px outside its image: the mid offsets move a coordinate by at most 8 px, so the risk band
    never flags such a row and its 3-pass launches get 0 rows."""
    g = torch.Generator().manual_seed(seed)
    d = 9.0 + 21.0 * torch.rand(n, 4, generator=g)
    far = torch.tensor([W, H, W, H], dtype=torch.float32) - 1.0 + d
    return torch.where(torch.rand(n, 4, generator=g) < 0.5, -d, far)


# name -> rows.  1-pass conv tiles: 2 ceil(n / 2) (256-wide), 3-pass: 4 ceil(n / 2); FC layers: 4 and 2 per 128 rows;
# shared-window prefix: 2 ((n / 4 + 3) / 2)
ROW_SETS = {
    'n1': lambda: _random_rows(1, 1, True),
    'n2': lambda: _random_rows(2, 2, False),
    'n131': lambda: _random_rows(131, 131, False),        # odd; 132 conv tiles: 131 + 1, 114 + 18
    'n228': lambda: _random_rows(228, 228, True),         # 228 = 2 x 114 conv tiles, 456 = 4 x 114 3-pass ones
    'n263': lambda: _random_rows(263, 263, False),        # odd; 264 = 2 x 131 + 2 conv tiles, FC 12 / 6
    'anchors': lambda: torch.cat([_anchor_rows(262, H, W, 17),     # 2099 rows, the last group partial: prefix 526
                                  torch.tensor([[3.5, 4.5, 100.2, 60.7], [3.5, 4.5, 100.2, 60.7],
                                                [W - 1.0, H - 1.0, 0.0, 0.0]])]),
    'outside': lambda: _outside_rows(57, 5),               # the band launches get 0 rows
}

# name -> options changed from the shipped configuration (mid: 1-pass + 3-pass risk band 26, fine: 1-pass)
REFINE_CONFIGS = {
    'shipped': {},
    'tc31': {'mid_band': 0},
    'tc33': {'mid_band': 0, 'fine_passes': 3},
    'fuse_gather1': {'fuse_gather': 1},
    'fuse_gather0': {'fuse_gather': 0},
    'share_windows0': {'share_windows': 0},
    'epi_async0': {'epi_async': 0},
    'fc_impl0': {'fc_impl': 0},
}


@pytest.fixture(scope='module')
def refine_ref(net, consensus_sd):
    """Features of one 128x160 pair and, for every row set, the oracle's mid on the rows and fine on that mid."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.synth import synthetic_pair_shifted
    f1, f2, c1, c2 = _feats(net, *synthetic_pair_shifted(9, H, W))
    ref = {}
    with torch.no_grad():
        for name, make in ROW_SETS.items():
            m = make()
            o_mid, o_midp = O.forward_fine_match(c1, c2, [m], consensus_sd, 'regress_mid.')
            o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, consensus_sd, 'regress_fine.')
            ref[name] = (m, o_mid[0].reshape(-1, 4), o_midp[0].reshape(-1), o_fine[0].reshape(-1, 4),
                         o_finep[0].reshape(-1))
    return f1, f2, ref


def _refine_once(net, f1, f2, m, o_mid):
    """mid on m, fine on the oracle's mid, and the rows the mid call re-ran 3-pass / shared a window half for."""
    mid, midp = net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', net.regress_mid)
    h = net._handle
    counts = torch.tensor([h.get_option('band_rows'), h.get_option('shared_rows')])
    fine, finep = net.forward_fine_match(f1, f2, [o_mid.cuda()], 16, 'center', net.regress_fine)
    return [mid[0], midp[0], fine[0], finep[0], counts]


@pytest.mark.parametrize('config', list(REFINE_CONFIGS))
def test_refine(net, refine_ref, config):
    f1, f2, ref = refine_ref
    opts = dict(DEFAULTS, **REFINE_CONFIGS[config])
    band = opts['mid_band'] > 0
    # only the window-map 1-pass conv1 shares windows: the risk band's first mid pass
    shares = band and opts['share_windows'] == 1 and opts['fuse_gather'] == 3
    mid_tol = 0.05 if band else 2e-4
    fine_tol = 2e-4 if opts['fine_passes'] == 3 else 0.05
    h = net._handle
    try:
        for k, v in opts.items():
            h.set_option(k, v)
        for name, (m, o_mid, o_midp, o_fine, o_finep) in ref.items():
            out = _over_grids(h, lambda: _refine_once(net, f1, f2, m, o_mid))
            for grid in TOL_GRIDS:
                mid, midp, fine, finep, counts = out[grid]
                what = (config, name, grid)
                assert (mid - o_mid).abs().max().item() < mid_tol, what
                assert (fine - o_fine).abs().max().item() < fine_tol, what
                assert (midp - o_midp).abs().max().item() < 1e-3 and (finep - o_finep).abs().max().item() < 1e-3, what
                # no fine window moved by a pixel, unless the oracle's own mid is within fp32 noise of an integer
                straddle = (mid.long() != o_mid.long()).any(1) & ~((o_mid - o_mid.round()).abs() < 2e-4).any(1)
                assert not straddle.any(), (what, int(straddle.sum()))
            band_rows, shared_rows = out[0][4].tolist()
            if name == 'outside' or not band:
                assert band_rows == 0, (config, name, band_rows)
            if name == 'anchors':
                if band:
                    assert band_rows > max(GRIDS), (config, band_rows)  # the band launches have more rows than CTAs
                assert (shared_rows > 0) == shares, (config, shared_rows)
            _assert_grid_independent(out, (config, name))
    finally:
        _restore(h)


# ------------------------------------------------------------------------------------------------
# 4. the schedules really are the ones named: per-tile traces (stamp 6 = CTA index + 1)
# ------------------------------------------------------------------------------------------------
def _traces(net, f1, f2, m, o_mid, grid):
    """{tag: CTA index of each tile} of the mid call on m and the fine call on o_mid at `grid` CTAs."""
    h = net._handle
    try:
        h.set_option('num_sms', grid)
        h.set_option('tile_trace', 1)
        with torch.no_grad():
            _refine_once(net, f1, f2, m, o_mid)
        band_rows = h.get_option('band_rows')
        traces = h.tile_traces()
    finally:
        _restore(h)
    out = {}
    for tag, st in traces:
        assert tag not in out, tag
        out[tag] = st[:, 6].astype(np.int64) - 1
    return out, band_rows


def test_schedule_trace(net, refine_ref):
    """Tags: stage * 8 + launch (stage 0 mid, 1 fine, 2 mid risk band; launch 0 conv1, 1-3 shared-window conv1
    prefix / continuation / unshared rows, 4 conv2).  Tile t of a launch with c column tiles has column t % c."""
    f1, f2, ref = refine_ref
    m, o_mid = ref['anchors'][0], ref['anchors'][1]
    n = m.shape[0]
    ctas, band_rows = _traces(net, f1, f2, m, o_mid, 1)
    assert band_rows > 0
    expect = {4: 2 * ((n + 1) // 2), 8: 2 * ((n + 1) // 2), 12: 2 * ((n + 1) // 2), 16: 4 * ((band_rows + 1) // 2),
              20: 4 * ((band_rows + 1) // 2)}
    for tag, tiles in expect.items():       # one CTA ran every tile of the mid conv2, the fine convs and the band convs
        assert tag in ctas and len(ctas[tag]) == tiles and (ctas[tag] == 0).all(), (tag, len(ctas.get(tag, ())), tiles)
    assert all((c == 0).all() for c in ctas.values())
    ctas, _ = _traces(net, f1, f2, m, o_mid, 3)
    for tag, tiles in expect.items():       # ... and at 3 CTAs some CTA ran tiles of two different column tiles
        c = ctas[tag]
        assert len(c) == tiles and set(c.tolist()) == {0, 1, 2}, tag
        cols = np.arange(tiles) % (4 if tag >= 16 else 2)
        assert any(len(set(cols[c == b].tolist())) > 1 for b in range(3)), tag


# ------------------------------------------------------------------------------------------------
# 5. end to end on a benchmark-workload pair
# ------------------------------------------------------------------------------------------------
def test_match_from_feats(net):
    from patch2pix_b200.synth import synthetic_pair_shifted
    f1, f2, _, _ = _feats(net, *synthetic_pair_shifted(6, 240, 320))

    def run():
        np.random.seed(6)
        fine, finep, mid, midp, cm = net.match_from_feats(f1, f2, 2, 0.0, True, 100, return_all=True)
        return [fine[0], finep[0], mid[0], midp[0], cm[0]]
    out = _over_grids(net._handle, run, (0,) + tuple(g for g in (1, 3, 114) if g in _grids()))
    assert out[0][4].shape == (800, 4)
    _assert_grid_independent(out, 'match_from_feats')
