"""The fragment epilogues of the 256-wide conv1 / conv2 launches (epi_async = 1, default) against the staged epilogue
(epi_async = 0): the per-element arithmetic and the pooling max are the same, so matches and probabilities must be
equal bit for bit on every path that runs those launches -- the benchmark workload (shared anchor windows: prefix,
continuation and unshared launches), an odd patch count, a mixed shared / unshared input, conv1 fed by the patch
tensor (fuse_gather = 0), and a pair of images of different sizes."""
from argparse import Namespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHIFTS = ((-8, -8), (8, -8), (-8, 8), (8, 8))


@pytest.fixture(scope='module')
def net(consensus_sd):
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    cfg = Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=consensus_sd, change_stride=True, regressor_config=rc)
    return Patch2PixB200(cfg)


def _pyramids(net, im1, im2):
    with torch.no_grad():
        return (net.extract.forward_all(im1.cuda(), [], early_feat=True),
                net.extract.forward_all(im2.cuda(), [], early_feat=True))


def _both(net, fn, **opts):
    """fn() with epi_async 0 and 1 (and opts), as host tensors."""
    outs = []
    try:
        for k, v in opts.items():
            net.set_option(k, v)
        for e in (0, 1):
            net.set_option('epi_async', e)
            before = net._handle.get_option('frag_epi_launches')
            with torch.no_grad():
                r = fn()
            torch.cuda.synchronize()
            outs.append([t.cpu() for t in r])
            ran = net._handle.get_option('frag_epi_launches') - before
            assert (ran > 0) == bool(e), (e, ran)   # 1 really runs the fragment epilogues, 0 never does
    finally:
        net.set_option('epi_async', 1)
        for k, v in {'mid_passes': 3, 'mid_band': 26, 'fuse_gather': 3, 'share_windows': 1}.items():
            net.set_option(k, v)
    return outs


def _assert_equal(outs, what):
    a, b = outs
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x, y), (what, i, int((x != y).sum()) if x.shape == y.shape else None)


def _refine(net, f1, f2, m, which):
    reg = net.regress_mid if which == 'mid' else net.regress_fine
    c, p = net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', reg)
    return c[0], p[0]


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


def test_benchmark_workload(net):
    from patch2pix_b200.synth import synthetic_pair_shifted
    H, W = 480, 640
    for pair in (0, 3):
        f1, f2 = _pyramids(net, *synthetic_pair_shifted(pair, H, W))

        def run():
            np.random.seed(pair)
            g = net.match_from_feats(f1, f2, 2, 0.0, True, 400, return_all=True)
            return [t for t in g if torch.is_tensor(t)] + [t for x in g if isinstance(x, (list, tuple))
                                                             for t in x if torch.is_tensor(t)]
        outs = _both(net, run)
        assert sum(t.numel() for t in outs[0]) > 0
        _assert_equal(outs, f'pair {pair}')


@pytest.mark.parametrize('fuse_gather', [3, 0])
def test_odd_count_mixed_sharing(net, fuse_gather):
    """3203 rows (odd, a partial last group), shared and unshared half-groups; mid at 1 pass and with the risk band,
    then the fine stage."""
    from patch2pix_b200.synth import synthetic_pair_shifted
    H, W = 128, 160
    f1, f2 = _pyramids(net, *synthetic_pair_shifted(9, H, W))
    m = torch.cat([_anchor_rows(400, H, W, 17), torch.tensor([[3.5, 4.5, 100.2, 60.7], [3.5, 4.5, 100.2, 60.7],
                                                              [W - 1.0, H - 1.0, 0.0, 0.0]])])
    assert m.shape[0] % 2 == 1
    for passes, band in ((1, 0), (3, 26)):
        outs = _both(net, lambda: _refine(net, f1, f2, m, 'mid'), mid_passes=passes, mid_band=band,
                     fuse_gather=fuse_gather)
        _assert_equal(outs, f'mid, passes {passes}, fuse_gather {fuse_gather}')
    mid = outs[1][0]
    _assert_equal(_both(net, lambda: _refine(net, f1, f2, mid, 'fine'), fuse_gather=fuse_gather),
                  f'fine, fuse_gather {fuse_gather}')


def test_unequal_sizes(net):
    from patch2pix_b200.synth import synthetic_pair_sized
    f1, f2 = _pyramids(net, *synthetic_pair_sized(21, (128, 160), (96, 224)))
    assert f1[-1].shape[2:] != f2[-1].shape[2:]

    def run():
        np.random.seed(0)
        g = net.match_from_feats(f1, f2, 2, 0.0, True, 400, return_all=True)
        return [t for t in g if torch.is_tensor(t)] + [t for x in g if isinstance(x, (list, tuple))
                                                         for t in x if torch.is_tensor(t)]
    outs = _both(net, run)
    assert sum(t.numel() for t in outs[0]) > 0
    _assert_equal(outs, 'unequal sizes')


def test_tile_trace(net):
    """The per-tile phase trace: one stamp row per tile of every traced launch, in phase order; off, nothing is recorded."""
    from patch2pix_b200.synth import synthetic_pair_shifted
    H, W = 128, 160
    f1, f2 = _pyramids(net, *synthetic_pair_shifted(9, H, W))
    m = _anchor_rows(100, H, W, 3)
    h = net._handle
    try:
        h.set_option('tile_trace', 1)
        with torch.no_grad():
            _refine(net, f1, f2, m, 'mid')
        traces = h.tile_traces()
    finally:
        h.set_option('tile_trace', 0)
    tags = [t for t, _ in traces]
    assert 0 * 8 + 4 in tags and {1, 2} <= set(tags), tags        # conv2, prefix and continuation of the mid stage
    for tag, st in traces:
        s = st.astype(np.int64)
        assert s.shape[0] > 0 and (s[:, :6] > 0).all()
        assert (np.diff(s[:, 1:6], axis=1) >= 0).all(), tag
    assert h.get_option('tile_traces') == 0
