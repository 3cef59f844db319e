"""Mid-stage conv1 with shared anchor windows (share_windows = 1) against every row's whole conv1 (share_windows = 0).

A half-group of 4 rows whose window origins on one image are equal computes that image's half of conv1 once; its rows
add the partial sum to their own half.  Rows outside such half-groups must keep the unshared arithmetic bit for bit;
shared rows differ by one reordering of a 1-pass fp32-accumulated sum.
"""
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


def _feats(net, pair_idx, H, W):
    from patch2pix_b200.synth import synthetic_pair_shifted
    im1, im2 = synthetic_pair_shifted(pair_idx, H, W)
    with torch.no_grad():
        return (net.extract.forward_all(im1.cuda(), [], early_feat=True),
                net.extract.forward_all(im2.cuda(), [], early_feat=True))


def _run(net, f1, f2, m, share, which='mid', mid_passes=3, mid_band=26):
    """(coords, probs) of one refine stage on matches m, and the shared-row counter of the call."""
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
        net.set_option('share_windows', 1)
        net.set_option('mid_passes', 3)
        net.set_option('mid_band', 26)
    return c[0].cpu(), p[0].cpu().reshape(-1), shared


def _origins(m, H, W):
    """Window origins of both images as the kernels compute them: trunc, then clamp to [-7, size + 8]."""
    t = m.long() if m.is_floating_point() else m.clone()
    lim = torch.tensor([W, H, W, H])
    return torch.minimum(torch.maximum(t, torch.full_like(t, -7)), lim + 8)


def _shared_mask(m, H, W):
    """Per row: does it belong to a half-group with equal origins on the shared image (host-side classification)."""
    o = _origins(m, H, W)
    n = m.shape[0]
    mask = torch.zeros(n, dtype=torch.bool)
    for g in range(n // 8):
        a = o[8 * g:8 * g + 4, 2:]
        b = o[8 * g + 4:8 * g + 8, :2]
        mask[8 * g:8 * g + 4] = bool((a == a[0]).all())
        mask[8 * g + 4:8 * g + 8] = bool((b == b[0]).all())
    return mask


def _anchor_groups(n_groups, H, W, seed, frac):
    """shift_to_anchors-style groups: rows 0-3 move point 1 by (+-8, +-8), rows 4-7 move point 2."""
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
    m = torch.stack(rows)
    if frac:
        m = m + torch.rand(m.shape, generator=g) * 0.9    # float matches, same trunc as the integer ones
    return m


def _assert_close(c0, p0, c1, p1, rows, tol_c, tol_p, what):
    dc = (c1[rows] - c0[rows]).abs().max().item() if rows.any() else 0.0
    dp = (p1[rows] - p0[rows]).abs().max().item() if rows.any() else 0.0
    assert dc < tol_c and dp < tol_p, (what, dc, dp)
    return dc, dp


def test_benchmark_workload_shares_every_row(net):
    """640x480, ptmax 400, panc 8: every anchor row shares a window half; mid and fine stay within the tolerances."""
    H, W = 480, 640
    for pair in (0, 3, 5):
        f1, f2 = _feats(net, pair, H, W)
        np.random.seed(pair)
        with torch.no_grad():
            g = net.match_from_feats(f1, f2, 2, 0.0, True, 400, return_all=True)
        anch = g[4][0].reshape(-1, 4)
        assert anch.shape[0] == 3200
        mid0, mp0, s0 = _run(net, f1, f2, anch, 0)
        mid1, mp1, s1 = _run(net, f1, f2, anch, 1)
        assert s0 == 0 and s1 == 3200, (s0, s1)
        assert torch.equal(mid0.long(), mid1.long()), int((mid0.long() != mid1.long()).any(1).sum())
        everything = torch.ones(3200, dtype=torch.bool)
        _assert_close(mid0, mp0, mid1, mp1, everything, 0.03, 5e-4, 'mid')
        fine0, fp0, _ = _run(net, f1, f2, mid0, 0, 'fine')
        fine1, fp1, _ = _run(net, f1, f2, mid1, 1, 'fine')
        _assert_close(fine0, fp0, fine1, fp1, everything, 0.05, 1e-3, 'fine')


def _mixed_matches(H, W):
    m = _anchor_groups(400, H, W, 17, frac=True)
    n = m.shape[0]
    for k in range(0, 400, 7):                 # break half-group A: one row's point 2 moves by a pixel
        m[8 * k + 1 + k % 3, 2 + k % 2] += 1.0
    for k in range(3, 400, 11):                # break half-group B: one row's point 1 moves
        m[8 * k + 4 + k % 4, k % 2] -= 1.0
    for k in range(5, 400, 13):                # clamped windows: distinct raw values, equal clamped origins
        m[8 * k:8 * k + 4, 2] = torch.tensor([-7.9, -9.0, -8.5, -7.0])
        m[8 * k + 4:8 * k + 8, 1] = torch.tensor([H + 8.5, H + 9.9, H + 8.0, H + 9.25])
    extra = torch.tensor([[3.5, 4.5, 100.2, 60.7], [3.5, 4.5, 100.2, 60.7], [W - 1.0, H - 1.0, 0.0, 0.0]])
    m = torch.cat([m, extra])                  # partial last group: n = 3203
    assert m.shape[0] == n + 3
    return m


def test_mixed_input_unshared_rows_bit_identical(net):
    H, W = 128, 160
    f1, f2 = _feats(net, 9, H, W)
    m = _mixed_matches(H, W)
    mask = _shared_mask(m, H, W)
    assert 0 < int(mask.sum()) < m.shape[0] - 3
    mid0, mp0, _ = _run(net, f1, f2, m, 0, mid_passes=1, mid_band=0)
    mid1, mp1, shared = _run(net, f1, f2, m, 1, mid_passes=1, mid_band=0)
    assert shared == int(mask.sum())
    assert torch.equal(mid1[~mask], mid0[~mask]) and torch.equal(mp1[~mask], mp0[~mask])
    _assert_close(mid0, mp0, mid1, mp1, mask, 0.03, 5e-4, 'shared rows')
    # integer matches and the default (risk-band) mid stage
    mi = m.floor().long()
    maski = _shared_mask(mi, H, W)
    c0, q0, _ = _run(net, f1, f2, mi, 0)
    c1, q1, shared = _run(net, f1, f2, mi, 1)
    assert shared == int(maski.sum())
    assert torch.equal(c1[~maski], c0[~maski]) and torch.equal(q1[~maski], q0[~maski])
    _assert_close(c0, q0, c1, q1, maski, 0.03, 5e-4, 'shared rows, integer')


def test_permuting_groups_permutes_outputs(net):
    H, W = 128, 160
    f1, f2 = _feats(net, 9, H, W)
    m = _mixed_matches(H, W)[:3200]
    perm = torch.randperm(400, generator=torch.Generator().manual_seed(3))
    rows = (perm[:, None] * 8 + torch.arange(8)).reshape(-1)
    c, p, s = _run(net, f1, f2, m, 1, mid_passes=1, mid_band=0)
    cp, pp, sp = _run(net, f1, f2, m[rows], 1, mid_passes=1, mid_band=0)
    assert s == sp and s > 0
    assert torch.equal(cp, c[rows]) and torch.equal(pp, p[rows])


def test_fine_stage_inputs(net):
    """Refined float mids: the fine stage never shares (bit-identical), and the mid stage's classification of such rows
    matches the host's."""
    H, W = 128, 160
    f1, f2 = _feats(net, 9, H, W)
    m = _anchor_groups(200, H, W, 5, frac=False)
    mid, _, _ = _run(net, f1, f2, m, 1)
    fine0, fp0, _ = _run(net, f1, f2, mid, 0, 'fine')
    fine1, fp1, _ = _run(net, f1, f2, mid, 1, 'fine')
    assert torch.equal(fine0, fine1) and torch.equal(fp0, fp1)
    mask = _shared_mask(mid, H, W)
    c0, q0, _ = _run(net, f1, f2, mid, 0, mid_passes=1, mid_band=0)
    c1, q1, shared = _run(net, f1, f2, mid, 1, mid_passes=1, mid_band=0)
    assert shared == int(mask.sum())
    assert torch.equal(c1[~mask], c0[~mask]) and torch.equal(q1[~mask], q0[~mask])
    _assert_close(c0, q0, c1, q1, mask, 0.03, 5e-4, 'refined mids')
