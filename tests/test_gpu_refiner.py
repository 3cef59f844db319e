"""The refiner workflow (Patch2Pix refining another matcher's coarse matches) on images of any size >= 8 x 8, on the
GPU: against the CPU oracle and against fixtures of the live reference (tests/golden/make_refiner_golden.py).

Tolerances are those of test_gpu_parity.py: every refined coordinate within 0.5 px and every confidence within 1e-3.
A row whose mid-stage coordinate truncates to another integer than the reference's ("straddle": the fine window moves
by a pixel) is exempt only where the reference's own mid coordinate lies within 2e-4 px of an integer, i.e. where its
trunc() is an fp32 coin flip in any implementation."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
REFINE = ['refiner_refine_97x133_120x161', 'refiner_refine_9x203_64x15', 'refiner_refine_682x1024_768x1023']
LOAD_CASES = [((45, 61), None), ((130, 97), 64), ((61, 90), 50), ((37, 203), 100)]     # as make_refiner_golden.py
FILE_CASES = [((150, 203), (161, 190), None), ((150, 203), (161, 190), 128)]
DEFAULTS = {'gemm_impl': 0, 'mid_passes': 3, 'fine_passes': 1, 'mid_band': 26, 'fuse_gather': 3, 'fc_impl': 1,
            'share_windows': 1}
ODD = (31, (97, 133), (120, 161))          # pair index, image 1 (H, W), image 2 (H, W)
TIE = 2e-4


def _restore(net):
    for k, v in DEFAULTS.items():
        net.set_option(k, v)


@pytest.fixture(scope='module')
def net(seeded_sd):
    from argparse import Namespace
    from patch2pix_b200.model import Patch2PixB200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=1, shared=False)
    cfg = Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=seeded_sd, change_stride=True, regressor_config=rc)
    return Patch2PixB200(cfg)


def _feats(net, im1, im2):
    with torch.no_grad():
        return (net.extract.forward_all(im1.cuda(), [], early_feat=True),
                net.extract.forward_all(im2.cuda(), [], early_feat=True))


def _mid_fine(net, f1, f2, rows):
    with torch.no_grad():
        mid, midp = net.forward_fine_match(f1, f2, [rows.cuda()], 16, 'center', net.regress_mid)
        fine, finep = net.forward_fine_match(f1, f2, mid, 16, 'center', net.regress_fine)
    torch.cuda.synchronize()
    return mid[0].cpu().reshape(-1, 4), fine[0].cpu().reshape(-1, 4), finep[0].cpu().reshape(-1)


def _check_rows(mid, fine, finep, ref_mid, ref_fine, ref_finep):
    """Every row within 0.5 px / 1e-3; a straddle row only where the reference's mid is an fp32 tie."""
    ref_mid, ref_fine, ref_finep = (torch.as_tensor(np.asarray(a)) for a in (ref_mid, ref_fine, ref_finep))
    strad = (mid.long() != ref_mid.long()).any(1)
    tie = ((ref_mid - ref_mid.round()).abs() < TIE).any(1)
    assert not (strad & ~tie).any(), torch.nonzero(strad & ~tie).flatten()[:8].tolist()
    keep = ~(strad & tie)
    err = (fine - ref_fine).abs().max(1)[0][keep]
    perr = (finep - ref_finep).abs()[keep]
    assert err.numel() == 0 or (err.max().item() < 0.5 and perr.max().item() < 1e-3), (err.max().item(), perr.max().item())


def _random_rows(n, s1, s2, seed, integer):
    (h1, w1), (h2, w2) = s1, s2
    g = torch.Generator().manual_seed(seed)
    dims = torch.tensor([w1, h1, w2, h2], dtype=torch.float32)
    m = torch.rand(n, 4, generator=g) * dims * 1.1 - 0.05 * dims
    m[0] = torch.tensor([0.0, 0.0, w2 - 1.0, h2 - 1.0])
    if n > 1:
        m[1] = torch.tensor([w1 - 1.0, h1 - 0.5, w2 - 0.25, h2 + 3.0])
    return m.long() if integer else m


# ------------------------------------------------------------------------------------------------
# against the live reference
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', REFINE)
def test_refine_against_reference_fixtures(net, name):
    from patch2pix_b200.synth import synthetic_pair_sized
    g = np.load(os.path.join(GOLD, name + '.npz'))
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    f1, f2 = _feats(net, im1, im2)
    cm = torch.from_numpy(g['coarse_in'])
    for tag, rows in (('', cm), ('_i', cm.long())):
        mid, fine, finep = _mid_fine(net, f1, f2, rows)
        _check_rows(mid, fine, finep, g['mid' + tag], g['refined' + tag], g['scores' + tag])
        if tag == '':
            strad = (mid.long() != torch.from_numpy(g['mid']).long()).any(1).numpy()
    with torch.no_grad():
        r, s, c = net.refine_matches(im1.cuda(), im2.cuda(), cm.cuda(), 0.0)
        rt, st, ct = net.refine_matches(im1.cuda(), im2.cuda(), g['coarse_in'], 0.5)
    assert r.dtype == np.float32 and s.dtype == np.float32 and c.dtype == np.float32
    assert np.array_equal(c, g['coarse'])
    assert np.abs(r - g['refined']).max(1)[~strad].max() < 0.5 and np.abs(s - g['scores'])[~strad].max() < 1e-3
    if not (np.abs(g['scores'] - 0.5) < 1e-3).any():          # the same rows pass io_thres 0.5
        assert np.array_equal(ct, g['coarse_t']) and rt.shape == g['refined_t'].shape


# ------------------------------------------------------------------------------------------------
# against the oracle: row counts, match dtypes, both prepare entries
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prep', ['nchw32', 'nhwc16'])
@pytest.mark.parametrize('integer', [True, False])
@pytest.mark.parametrize('n', [1, 129, 1201])
def test_refine_against_oracle(net, seeded_sd, n, integer, prep):
    """fp32 NCHW pyramids (p2p_refine_prepare) and channels-last fp16 ones (p2p_refine_prepare_nhwc16; the oracle then
    reads the same fp16-rounded values) at an odd-sized pair."""
    from oracle import p2p_oracle as O
    from patch2pix_b200.synth import synthetic_pair_sized
    idx, s1, s2 = ODD
    im1, im2 = synthetic_pair_sized(idx, s1, s2)
    f1, f2 = _feats(net, im1, im2)
    if prep == 'nhwc16':
        f1, f2 = ([f[0]] + [t.half().to(memory_format=torch.channels_last) for t in f[1:]] for f in (f1, f2))
    rows = _random_rows(n, s1, s2, 100 + n, integer)
    mid, fine, finep = _mid_fine(net, f1, f2, rows)
    c1, c2 = ([t.float().cpu() for t in f] for f in (f1, f2))
    with torch.no_grad():
        o_mid, _ = O.forward_fine_match(c1, c2, [rows], seeded_sd, 'regress_mid.')
        o_fine, o_finep = O.forward_fine_match(c1, c2, o_mid, seeded_sd, 'regress_fine.')
    _check_rows(mid, fine, finep, o_mid[0].reshape(-1, 4), o_fine[0].reshape(-1, 4), o_finep[0].reshape(-1))


# ------------------------------------------------------------------------------------------------
# paths that must agree at odd sizes
# ------------------------------------------------------------------------------------------------
def _anchor_rows(s1, s2, n_groups=48):
    """shift_to_anchors-style groups (rows 0-3 move point 1 by (+-8, +-8), rows 4-7 point 2) over each image's own
    range, including groups at the far borders, plus a partial last group."""
    (h1, w1), (h2, w2) = s1, s2
    g = torch.Generator().manual_seed(5)
    base = (torch.rand(n_groups, 4, generator=g) * torch.tensor([w1, h1, w2, h2], dtype=torch.float32)).floor()
    base[::5] = torch.tensor([w1 - 1.0, h1 - 1.0, w2 - 1.0, h2 - 1.0])
    rows = []
    for k in range(n_groups):
        for h in range(2):
            for dx, dy in ((-8, -8), (8, -8), (-8, 8), (8, 8)):
                r = base[k].clone()
                r[2 * h] += dx
                r[2 * h + 1] += dy
                rows.append(r)
    m = torch.stack(rows) + 0.5
    return torch.cat([m, m[:3] + 0.25])


@pytest.mark.parametrize('rows_kind', ['random', 'anchors'])
def test_refine_paths_agree_at_odd_sizes(net, rows_kind):
    """1-pass and 3-pass mid: the window maps (fuse_gather 3) and the fused gathers (1, 2) give the same bits, the
    materialised patch tensor (0) stays within one fp16 rounding of the features.  Sharing anchor windows
    (share_windows, which only the window-map path does) changes only the rows of shared half-groups, within the same
    bound, and leaves the other paths untouched."""
    from patch2pix_b200.synth import synthetic_pair_sized
    idx, s1, s2 = ODD
    f1, f2 = _feats(net, *synthetic_pair_sized(idx, s1, s2))
    rows = _random_rows(333, s1, s2, 11, False) if rows_kind == 'random' else _anchor_rows(s1, s2)
    out = {}
    try:
        for passes in (1, 3):
            for share in (0, 1):
                for fuse in (3, 1, 2, 0):
                    net.set_option('mid_passes', passes)
                    net.set_option('mid_band', 0)
                    net.set_option('share_windows', share)
                    net.set_option('fuse_gather', fuse)
                    out[passes, share, fuse] = _mid_fine(net, f1, f2, rows)
    finally:
        _restore(net)

    def same(a, b, what):
        for i in range(3):
            assert torch.equal(a[i], b[i]), (what, i, (a[i] - b[i]).abs().max().item())

    def close(a, b, what):
        win = (a[0].long() == b[0].long()).all(1)
        assert (a[0] - b[0]).abs().max().item() < 0.03, what
        assert (a[1] - b[1]).abs().max(1)[0][win].max().item() < 0.05 and (a[2] - b[2]).abs()[win].max().item() < 1e-3, what

    for passes in (1, 3):
        same(out[passes, 0, 3], out[passes, 0, 1], f'{passes}-pass: fuse_gather 3 vs 1')
        same(out[passes, 0, 3], out[passes, 0, 2], f'{passes}-pass: fuse_gather 3 vs 2')
        close(out[passes, 0, 3], out[passes, 0, 0], f'{passes}-pass: fuse_gather 3 vs 0')
        for fuse in (1, 2, 0):
            same(out[passes, 0, fuse], out[passes, 1, fuse], f'{passes}-pass fuse_gather {fuse}: share_windows 0 vs 1')
        close(out[passes, 0, 3], out[passes, 1, 3], f'{passes}-pass: share_windows 0 vs 1')
    if rows_kind == 'random':      # no half-group shares a window: sharing changes nothing
        same(out[1, 0, 3], out[1, 1, 3], 'random rows: share_windows 0 vs 1')


# ------------------------------------------------------------------------------------------------
# load_im_tensor and the file-to-matches entry point
# ------------------------------------------------------------------------------------------------
def test_load_im_tensor_bit_exact(tmp_path):
    """Against the reference's outputs and against Pillow's resize / convert('L') with to_tensor / normalize's float32
    arithmetic restated in numpy."""
    from PIL import Image
    from patch2pix_b200.preprocess import load_im_tensor, tensor_size
    from patch2pix_b200.synth import synthetic_photo_pair
    g = np.load(os.path.join(GOLD, 'refiner_load_im_tensor.npz'))
    mean = np.array([0.485, 0.456, 0.406], np.float32).reshape(3, 1, 1)
    std = np.array([0.229, 0.224, 0.225], np.float32).reshape(3, 1, 1)
    for k, (size, imsize) in enumerate(LOAD_CASES):
        img, _ = synthetic_photo_pair(10 + k, size, size)
        path = str(tmp_path / f'load{k}.png')
        Image.fromarray(img).save(path)
        im, gray, scale = load_im_tensor(path, 'cuda:0', imsize)
        assert im.is_cuda and gray.is_cuda and im.dtype == gray.dtype == torch.float32
        assert np.array_equal(im.cpu().numpy(), g[f'im{k}']) and np.array_equal(gray.cpu().numpy(), g[f'gray{k}']), k
        assert scale == tuple(g[f'scale{k}']), k
        pil = Image.open(path)
        wt, ht = tensor_size(pil.width, pil.height, imsize)
        if (wt, ht) != pil.size:
            pil = pil.resize((wt, ht), Image.BICUBIC)
        assert np.array_equal(gray.cpu().numpy()[0, 0], np.asarray(pil.convert('L')).astype(np.float32) / np.float32(255))
        x = np.asarray(pil).astype(np.float32).transpose(2, 0, 1) / np.float32(255)
        assert np.array_equal(im.cpu().numpy()[0], (x - mean) / std), k
        im2, scale2 = load_im_tensor(path, 'cuda:0', imsize, with_gray=False)
        assert torch.equal(im2, im) and scale2 == scale


def _write_pair(tmp_path, k, size1, size2):
    from PIL import Image
    from patch2pix_b200.synth import synthetic_photo_pair
    a, b = synthetic_photo_pair(20 + k, size1, size2)
    p1, p2 = str(tmp_path / f'f{k}a.png'), str(tmp_path / f'f{k}b.png')
    Image.fromarray(a).save(p1)
    Image.fromarray(b).save(p2)
    return p1, p2


@pytest.mark.parametrize('k', range(len(FILE_CASES)))
def test_refine_matches_from_files(net, tmp_path, k):
    from patch2pix_b200.eval_helper import refine_matches
    from patch2pix_b200.synth import grid_coarse_matcher
    g = np.load(os.path.join(GOLD, 'refiner_files.npz'))
    size1, size2, imsize = FILE_CASES[k]
    p1, p2 = _write_pair(tmp_path, k, size1, size2)
    r, s, c = refine_matches(p1, p2, net, grid_coarse_matcher(), io_thres=0.0, imsize=imsize)
    assert r.dtype == np.float64 and c.dtype == np.float64 and s.dtype == np.float32
    assert r.shape == g[f'refined{k}'].shape and np.array_equal(c, g[f'coarse{k}'])
    # in the loaded image's pixels; a row off by more is a straddle, allowed only on the reference's fp32 ties
    err = (np.abs(r - g[f'refined{k}']) / np.array([_scales(size1, size2, imsize)])).max(1)
    bad = err >= 0.5
    assert not (bad & ~g[f'mid_tie{k}']).any(), np.nonzero(bad & ~g[f'mid_tie{k}'])[0][:8]
    assert np.abs(s - g[f'scores{k}'])[~bad].max() < 1e-3
    rt, st, ct = refine_matches(p1, p2, net, grid_coarse_matcher(), io_thres=0.5, imsize=imsize)
    if not (np.abs(g[f'scores{k}'] - 0.5) < 1e-3).any():
        assert np.array_equal(ct, g[f'coarse{k}_t']) and rt.shape == g[f'refined{k}_t'].shape
    co, none1, none2 = refine_matches(p1, p2, net, grid_coarse_matcher(), imsize=imsize, coarse_only=True)
    assert none1 is None and none2 is None and np.array_equal(co, g[f'coarse_only{k}'])
    # other coarse-match types: float64 rows refine as their float32 values (and come back as float64); numpy rows
    # run as device rows do; int64 rows keep their integer values
    r64, s64, c64 = refine_matches(p1, p2, net, grid_coarse_matcher(dtype=torch.float64), imsize=imsize)
    assert np.array_equal(r64, r) and np.array_equal(s64, s)
    rows64 = grid_coarse_matcher(dtype=torch.float64)(*_greys(size1, size2, imsize)).numpy()
    assert np.array_equal(c64, np.array([_scales(size1, size2, imsize)]) * rows64)
    rn, sn, cn = refine_matches(p1, p2, net, lambda a, b: grid_coarse_matcher()(a, b).cpu().numpy(), imsize=imsize)
    assert np.array_equal(rn, r) and np.array_equal(sn, s) and np.array_equal(cn, c)
    ri, si, ci = refine_matches(p1, p2, net, grid_coarse_matcher(dtype=torch.int64), imsize=imsize)
    assert ri.shape == r.shape and np.array_equal(ci, np.array([_scales(size1, size2, imsize)]) *
                                                  grid_coarse_matcher(dtype=torch.int64)(*_greys(size1, size2, imsize)).numpy())


def _loaded_size(size, imsize):
    from patch2pix_b200.preprocess import tensor_size
    wt, ht = tensor_size(size[1], size[0], imsize)
    return ht, wt


def _scales(size1, size2, imsize):
    (h1, w1), (h2, w2) = _loaded_size(size1, imsize), _loaded_size(size2, imsize)
    return (size1[1] / w1, size1[0] / h1, size2[1] / w2, size2[0] / h2)


def _greys(size1, size2, imsize):
    return torch.zeros(1, 1, *_loaded_size(size1, imsize)), torch.zeros(1, 1, *_loaded_size(size2, imsize))


def test_refine_size_limits(net):
    """Images below 8 x 8 are refused (the reference's level-3 clamp bound would be -1)."""
    from patch2pix_b200.synth import synthetic_pair_sized
    im1, im2 = synthetic_pair_sized(1, (7, 64), (64, 64))
    with pytest.raises(RuntimeError):
        net.refine_matches(im1.cuda(), im2.cuda(), np.zeros((3, 4), np.float32), 0.0)
    im1, im2 = synthetic_pair_sized(1, (8, 8), (8, 9))
    with torch.no_grad():
        r, s, c = net.refine_matches(im1.cuda(), im2.cuda(), np.array([[3.5, 4.5, 8.0, 7.0]], np.float32), 0.0)
    assert r.shape == (1, 4) and np.isfinite(r).all() and 0 <= s[0] <= 1
