"""SuperPoint keypoints, descriptors and exact nearest-neighbour matching on the GPU (csrc/keypoints.cu) against the CPU
restatement (oracle/superpoint_oracle.py), and SuperPoint + NN as the coarse matcher of Patch2Pix's refiner."""
import os

import numpy as np
import pytest
import torch

from oracle import superpoint_oracle as O
from patch2pix_b200 import superpoint as SP

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _logits(seed, B, hc, wc, kind='random'):
    g = torch.Generator().manual_seed(seed)
    if kind == 'random':
        x = torch.randn(B, 65, hc, wc, generator=g) * 3
    elif kind == 'ties':           # few distinct logits: equal scores inside cells and plateaus across them
        x = torch.randint(0, 3, (B, 65, hc, wc), generator=g).float()
    elif kind == 'flat':           # every score 1/65: one plateau over the image
        x = torch.zeros(B, 65, hc, wc)
    else:                          # 'zero': the dustbin takes everything, scores underflow to 0
        x = torch.zeros(B, 65, hc, wc)
        x[:, 64] = 200.0
    return x


def _check_keypoints(logits, r=4, thr=0.005, border=4, k=-1):
    kps, scs, smap = SP.detect_keypoints(logits.to(DEV), r, thr, k, border, return_score_map=True)
    smap = smap.cpu()
    for b in range(logits.shape[0]):
        ref = torch.from_numpy(O.score_map(logits[b]))
        assert (smap[b] - ref).abs().max().item() < 1e-6
        okp, osc = O.keypoints(smap[b].numpy(), r, thr, border, k)
        assert np.array_equal(kps[b].cpu().numpy(), okp), (b, len(kps[b]), len(okp))
        assert np.array_equal(scs[b].cpu().numpy(), osc)
    return kps, scs, smap


@pytest.mark.parametrize('kind', ['random', 'ties', 'flat', 'zero'])
@pytest.mark.parametrize('k', [-1, 0, 7, 300])
def test_keypoints_equal_oracle_on_the_kernel_score_map(kind, k):
    _check_keypoints(_logits(1, 3, 13, 17, kind), k=k)


@pytest.mark.parametrize('hc, wc, r, border', [(1, 1, 4, 4), (1, 1, 0, 0), (1, 7, 2, 0), (3, 5, 1, 2), (5, 3, 16, 3),
                                               (9, 11, 0, 9)])
def test_keypoints_tiny_and_odd_sizes(hc, wc, r, border):
    for kind in ('random', 'ties'):
        _check_keypoints(_logits(hc * 31 + wc, 2, hc, wc, kind), r=r, border=border)
        _check_keypoints(_logits(hc * 31 + wc, 2, hc, wc, kind), r=r, border=border, k=3)


def test_threshold_equal_to_a_score_is_excluded():
    logits = _logits(5, 1, 12, 12)
    _, scs, _ = _check_keypoints(logits)
    for thr in (float(scs[0][0]), float(scs[0].max()), float(scs[0].min()), -1.0):
        _, s, _ = _check_keypoints(logits, thr=thr)
        assert (s[0] > thr).all()


def test_keypoints_1600x1200():
    _check_keypoints(_logits(7, 1, 150, 200), k=-1)
    _check_keypoints(_logits(7, 1, 150, 200, 'ties'), k=2048)


def test_descriptors_within_1e6_of_float64_oracle():
    g = torch.Generator().manual_seed(3)
    B, D, hc, wc = 2, 256, 11, 14
    desc = torch.randn(B, D, hc, wc, generator=g)
    desc[0, :, 2, 3] = 0                                          # a zero cell (normalised by eps)
    kps = [torch.tensor([[0, 0], [8 * wc - 1, 8 * hc - 1], [3, 4], [57, 33], [100, 2]], dtype=torch.float32),
           torch.stack([torch.randint(0, 8 * wc, (400,), generator=g), torch.randint(0, 8 * hc, (400,), generator=g)],
                       1).float()]
    out = SP.sample_descriptors(desc.to(DEV), [k.to(DEV) for k in kps])
    for b in range(B):
        ref = O.sample_descriptors(desc[b].numpy(), kps[b].numpy())
        assert np.abs(out[b].cpu().double().numpy() - ref).max() < 1e-6
    empty = SP.sample_descriptors(desc.to(DEV), [kps[0][:0].to(DEV), kps[1].to(DEV)])
    assert empty[0].shape == (0, D)


def _unit(g, n, d):
    x = torch.randn(n, d, generator=g)
    return (x / x.norm(dim=1, keepdim=True)).float()


def _adversarial(g, n, m, d):
    a, b = _unit(g, n, d), _unit(g, m, d)
    if n >= 4 and m >= 4:
        b[1] = b[0]                                               # duplicated columns: exact ties
        a[1] = a[0]                                               # duplicated rows: exact column ties
        a[2] = b[2]
        b[3] = b[2].clone()
        b[3, 0] = torch.nextafter(b[3, 0], torch.tensor(2.0))     # a near-tie one ulp away
        a[3] = b[3]
    return a, b


def _check_match(a, b, **kw):
    S = O.similarity(a.numpy(), b.numpy())
    om, os_ = O.match(a.numpy(), b.numpy(), S=S, **kw)
    h = SP._handle(DEV)
    for impl in (1, 0):                     # tensor-core pass + float64 fix-up, float64 only
        h.set_option('match_impl', impl)
        try:
            probe = {} if impl == 1 else None
            m, s = SP._match_batch([a.to(DEV)], [b.to(DEV)], kw.get('mutual', True), kw.get('min_sim'),
                                   kw.get('ratio'), probe)[0]
        finally:
            h.set_option('match_impl', 1)
        assert np.array_equal(m.cpu().numpy(), om), impl
        assert np.array_equal(s.cpu().numpy(), os_), impl
        if probe is not None and len(a) and len(b):
            # the measured tensor-core error stays below the derived bound
            tc, idx, eps = probe['tc_sim'].cpu().numpy(), probe['tc_idx'].cpu().numpy(), float(probe['eps'][0])
            err = np.abs(tc - S[np.arange(len(a)), idx]).max()
            assert err < eps, (err, eps)
    return m, s


@pytest.mark.parametrize('d', [64, 128, 256])
@pytest.mark.parametrize('n, m', [(0, 5), (5, 0), (1, 1), (1, 9), (9, 1), (70, 130), (300, 257)])
def test_matching_equals_float64_oracle_exactly(d, n, m):
    g = torch.Generator().manual_seed(d * 1000 + n * 7 + m)
    a, b = _adversarial(g, n, m, d)
    for kw in (dict(), dict(mutual=False), dict(mutual=True, min_sim=0.1), dict(mutual=False, ratio=0.9),
               dict(mutual=True, min_sim=-0.05, ratio=0.95)):
        _check_match(a, b, **kw)


def test_matching_near_ties_inside_the_last_bits():
    g = torch.Generator().manual_seed(11)
    base = _unit(g, 1, 256)
    b = base.repeat(64, 1)
    for j in range(64):                                           # columns apart by a few ulps in one component
        b[j, j % 256] = torch.nextafter(b[j, j % 256], torch.tensor(2.0 if j % 2 else -2.0))
    a = torch.cat([base, b[::3], _unit(g, 40, 256)])
    for kw in (dict(), dict(mutual=False), dict(mutual=False, ratio=0.999999)):
        _check_match(a, b, **kw)


def test_batch_equals_single_calls_without_host_sync():
    g = torch.Generator().manual_seed(2)
    sizes = [(37, 40), (0, 3), (5, 0), (300, 120), (1, 1), (64, 64)]
    l0 = [_unit(g, n, 128).to(DEV) for n, _ in sizes]
    l1 = [_unit(g, m, 128).to(DEV) for _, m in sizes]
    SP.match_descriptors_batch(l0, l1)                            # warm the handle and scratch
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = SP.match_descriptors_batch(l0, l1, ratio=0.95)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    for k, (a, b) in enumerate(zip(l0, l1)):
        m, s = SP.match_descriptors(a, b, ratio=0.95)
        assert torch.equal(out[k][0], m) and torch.equal(out[k][1], s)


def test_tensor_core_error_bound_and_fixup_count():
    g = torch.Generator().manual_seed(21)
    for d in (64, 256):
        a, b = _unit(g, 2000, d), _unit(g, 1500, d)
        b[:40] = a[:40]                                             # exact ties: rows that must be fixed up
        S = O.similarity(a.numpy(), b.numpy())
        probe = {}
        m, s = SP._match_batch([a.to(DEV)], [b.to(DEV)], True, None, 0.9, probe)[0]
        om, os_ = O.match(a.numpy(), b.numpy(), True, None, 0.9, S=S)
        assert np.array_equal(m.cpu().numpy(), om) and np.array_equal(s.cpu().numpy(), os_)
        tc, idx, eps = probe['tc_sim'].cpu().numpy(), probe['tc_idx'].cpu().numpy(), float(probe['eps'][0])
        assert np.abs(tc - S[np.arange(len(a)), idx]).max() < eps < 1e-4
        fixed = probe['n_fixed'].cpu().tolist()
        assert fixed[0] < len(a) // 10 and fixed[1] < len(b) // 10


def test_matching_argument_checks():
    a = torch.zeros(4, 24, device=DEV)
    with pytest.raises(RuntimeError, match='dim'):
        SP.match_descriptors(a, a)
    with pytest.raises(ValueError):
        SP.match_descriptors(a.double(), a.double())
    with pytest.raises(ValueError):
        SP.match_descriptors(torch.zeros(4, 32, device=DEV), torch.zeros(4, 48, device=DEV))
    with pytest.raises(ValueError):
        SP.match_descriptors(torch.zeros(4, 32, device=DEV), torch.zeros(4, 32, device=DEV), ratio=-1)


@pytest.fixture(scope='module')
def sp():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    net = SP.SuperPoint(max_keypoints=400)
    net.load_state_dict(O.seeded_state_dict(0))
    return net.to(DEV)


def test_superpoint_end_to_end_against_cpu_oracle(sp):
    from patch2pix_b200.synth import synthetic_photo_pair
    im, _ = synthetic_photo_pair(3, (120, 161), (120, 161))
    grey = torch.from_numpy(im.mean(2, dtype=np.float64) / 255.0).float()[None, None]
    out = sp({'image': grey.to(DEV)})
    sd = O.seeded_state_dict(0)
    with torch.no_grad():
        logits, desc = O.heads(sd, grey)
    smap = O.score_map(logits[0])
    okp, _ = O.keypoints(smap, 4, 0.005, 4, 400)
    got = {tuple(p) for p in out['keypoints'][0].cpu().numpy().astype(int).tolist()}
    want = {tuple(p) for p in okp.astype(int).tolist()}
    # a keypoint may differ only where its score is within MARGIN of the threshold, of an NMS rival within 3r, or of
    # the 400th score (the top-k cut): fp32 convolutions in another order move scores by ~1e-7
    MARGIN = 1e-5
    cut = float(np.sort(O.nms(smap, 4)[4:-4, 4:-4].ravel())[::-1][399])
    for x, y in got ^ want:
        s = smap[y, x]
        win = smap[max(0, y - 12):y + 13, max(0, x - 12):x + 13]
        near_rival = (np.abs(win - s) < MARGIN).sum() > 1
        assert abs(s - 0.005) < MARGIN or abs(s - cut) < MARGIN or near_rival, (x, y, s)
    assert len(got ^ want) <= max(2, len(want) // 100)
    assert out['descriptors'][0].shape == (256, len(got))
    common = [i for i, p in enumerate(out['keypoints'][0].cpu().numpy().astype(int).tolist()) if tuple(p) in want]
    kp_c = out['keypoints'][0][common].cpu().numpy()
    ref = O.sample_descriptors(desc[0].numpy(), kp_c)
    assert np.abs(out['descriptors'][0][:, common].T.cpu().double().numpy() - ref).max() < 1e-4


@pytest.fixture(scope='module')
def p2p_net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


def test_refine_matches_with_superpoint_nn(sp, p2p_net, tmp_path):
    from PIL import Image
    from patch2pix_b200.eval_helper import refine_matches
    from patch2pix_b200.synth import synthetic_photo_pair
    a, b = synthetic_photo_pair(4, (150, 203), (161, 190))
    p1, p2 = str(tmp_path / 'a.png'), str(tmp_path / 'b.png')
    Image.fromarray(a).save(p1)
    Image.fromarray(b).save(p2)
    matcher = SP.superpoint_nn_matcher(sp)
    coarse, _, _ = refine_matches(p1, p2, p2p_net, matcher, coarse_only=True)
    assert coarse.shape[1] == 4 and len(coarse) > 0
    rows = []

    def recorded(g1, g2):
        r = matcher(g1, g2)
        rows.append(r)
        return r
    refined, scores, coarse2 = refine_matches(p1, p2, p2p_net, recorded, io_thres=0.0)
    fixed, fscores, _ = refine_matches(p1, p2, p2p_net, lambda g1, g2: rows[0].clone(), io_thres=0.0)
    assert np.array_equal(coarse, coarse2) and np.array_equal(refined, fixed) and np.array_equal(scores, fscores)
    assert np.isfinite(refined).all() and refined.shape == coarse.shape
    # SuperPoint's rows are integer pixels of the grey images, mutual nearest neighbours: one row per keypoint at most
    g = rows[0].cpu().numpy()
    assert np.array_equal(g, np.round(g)) and len(np.unique(g[:, :2], axis=0)) == len(g)


def test_eval_hpatches_with_sp_patch2pix_matcher(sp, p2p_net, tmp_path):
    from patch2pix_b200 import hpatches as HP
    from patch2pix_b200.synth import synthetic_hpatches_tree
    root = str(tmp_path / 'hp')
    os.makedirs(root)
    synthetic_hpatches_tree(root, 7, [('i_a', (200, 150)), ('v_c', (240, 176))])
    res = HP.eval_hpatches(SP.sp_patch2pix_matcher(p2p_net, sp, 0.0, 1024), root, lprint_=lambda s: None)
    assert res['n_pairs'] == 10
    assert not any(r.match_failed for r in res['records'])
    assert all(r.N > 0 for r in res['records'])
