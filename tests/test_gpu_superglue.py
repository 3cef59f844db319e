"""SuperGlue's optimal transport and extraction on the GPU (csrc/superglue.cu, p2p_sg_sinkhorn) and the whole module
(patch2pix_b200/superglue.py) against the float64 restatement (oracle/superglue_oracle.py), and SuperPoint + SuperGlue
as the coarse matcher of Patch2Pix's refiner.

Decisions are compared on every row and column whose margins exceed twice the error bound (oracle.decidable): log_assign
is within the bound of float64, so no decision with a larger margin can differ."""
import os

import numpy as np
import pytest
import torch

from oracle import superglue_oracle as O
from patch2pix_b200 import superglue as SG

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
# allowed |scores_fp32 - scores_fp64| of the GNN path with TF32 off (measured about 3e-5 on scores of magnitude ~50)
GNN_TOL = 1e-3


def _planted_scores(seed, B, n, m, d=64, frac=0.7, scale=20.0):
    """scale x cosine similarities of seeded unit descriptors, frac of the smaller side planted as near-duplicates."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(B):
        def unit(k):
            x = torch.randn(k, d, generator=g, dtype=torch.float64)
            return x / x.norm(dim=1, keepdim=True)
        a, b = unit(n), unit(m)
        k = int(frac * min(n, m))
        pi, pj = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        b[pj] = a[pi] + 0.3 * unit(k)
        b = b / b.norm(dim=1, keepdim=True)
        out.append(a @ b.T * scale)
    return torch.stack(out).float()


def _compare(got, ref_la, thr, tol, ms_tol):
    """got: one pair's GPU outputs (numpy); ref_la the float64 log_assign.  -> excluded rows + columns, total."""
    e = O.extract(ref_la, thr)
    rows, cols = O.decidable(ref_la, thr, tol)
    assert np.array_equal(got['matches0'][rows], e['matches0'][rows])
    assert np.array_equal(got['matches1'][cols], e['matches1'][cols])
    assert np.array_equal(got['mscores0'][rows] > 0, e['mutual0'][rows])
    assert np.array_equal(got['mscores1'][cols] > 0, e['mutual1'][cols])
    for k, sel in (('mscores0', rows), ('mscores1', cols)):
        ref = e[k][sel]
        assert (np.abs(got[k][sel] - ref) <= ref * ms_tol + 1e-30).all(), k
    return int((~rows).sum() + (~cols).sum()), len(rows) + len(cols)


def _check_sinkhorn(scores, alpha, iters, thr):
    B, n, m = scores.shape
    out = SG._sinkhorn(scores.to(DEV), torch.tensor(alpha, device=DEV), iters, thr, log_assign=True)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    excluded = total = 0
    for b in range(B):
        ref, vmax = O.log_optimal_transport(scores[b].double().numpy(), alpha, iters)
        amax = max(abs(alpha), float(scores[b].abs().max()))
        bound = O.sinkhorn_bound(n, m, amax, vmax, iters)
        err = float(np.abs(got['log_assign'][b].astype(np.float64) - ref).max())
        assert err <= bound, (err, bound)
        ex, tot = _compare({k: got[k][b] for k in ('matches0', 'matches1', 'mscores0', 'mscores1')}, ref, thr,
                           2 * bound, np.expm1(bound) + 2.0 ** -21)
        excluded += ex
        total += tot
    return out, excluded / total


@pytest.mark.parametrize('n, m, B, iters, alpha, thr', [
    (300, 300, 1, 100, 1.0, 0.2),
    (257, 411, 1, 100, 1.0, 0.2),
    (411, 257, 1, 100, 1.0, 0.2),
    (1, 50, 1, 100, 1.0, 0.2),
    (60, 1, 1, 100, 1.0, 0.2),
    (1, 1, 1, 100, 1.0, 0.2),
    (120, 90, 3, 100, 1.0, 0.2),
    (200, 150, 1, 0, 1.0, 0.2),
    (200, 150, 1, 1, 1.0, 0.2),
    (180, 240, 2, 100, -2.0, 0.05),
    (180, 240, 1, 100, 3.5, 0.5),
])
def test_sinkhorn_equals_float64_oracle(n, m, B, iters, alpha, thr):
    _, frac = _check_sinkhorn(_planted_scores(n * 7 + m + B, B, n, m), alpha, iters, thr)
    if min(n, m) >= 90 and iters > 0:
        assert frac < 0.1, frac                      # the decision rule leaves most rows and columns checked


def test_sinkhorn_past_l2():
    # 48 MB of scores plus its 48 MB transposed copy: every pass reads from HBM
    _, frac = _check_sinkhorn(_planted_scores(5, 1, 4000, 3000), 1.0, 25, 0.2)
    assert frac < 0.1, frac


def test_sinkhorn_argument_checks():
    s = torch.zeros(1, 4, 5, device=DEV)
    with pytest.raises(ValueError):
        SG._sinkhorn(s, 1.0, -1, 0.2)
    with pytest.raises(ValueError):
        SG._sinkhorn(s[:, :0], 1.0, 10, 0.2)
    with pytest.raises(RuntimeError, match='match_threshold'):
        SG._sinkhorn(s, 1.0, 10, float('inf'))
    with pytest.raises(RuntimeError, match='2\\^20'):
        SG._sinkhorn(torch.zeros(1, 1, (1 << 20) + 1, device=DEV), 1.0, 1, 0.2)


def test_grid_size_and_batch_invariance():
    scores = _planted_scores(3, 3, 700, 500).to(DEV)
    alpha = torch.tensor(0.5, device=DEV)
    h = SG._lib.default_handle(DEV)
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    runs = []
    try:
        for v in (0, 1, 2, 3, 7, 114, 131):
            h.set_option('num_sms', min(v, n_sm))
            runs.append(SG._sinkhorn(scores, alpha, 100, 0.2, log_assign=True))
    finally:
        h.set_option('num_sms', 0)
    for r in runs[1:]:
        for k in r:
            assert torch.equal(r[k], runs[0][k]), k
    for b in range(3):
        single = SG._sinkhorn(scores[b:b + 1].contiguous(), alpha, 100, 0.2, log_assign=True)
        for k in single:
            assert torch.equal(single[k][0], runs[0][k][b]), (b, k)


def test_log_optimal_transport_no_host_sync():
    scores = _planted_scores(4, 1, 64, 80).to(DEV)
    alpha = torch.nn.Parameter(torch.tensor(1.0, device=DEV))
    SG.log_optimal_transport(scores, alpha, 100)                  # grow the scratch
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        la = SG.log_optimal_transport(scores, alpha, 100)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert la.shape == (1, 65, 81)
    ref, _ = O.log_optimal_transport(scores[0].double().cpu().numpy(), 1.0, 100)
    assert np.abs(la[0].cpu().double().numpy() - ref).max() < 1e-3


def _planted_data(seed, n, m, k):
    g = torch.Generator().manual_seed(seed)

    def desc(c):
        d = torch.randn(1, 256, c, generator=g)
        return d / d.norm(dim=1, keepdim=True)
    d0, d1 = desc(n), desc(m)
    pi, pj = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
    d1[0][:, pj] = d0[0][:, pi]
    data = {'image0': torch.zeros(1, 1, 120, 160), 'image1': torch.zeros(1, 1, 96, 128),
            'keypoints0': torch.stack([torch.rand(1, n, generator=g) * 159, torch.rand(1, n, generator=g) * 119], 2),
            'keypoints1': torch.stack([torch.rand(1, m, generator=g) * 127, torch.rand(1, m, generator=g) * 95], 2),
            'scores0': torch.rand(1, n, generator=g), 'scores1': torch.rand(1, m, generator=g),
            'descriptors0': d0, 'descriptors1': d1}
    return data, pi.numpy(), pj.numpy()


def test_superglue_forward_against_float64_oracle():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = O.seeded_state_dict(0, proj_gain=16.0, bin_score=1.0)
    sg = SG.SuperGlue()
    sg.load_state_dict(sd)
    sg = sg.to(DEV)
    data, pi, pj = _planted_data(2, 150, 170, 100)
    gdata = {k: v.to(DEV) for k, v in data.items()}
    sg(gdata)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = sg(gdata)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    with torch.no_grad():
        s32 = sg.score_matrix(gdata)[0].double().cpu().numpy()
    npd = O.to_numpy(sd)
    ref_s = O.scores(npd, *[data[k][0].double().numpy() for k in ('keypoints0', 'keypoints1', 'scores0', 'scores1',
                                                                      'descriptors0', 'descriptors1')],
                     (120, 160), (96, 128), sg.config['GNN_layers'], 5)
    gnn_dev = float(np.abs(s32 - ref_s).max())
    assert gnn_dev < GNN_TOL, gnn_dev
    ref_la, vmax = O.log_optimal_transport(ref_s, float(sd['bin_score']), 100)
    # a score perturbation of gnn_dev moves each half-iteration's u or v by at most gnn_dev (LSE is 1-Lipschitz), and
    # log_assign by (4 iters + 1) gnn_dev; the kernel's rounding adds its own bound
    tol = O.sinkhorn_bound(150, 170, float(np.abs(ref_s).max()) + 1, vmax, 100) + 401 * gnn_dev
    got = {'matches0': out['matches0'][0].cpu().numpy(), 'matches1': out['matches1'][0].cpu().numpy(),
           'mscores0': out['matching_scores0'][0].cpu().numpy(), 'mscores1': out['matching_scores1'][0].cpu().numpy()}
    assert out['matches0'].dtype == torch.int64 and out['matching_scores0'].dtype == torch.float32
    excluded, total = _compare(got, ref_la, 0.2, 2 * tol, np.expm1(tol) + 2.0 ** -21)
    assert excluded < 0.35 * total, (excluded, total)
    assert (got['matches0'][pi] == pj).mean() > 0.9                  # the planted pairs are found


@pytest.fixture(scope='module')
def sp_sg():
    from oracle import superpoint_oracle as SPO
    from patch2pix_b200 import superpoint as SP
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sp = SP.SuperPoint(max_keypoints=400)
    sp.load_state_dict(SPO.seeded_state_dict(0))
    sg = SG.SuperGlue({'match_threshold': 0.0})       # every mutual pair: never an empty coarse set
    sg.load_state_dict(O.seeded_state_dict(1, proj_gain=16.0))
    return sp.to(DEV), sg.to(DEV)


@pytest.fixture(scope='module')
def p2p_net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


def test_refine_matches_with_superglue(sp_sg, p2p_net, tmp_path):
    from PIL import Image
    from patch2pix_b200.eval_helper import refine_matches
    from patch2pix_b200.synth import synthetic_photo_pair
    sp, sg = sp_sg
    a, b = synthetic_photo_pair(4, (150, 203), (161, 190))
    p1, p2 = str(tmp_path / 'a.png'), str(tmp_path / 'b.png')
    Image.fromarray(a).save(p1)
    Image.fromarray(b).save(p2)
    matcher = SG.superglue_matcher(sp, sg)
    rows = []

    def recorded(g1, g2):
        r = matcher(g1, g2)
        rows.append(r)
        return r
    refined, scores, coarse = refine_matches(p1, p2, p2p_net, recorded, io_thres=0.0)
    assert len(coarse) > 0 and coarse.shape[1] == 4
    fixed, fscores, coarse2 = refine_matches(p1, p2, p2p_net, lambda g1, g2: rows[0].clone(), io_thres=0.0)
    assert np.array_equal(coarse, coarse2) and np.array_equal(refined, fixed) and np.array_equal(scores, fscores)
    assert np.isfinite(refined).all() and refined.shape == coarse.shape
    # SuperGlue's rows are integer keypoints, one-to-one
    g = rows[0].cpu().numpy()
    assert np.array_equal(g, np.round(g))
    assert len(np.unique(g[:, :2], axis=0)) == len(g) and len(np.unique(g[:, 2:], axis=0)) == len(g)


def test_eval_hpatches_with_sp_superglue_patch2pix_matcher(sp_sg, p2p_net, tmp_path):
    from patch2pix_b200 import hpatches as HP
    from patch2pix_b200 import superpoint as SP
    from patch2pix_b200.synth import synthetic_hpatches_tree
    sp, sg = sp_sg
    root = str(tmp_path / 'hp')
    os.makedirs(root)
    synthetic_hpatches_tree(root, 7, [('i_a', (200, 150)), ('v_c', (240, 176))])
    res = HP.eval_hpatches(SP.sp_patch2pix_matcher(p2p_net, sp, 0.0, 1024, sg=sg), root, lprint_=lambda s: None)
    assert res['n_pairs'] == 10
    assert not any(r.match_failed for r in res['records'])
