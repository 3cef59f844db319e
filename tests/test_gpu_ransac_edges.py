"""The RANSAC engine's fp32 inlier decisions (verify_common.cuh, pose.cu, abspose.cu) against float64, outside the
derived per-row bound of oracle/ransac_bound.py, on large images, hard geometries and degenerate match sets.

a. Planted near-threshold rows: scenes of low-noise inliers, about 1500 rows planted at e = th^2 (1 +- up to 2 %) and
   outliers.  After each public entry point, single and batched, every row outside the bound must be decided as fp64
   decides it under the returned model, the count must equal the mask's, and enough rows must lie within 4 bounds of
   th^2 for the check to be sharp.  No agreement with the oracle's RANSAC is needed.
b. Every slot of the first hypotheses, degenerate samples included: the GPU count of each model equals the fp64 count of
   that same model up to the rows within the bound; empty slots read -1; a non-finite model counts 0.
c. Hard geometries end to end against the oracles' find_model / find_essential / find_absolute_pose, the way
   test_gpu_verify._compare_final compares, with the near-threshold rows taken from the bound."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import abspose_oracle as AO
from oracle import degensac_oracle as DO
from oracle import pose_oracle as PO
from oracle import ransac_bound as B
from oracle import verify_oracle as VO
from patch2pix_b200 import _lib
from patch2pix_b200 import localize as L
from patch2pix_b200 import pose as PP
from patch2pix_b200 import verify as VV
from patch2pix_b200.synth import INLOC_FOCAL
from test_ransac_bound_host import abs_scene, centred, intr8, two_view, two_view_rows

pytestmark = pytest.mark.gpu

KIND = {'F': 0, 'DEGENSAC': 0, 'H': 1, 'E': 3, 'ABS': 4}
STATS = {}                  # kind -> [exempt rows, checked rows, max fp32 error / bound] over part a


# ---- calls that also return the device's inlier count --------------------------------------------------------------
def _two_view_call(which, rows, th, seed, intr=None):
    """(model or None, mask, count) of one pair through the single-pair entry point's own buffer, checked equal to the
    public single and batched calls."""
    p1, p2 = rows[:, :2].copy(), rows[:, 2:].copy()
    n = len(rows)
    dev = torch.device('cuda', torch.cuda.current_device())
    h = _lib.default_handle(dev)
    rt = torch.from_numpy(np.ascontiguousarray(rows)).to(dev)
    if which == 'E':
        out = torch.empty(PP.out_size(n), dtype=torch.float64, device=dev)
        K1 = np.array([[intr[0], 0, intr[2]], [0, intr[1], intr[3]], [0, 0, 1.0]])
        K2 = np.array([[intr[4], 0, intr[6]], [0, intr[5], intr[7]], [0, 0, 1.0]])
        PP.find_essential_into(h, rt, 4, n, None, PP.intrinsics(K1, K2), th, 0.999, 1000, seed, out)
        host = out.cpu().numpy()
        count = int(host[9:10].view(np.int32)[0])
        M, mask = PP.parse_host(host, n)[:2]
        single = PP.find_essential_matrix(p1, p2, K1, K2, th, seed=seed)
        batch = PP.find_essential_matrices([p1[:50], p1], [p2[:50], p2], [K1, K1], [K2, K2], th, seed=seed)[1]
    else:
        mid = {'F': VV.MODEL_F, 'H': VV.MODEL_H, 'DEGENSAC': VV.MODEL_F_DEGENSAC}[which]
        out = torch.empty(VV.out_size(n), dtype=torch.float64, device=dev)
        VV.find_model_into(h, mid, rt, 4, n, None, th, 0.999, 10000, seed, out)
        host = out.cpu().numpy()
        count = int(host[9:10].view(np.int32)[0])
        M, mask = VV.parse_host(host, n)
        if which == 'H':
            single = VV.find_homography(p1, p2, th, seed=seed)
            batch = VV.find_homographies([p1[:50], p1], [p2[:50], p2], th, seed=seed)[1]
        else:
            dg = which == 'DEGENSAC'
            single = VV.find_fundamental_matrix(p1, p2, th, seed=seed, degeneracy_check=dg)
            batch = VV.find_fundamental_matrices([p1[:50], p1], [p2[:50], p2], th, seed=seed, degeneracy_check=dg)[1]
    for other in (single, batch):
        assert (M is None) == (other[0] is None) and np.array_equal(mask, other[1])
        assert M is None or M.tobytes() == other[0].tobytes()
    return M, mask, count


def _abs_call(rows_list, intr_list, th, seed=0):
    """[(R, t, mask, count)] of a batch of queries through p2p_find_absolute_pose_batch (as localize.find_absolute_poses,
    keeping the counts)."""
    rows, offsets, _ = L._query_rows([r[:, :2] for r in rows_list], [r[:, 2:] for r in rows_list])
    nq, N = offsets.size - 1, int(offsets[-1])
    dev = torch.device('cuda', torch.cuda.current_device())
    intr = np.stack([L._camera(k) for k in intr_list])
    extra = np.concatenate([intr.reshape(-1), offsets.view(np.float64)])
    d = torch.from_numpy(np.concatenate([np.concatenate(rows, 0).reshape(-1), extra])).to(dev)
    rd, ex = d[:5 * N].view(N, 5), d[5 * N:]
    out = torch.empty(12 * nq + (nq + 1) // 2 + (N + 7) // 8 + 1, dtype=torch.float64, device=dev)
    base = out.data_ptr()
    L.find_absolute_pose_batch_into(_lib.default_handle(dev), rd, 5, ex[4 * nq:].view(torch.int64), offsets, None,
                                    ex.data_ptr(), float(th), None, 0.99999, 10000, seed, base,
                                    base + 8 * (12 * nq + (nq + 1) // 2), base + 96 * nq)
    host = out.cpu().numpy()
    counts = host[12 * nq:12 * nq + (nq + 1) // 2].view(np.int32)[:nq]
    masks = host[12 * nq + (nq + 1) // 2:].view(np.uint8)
    return [(host[12 * k:12 * k + 9].reshape(3, 3).copy(), host[12 * k + 9:12 * k + 12].copy(),
             masks[offsets[k]:offsets[k + 1]].astype(bool), int(counts[k])) for k in range(nq)]


# ---- the check of one final result ---------------------------------------------------------------------------------
def _check_final(kind, model, mask, count, rows, th2, intr=None, mean=None, sharp_min=20, tag=''):
    """mask == (e64 < th2) outside the bound, count == mask.sum(), and at least sharp_min rows checked within
    [1, 4] bounds of th2.  Records the exempt rows and the largest emulated fp32 error / bound."""
    assert count == int(mask.sum()), (tag, count, int(mask.sum()))
    e = B.exact_error(kind, model, rows, th2, intr, mean)
    W = B.decision_bound(kind, model, rows, th2, intr, mean)
    gap = np.abs(e - th2)
    out = gap > W
    wrong = out & (mask != (e < th2))
    assert not wrong.any(), (tag, np.nonzero(wrong)[0][:10], ((e[wrong] - th2) / W[wrong])[:10])
    sharp = int((out & (gap <= 4 * W)).sum())
    assert sharp >= sharp_min, (tag, sharp, int((~out).sum()))
    fin = np.isfinite(W) & (W > 0) & (gap < 0.5 * th2)
    ratio = max(float(np.max(np.abs(err[fin]) / W[fin], initial=0.0))
                for _, err in (B.fp32_decision(kind, model, rows, th2, f, intr, mean) for f in (False, True)))
    s = STATS.setdefault(kind, [0, 0, 0.0])
    s[0] += int((~out).sum())
    s[1] += int(out.sum())
    s[2] = max(s[2], ratio)
    return sharp


# ---- a. planted near-threshold rows -------------------------------------------------------------------------------
SIZES_A = [(640, 480, 0.0), (1600, 1200, 0.0), (4032, 3024, 0.0), (1600, 1200, 2e4)]
NOISY = (640, 480, 0.3)             # (w, h, inlier noise px): LO moves the model, no sharpness asked


def _noisy(rng, rows, lab, sigma, cols=None):
    rows = rows.copy()
    sel = lab == 0
    cols = cols or rows.shape[1]
    rows[sel, :cols] += rng.normal(0.0, sigma, (int(sel.sum()), cols))
    return rows


# H skips the offset: at H[2][2] = 1 (the kernels' normalisation) an H in those coordinates has (H x)_z < 0 over the
# whole image, so no row can pass the w > 1e-8 gate
@pytest.mark.parametrize('which, size', [(w, s) for w in ('F', 'DEGENSAC', 'H', 'E') for s in SIZES_A + ['noisy']
                                         if not (w == 'H' and s == SIZES_A[3])],
                         ids=lambda v: v if isinstance(v, str) else f'{v[0]}x{v[1]}+{int(v[2])}')
def test_planted_rows_two_view(which, size):
    """Exact inliers, planted rows mostly inside the threshold (the scene's model then keeps the most rows, so RANSAC
    returns it and the planted rows stay near th^2 under it); 'noisy': inliers with 0.3 px noise, where LO refits."""
    w, h, off = (640, 480, 0.0) if size == 'noisy' else size
    kind = KIND[which]
    rng = np.random.default_rng([kind, w, int(off), size == 'noisy'])
    th = 1.0 if kind != 1 else 2.0
    f = w * 0.9
    g = two_view(rng, w, h, f, f * 1.15 if which == 'E' else None, aspect=(1.0, 1.0), offset=off, plane=kind == 1)
    model = {0: g['F'], 1: g['H'], 3: g['E']}[kind]
    rows, lab = two_view_rows(rng, kind, g, model, 1000, 1500, 300, th, mirror=True, inside=0.8)
    if size == 'noisy':
        rows = _noisy(rng, rows, lab, NOISY[2])
    M, mask, count = _two_view_call(which, rows, th, seed=3, intr=intr8(g))
    assert M is not None
    sharp = 0 if size == 'noisy' else 20
    if kind == 3:
        _check_final(3, M, mask, count, PO.to_camera(rows, intr8(g)), PO.threshold(th, intr8(g)) ** 2, sharp_min=sharp,
                     tag=which)
    else:
        _check_final(kind, M, mask, count, rows, th * th, sharp_min=sharp, tag=which)
    assert (mask & (lab == 0)).mean() > 0.9 * (lab == 0).mean()


@pytest.mark.parametrize('cam', ['1024x768', 'fx!=fy', 'inloc', 'offset', 'noisy'])
def test_planted_rows_absolute_pose(cam):
    rng = np.random.default_rng([4, len(cam)])
    w, h, fx, fy, off = {'1024x768': (1024, 768, 900.0, 900.0, 0.0), 'fx!=fy': (1600, 1200, 1400.0, 1550.0, 0.0),
                         'inloc': (4032, 3024, INLOC_FOCAL, INLOC_FOCAL, 0.0),
                         'offset': (1600, 1200, 1500.0, 1500.0, 2e4), 'noisy': (1024, 768, 900.0, 950.0, 0.0)}[cam]
    th = 4.0 if w < 2000 else 2.0
    rows, lab, intr, _, _ = abs_scene(rng, w, h, fx, fy, n_in=1000, n_plant=1500, n_out=300, th=th, offset=off,
                                      mirror=True, inside=0.8)
    if cam == 'noisy':
        rows = _noisy(rng, rows, lab, 1.0, cols=2)
    res = _abs_call([rows[:60], rows], [intr, intr], th)
    R, t, mask, count = res[1]
    one = L.find_absolute_pose(rows[:, :2], rows[:, 2:], intr, th)
    assert np.array_equal(one[0], R) and np.array_equal(one[1], t) and np.array_equal(one[2], mask)
    mean = rows[:, 2:5].mean(0)
    _check_final(4, centred(R, t, mean), mask, count, rows, th * th, intr, mean, sharp_min=0 if cam == 'noisy' else 20,
                 tag=cam)
    assert (mask & (lab == 0)).mean() > 0.9 * (lab == 0).mean()


# ---- b. every hypothesis slot ---------------------------------------------------------------------------------------
def _base(kind, rng, n_in=150, n_plant=300, n_out=150):
    g = two_view(rng, 640, 480, 560.0, 600.0 if kind == 3 else None, plane=kind == 1)
    model = {0: g['F'], 1: g['H'], 3: g['E']}[kind]
    rows, lab = two_view_rows(rng, kind, g, model, n_in, n_plant, n_out, 1.0 if kind != 1 else 2.0)
    return g, rows, lab


def _grazing(rng):
    """An H at a grazing angle: its horizon (H x)_z = 0 crosses the image; rows on both sides, x2 = pi(H x1) + small
    offsets where (H x1)_z > 0 and random elsewhere."""
    H = np.array([[1.0, 0.1, 5.0], [0.05, 1.2, -3.0], [1.0 / 320, 0.4 / 240, -1.2]])
    x1 = rng.uniform([0, 0], [640, 480], (600, 2))
    q = np.concatenate([x1, np.ones((600, 1))], 1) @ H.T
    with np.errstate(divide='ignore'):
        x2 = q[:, :2] / q[:, 2:3] + rng.normal(0.0, 1.0, (600, 2))
    bad = (q[:, 2] <= 1e-3) | ~np.all(np.abs(x2) < 1e5, 1)
    x2[bad] = rng.uniform([0, 0], [640, 480], (int(bad.sum()), 2))
    return np.concatenate([x1, x2], 1)


def _degenerate_sets(kind, rng):
    g, rows, lab = _base(kind, rng)
    s = {0: 7, 1: 4, 3: 5}[kind]
    sets = {'dup2': np.repeat(rows, 2, 0), 'dup3': np.tile(rows, (3, 1)),
            'identical': np.repeat(rows[lab == 0][:1], 200, 0),
            'ksample': rows[lab == 0][:s], 'ksample+1': rows[lab == 0][:s + 1],
            'outliers95': np.concatenate([rows[lab == 0][:20], rng.uniform(0, 640, (380, 4))]),
            'outliers': rng.uniform([0, 0, 0, 0], [640, 480, 640, 480], (400, 4))}
    col = rows.copy()
    tt = rng.uniform(-1, 1, len(col))
    col[:, 0], col[:, 1] = 320 + 250 * tt, 240 + 120 * tt + rng.normal(0, 1e-9, len(col))
    sets['collinear'] = col
    if kind == 1:
        sets['grazing'] = _grazing(rng)
    return g, sets


def _check_slots(kind, models, counts, rows, th2, intr=None, mean=None, tag=''):
    """Every slot: -1 and zeros without a model; with one, lo <= count <= lo + near, 0 for a non-finite model."""
    n_models = 0
    for i in range(len(counts)):
        m, c = models[i], int(counts[i])
        if c < 0:
            assert c == -1 and not np.any(m), (tag, i, c)
            continue
        n_models += 1
        if not np.all(np.isfinite(m)):
            assert c == 0, (tag, i, c)
            continue
        e = B.exact_error(kind, m, rows, th2, intr, mean)
        W = B.decision_bound(kind, m, rows, th2, intr, mean)
        near = ~(np.abs(e - th2) > W)
        lo = int(((e < th2) & ~near).sum())
        assert lo <= c <= lo + int(near.sum()), (tag, i, c, lo, int(near.sum()))
    return n_models


@pytest.mark.parametrize('which', ['F', 'H', 'E'])
def test_hypothesis_counts_on_degenerate_sets(which):
    kind = KIND[which]
    g, sets = _degenerate_sets(kind, np.random.default_rng(40 + kind))
    total = 0
    for name, rows in sets.items():
        if kind == 3:
            K1, K2 = g['K1'], g['K2']
            gm, gc = PP.first_essential_hypotheses(rows[:, :2], rows[:, 2:], K1, K2, 1.0, 256, seed=5)
            total += _check_slots(3, gm, gc, PO.to_camera(rows, intr8(g)), PO.threshold(1.0, intr8(g)) ** 2,
                                  tag=name)
        else:
            th = 1.0 if kind == 0 else 2.0
            gm, gc = VV.first_hypotheses(kind, rows[:, :2], rows[:, 2:], th, 1024, seed=5)
            total += _check_slots(kind, gm, gc, rows, th * th, tag=name)
    assert total > 500, total


def test_absolute_pose_hypothesis_counts_on_degenerate_sets():
    rng = np.random.default_rng(44)
    rows, lab, intr, R, t = abs_scene(rng, 1024, 768, 900.0, 950.0, n_in=150, n_plant=300, n_out=150, th=4.0)
    inl = rows[lab == 0]
    col = rows.copy()
    tt = rng.uniform(-1, 1, len(col))
    col[:, 2:5] = inl[0, 2:5] + tt[:, None] * (inl[1, 2:5] - inl[0, 2:5])
    behind = rows.copy()
    behind[::2, 2:5] = 2 * (-R.T @ t) - behind[::2, 2:5]              # mirrored through the camera centre
    sets = {'dup2': np.repeat(rows, 2, 0), 'dup3': np.tile(rows, (3, 1)), 'identical': np.repeat(inl[:1], 200, 0),
            'ksample+1': inl[:4], 'ksample+2': inl[:5], 'collinear': col, 'behind': behind,
            'outliers95': np.concatenate([inl[:20], rows[lab == 2][:150], rows[lab == 2][:150] * [1, 1, 1.01, 1, 1]]),
            'outliers': rows[lab == 2]}
    with pytest.raises(RuntimeError, match='fewer than 4 rows'):         # kSample = 3 rows: refused, no round runs
        L.first_absolute_pose_hypotheses(inl[:3, :2], inl[:3, 2:], intr, 4.0, 16, seed=5)
    total = 0
    for name, r in sets.items():
        gm, gc = L.first_absolute_pose_hypotheses(r[:, :2], r[:, 2:], intr, 4.0, 512, seed=5)
        total += _check_slots(4, gm, gc, r, 16.0, intr, r[:, 2:5].mean(0), tag=name)
    assert total > 300, total


# ---- c. hard geometries end to end against the oracles --------------------------------------------------------------
def _compare(kind, rows, gmask, th, oracle, th2, intr=None):
    """GPU mask against the oracle's outside the bound under the oracle's model, when the oracle's winning margin
    exceeds the exempt rows.  Returns whether the comparison applied."""
    tr = {}
    M, omask, _ = oracle(tr)
    assert M is not None
    if kind == 4:
        mean = rows[:, 2:5].mean(0)
        R = M[:9].reshape(3, 3)
        Mc, r, extra = np.concatenate([M[:9], M[9:] + R @ mean]), rows, dict(intr=intr, mean=mean)
    elif kind == 3:
        Mc, r, extra = M, PO.to_camera(rows, intr), {}
    else:
        Mc, r, extra = M, rows, {}
    e = B.exact_error(kind, Mc, r, th2, **extra)
    near = ~(np.abs(e - th2) > B.decision_bound(kind, Mc, r, th2, **extra))
    if tr['margin'] <= int(near.sum()):
        return False
    diff = gmask != omask
    assert not (diff & ~near).any(), (np.nonzero(diff & ~near)[0][:10], tr)
    return True


GEOMETRIES = ['forward', 'rotation', 'planar', 'narrow', 'dup2', 'collinear']


def _hard_scene(geo, kind, seed):
    rng = np.random.default_rng([seed, kind, len(geo)])
    w, h, f = (1600, 1200, 1e4) if geo == 'narrow' else (640, 480, 560.0)
    g = two_view(rng, w, h, f, f * 1.1 if kind == 3 else None, motion=geo if geo in ('forward', 'rotation') else 'side',
                 plane=geo == 'planar' or kind == 1)
    model = {0: g['F'], 1: g['H'], 3: g['E']}[kind]
    # narrow FOV: a sideways baseline moves most points 10^3 px, so image 2 is taken 3 times as large
    rows, lab = two_view_rows(rng, kind, g, model, 500, 300, 400, 1.0 if kind != 1 else 2.0,
                              margin=1.0 if geo == 'narrow' else 0.0)
    rows = _noisy(rng, rows, lab, 0.3)
    if geo == 'dup2':
        rows = np.repeat(rows, 2, 0)
    elif geo == 'collinear':
        rows[:100, 0] = 100 + rows[:100, 1] * 0.5
    return g, rows


@pytest.mark.parametrize('which', ['F', 'DEGENSAC', 'H', 'E'])
def test_hard_geometries_match_oracle(which):
    kind = KIND[which]
    applied = cases = 0
    th = 1.0 if kind != 1 else 2.0
    for geo in (GEOMETRIES if kind != 1 else ['planar', 'narrow', 'dup2', 'collinear']):
        g, rows = _hard_scene(geo, kind, 1)
        p1, p2 = rows[:, :2], rows[:, 2:]
        if which == 'E':
            gm, mask = PP.find_essential_matrix(p1, p2, g['K1'], g['K2'], th, seed=4)
            oracle = lambda tr: PO.find_essential(rows, intr8(g), th, seed=4, trace=tr)  # noqa: E731
            th2 = PO.threshold(th, intr8(g)) ** 2
            a = _compare(3, rows, mask, th, oracle, th2, intr8(g))
        else:
            if which == 'H':
                gm, mask = VV.find_homography(p1, p2, th, seed=4)
                oracle = lambda tr: VO.find_model(1, rows, th, seed=4, trace=tr)  # noqa: E731
            elif which == 'F':
                gm, mask = VV.find_fundamental_matrix(p1, p2, th, seed=4)
                oracle = lambda tr: VO.find_model(0, rows, th, seed=4, trace=tr)  # noqa: E731
            else:
                gm, mask = VV.find_fundamental_matrix(p1, p2, th, seed=4, degeneracy_check=True)
                oracle = lambda tr: DO.find_model(rows, th, seed=4, trace=tr)  # noqa: E731
            a = _compare(kind, rows, mask, th, oracle, th * th)
        cases += 1
        applied += a
    assert applied >= cases // 2 + 1, (applied, cases)


def test_hard_absolute_poses_match_oracle_batch_and_repeat():
    scenes = []
    for k, (w, h, fx, fy) in enumerate([(1024, 768, 900.0, 900.0), (1600, 1200, 1e4, 1e4),
                                         (4032, 3024, INLOC_FOCAL, INLOC_FOCAL * 1.02), (1024, 768, 700.0, 760.0)]):
        rng = np.random.default_rng([50, k])
        rows, lab, intr, _, _ = abs_scene(rng, w, h, fx, fy, n_in=500, n_plant=200, n_out=400, th=4.0)
        rows[lab == 0, :2] += rng.normal(0.0, 0.5, (int((lab == 0).sum()), 2))
        if k == 3:
            rows = np.repeat(rows, 2, 0)
        scenes.append((rows, intr))
    batch = L.find_absolute_poses([r[:, :2] for r, _ in scenes], [r[:, 2:] for r, _ in scenes],
                                  [i for _, i in scenes], 4.0, seed=4)
    applied = 0
    for (rows, intr), (R, t, mask) in zip(scenes, batch):
        one = L.find_absolute_pose(rows[:, :2], rows[:, 2:], intr, 4.0, seed=4)
        two = L.find_absolute_pose(rows[:, :2], rows[:, 2:], intr, 4.0, seed=4)
        for x, y, z in zip(one, two, (R, t, mask)):
            assert x.tobytes() == y.tobytes() == z.tobytes()
        oracle = lambda tr: AO.find_absolute_pose(rows, intr, 4.0, seed=4, trace=tr)  # noqa: E731
        applied += _compare(4, rows, mask, 4.0, oracle, 16.0, intr)
    assert applied >= 3, applied


def test_hard_two_view_batch_equals_single_and_repeats():
    scenes = [_hard_scene(geo, 0, 2) for geo in GEOMETRIES]
    p1, p2 = [r[:, :2] for _, r in scenes], [r[:, 2:] for _, r in scenes]
    K1, K2 = [g['K1'] for g, _ in scenes], [g['K2'] for g, _ in scenes]
    for fn, single in ((lambda: VV.find_fundamental_matrices(p1, p2, 1.0, seed=6),
                        lambda k: VV.find_fundamental_matrix(p1[k], p2[k], 1.0, seed=6)),
                       (lambda: VV.find_fundamental_matrices(p1, p2, 1.0, seed=6, degeneracy_check=True),
                        lambda k: VV.find_fundamental_matrix(p1[k], p2[k], 1.0, seed=6, degeneracy_check=True)),
                       (lambda: VV.find_homographies(p1, p2, 2.0, seed=6),
                        lambda k: VV.find_homography(p1[k], p2[k], 2.0, seed=6)),
                       (lambda: PP.find_essential_matrices(p1, p2, K1, K2, 1.0, seed=6),
                        lambda k: PP.find_essential_matrix(p1[k], p2[k], K1[k], K2[k], 1.0, seed=6))):
        a, b = fn(), fn()
        for k in range(len(scenes)):
            s = single(k)
            for x, y, z in zip(a[k], b[k], s):
                assert (x is None) == (y is None) == (z is None)
                if x is not None:
                    assert x.tobytes() == y.tobytes() == z.tobytes(), k


def test_report():
    """The exempt-row counts and the largest emulated fp32 error / bound of part a, per kind (run with -s)."""
    for kind, (ex, ch, r) in sorted(STATS.items()):
        print(f'kind {kind}: {ex} exempt rows, {ch} checked, max fp32 error / bound {r:.3f}')
    assert all(r <= 1.0 for _, _, r in STATS.values())
