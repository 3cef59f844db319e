"""CPU checks of match verification: the numpy oracle of p2p_find_model (oracle/verify_oracle.py) solves noise-free
scenes exactly, draws valid samples, separates synthetic inliers from outliers and agrees with OpenCV; verify.cu
compiles for sm_90a without register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import verify_oracle as V
from patch2pix_b200.synth import synthetic_two_view


def _rows(sc):
    return np.concatenate([sc['pts1'], sc['pts2']], 1)


def test_verify_kernels_compile_without_spills(tmp_path):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'verify.cu'), '-o', str(tmp_path / 'v.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    spills, cur = {}, None
    for ln in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', ln)
        if m and cur is not None:
            spills[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    assert len(spills) == 7, sorted(spills)     # prep, round x2, select, lo x2, sampson
    assert not {k: v for k, v in spills.items() if v}, spills


def test_seven_point_reproduces_noise_free_f():
    sc = synthetic_two_view(3, 60, 0.0, 0.0)
    rows = _rows(sc)
    T = V.normalisation(rows)
    ns, ok = V.null_space(V.f7_rows(V.normalise(rows[None, :7], T)))
    assert ok[0]
    mn, okr = V.solve_f7(ns)
    Fs, okd = V.denormalise(0, mn.reshape(-1, 9), T)
    Fs = [F for F, a, b in zip(Fs, okr[0], okd) if a and b]
    assert Fs
    res = [V.errors(0, F, rows)[0].max() for F in Fs]
    F = Fs[int(np.argmin(res))]
    assert min(res) < 1e-9
    sv = np.linalg.svd(F, compute_uv=False)
    assert sv[2] < 1e-9 * sv[0] and sv[1] > 1e-6 * sv[0]
    assert min(np.abs(F - sc['F']).max(), np.abs(F + sc['F']).max()) < 1e-6


def test_dlt_reproduces_noise_free_h():
    sc = synthetic_two_view(4, 40, 0.0, 0.0, planar=True)
    rows = _rows(sc)
    T = V.normalisation(rows)
    P = V.normalise(rows[None, :4], T)
    assert V.h4_sample_ok(P)[0]
    ns, ok = V.null_space(V.h4_rows(P))
    assert ok[0]
    H, okd = V.denormalise(1, ns[:, 0], T)
    assert okd[0]
    assert V.errors(1, H[0], rows)[0].max() < 1e-9
    assert np.abs(H[0] - sc['H']).max() < 1e-9 * np.abs(sc['H']).max()
    # a sample with three collinear points yields no model
    Pc = P.copy()
    Pc[0, 2, :2] = 0.5 * (Pc[0, 0, :2] + Pc[0, 1, :2])
    assert not V.h4_sample_ok(Pc)[0]


@pytest.mark.parametrize('n', [4, 7, 8, 50, 100000])
def test_generator_never_repeats_an_index(n):
    for s in (4, 7):
        if n < s:
            continue
        idx, ok = V.draw_samples(5, np.arange(20000), n, s)
        assert idx.min() >= 0 and idx.max() < n
        srt = np.sort(idx[ok], 1)
        assert not (srt[:, 1:] == srt[:, :-1]).any()
        assert ok.mean() > (0.5 if n == s else 0.999)
    # stateless: a hypothesis' sample does not depend on which others are drawn with it
    a, _ = V.draw_samples(9, np.arange(100), 1000, 7)
    b, _ = V.draw_samples(9, np.arange(50, 60), 1000, 7)
    assert np.array_equal(a[50:60], b)


# The thresholds keep the true inliers' expected recall above 0.98: Sampson error ~ sigma^2 chi2(1), transfer error
# ~ 2 sigma^2 chi2(2) for a near-identity H.  F at 80 % outliers is not a case: there 2-3 % of uniformly random outliers
# fall inside the epipolar band of any threshold that keeps that recall, so precision stays near 0.92-0.96 whatever the
# estimator (and the fp64 oracle needs ~0.5 M hypotheses to get there, w^7 = 1.3e-5).
CASES = [('F', 0.2, 500), ('F', 0.5, 500), ('H', 0.2, 500), ('H', 0.5, 500), ('H', 0.8, 500)]
TH = {'F': 1.25, 'H': 3.0}


def _solve(kind, ratio, n, seed=0):
    sc = synthetic_two_view(seed, n, ratio, 0.5, planar=kind == 'H')
    rows = _rows(sc)
    M, mask, c = V.find_model(0 if kind == 'F' else 1, rows, TH[kind], max_iters=10000, seed=seed)
    return sc, M, mask, c


@pytest.mark.parametrize('kind, ratio, n', CASES)
def test_oracle_separates_inliers(kind, ratio, n):
    sc, M, mask, c = _solve(kind, ratio, n)
    lab = sc['inlier']
    tp = int((mask & lab).sum())
    assert M is not None and c == int(mask.sum())
    assert tp / lab.sum() >= 0.98, (tp, lab.sum())
    assert tp / mask.sum() >= 0.95, (tp, mask.sum())


@pytest.mark.parametrize('kind, ratio, n', CASES)
def test_oracle_count_matches_opencv(kind, ratio, n):
    cv2 = pytest.importorskip('cv2')
    sc, M, mask, c = _solve(kind, ratio, n)
    p1, p2 = sc['pts1'], sc['pts2']
    if kind == 'F':      # USAC_ACCURATE scores F by the Sampson error, as find_model does
        _, cm = cv2.findFundamentalMat(p1, p2, cv2.USAC_ACCURATE, TH[kind], 0.999, 10000)
    else:
        _, cm = cv2.findHomography(p1, p2, cv2.RANSAC, TH[kind], maxIters=10000, confidence=0.999)
    ref = int(cm.sum())
    assert abs(c - ref) <= 0.05 * ref, (c, ref)


def test_sampson_distance_is_the_reference_formula():
    sc = synthetic_two_view(6, 50, 0.5, 1.0)
    rows = _rows(sc)
    d = V.sampson_distance(rows, sc['F'])
    F = sc['F']
    x1 = np.c_[sc['pts1'], np.ones(50)]
    x2 = np.c_[sc['pts2'], np.ones(50)]
    l2, l1 = x1 @ F.T, x2 @ F
    ref = (np.sum(l2 * x2, 1) ** 2) / (1e-8 + l1[:, 0] ** 2 + l1[:, 1] ** 2 + l2[:, 0] ** 2 + l2[:, 1] ** 2)
    np.testing.assert_allclose(d, ref, rtol=1e-12)
