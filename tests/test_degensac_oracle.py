"""CPU checks of F RANSAC with the DEGENSAC degeneracy check (model 2 of p2p_find_model): its numpy oracle
(oracle/degensac_oracle.py) is exact on noise-free scenes, recovers the off-plane geometry of dominant-plane scenes that
plain F RANSAC loses, costs nothing on general scenes and agrees with OpenCV; degensac.cu compiles for sm_90a without
register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import degensac_oracle as D
from oracle import verify_oracle as V
from patch2pix_b200.synth import OFF_PLANE, PLANE, synthetic_dominant_plane, synthetic_two_view


def _rows(sc):
    return np.concatenate([sc['pts1'], sc['pts2']], 1)


def test_degensac_kernels_compile_without_spills(tmp_path):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'degensac.cu'), '-o', str(tmp_path / 'd.o')]
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
    assert len(spills) == 9, sorted(spills)     # prep, round F / parallax, degen, select, plane, parallax select, lo, hook
    assert not {k: v for k, v in spills.items() if v}, spills


def test_dominant_plane_scene_shares_one_camera_pair():
    sc = synthetic_dominant_plane(3, 400, 0.3, 0.2, 0.0)
    rows = _rows(sc)
    lab = sc['label']
    assert (lab == PLANE).sum() == 224 and (lab == OFF_PLANE).sum() == 56 and not sc['inlier'][lab == 2].any()
    assert V.errors(0, sc['F'], rows[sc['inlier']])[0].max() < 1e-12
    assert V.errors(1, sc['H'], rows[lab == PLANE])[0].max() < 1e-12
    assert V.errors(1, sc['H'], rows[lab == OFF_PLANE])[0].min() > 1e-2
    ref = synthetic_two_view(3, 400, 0.3, 0.0)                  # the general scene builder is untouched
    assert np.array_equal(ref['F'], sc['F'])


def test_induced_homography_is_the_plane():
    sc = synthetic_dominant_plane(4, 300, 0.0, 0.2, 0.0)
    rows = _rows(sc)[sc['label'] == PLANE]
    F = sc['F']
    for k in range(5):
        H = D.induced_homography(F, rows[3 * k:3 * k + 3])
        assert H is not None
        H = H / H[2, 2]
        assert np.abs(H - sc['H']).max() < 1e-6 * np.abs(sc['H']).max()
        S = F.T @ H
        assert np.abs(S + S.T).max() < 1e-12 * np.abs(S).max()
    # collinear points in image 1 give no H
    p = rows[:3].copy()
    p[2, :2] = 0.5 * (p[0, :2] + p[1, :2])
    assert D.induced_homography(F, p) is None


def test_degeneracy_test_on_noise_free_samples():
    sc = synthetic_dominant_plane(5, 400, 0.0, 0.5, 0.0)
    rows = _rows(sc)
    T = V.normalisation(rows)
    plane, off = rows[sc['label'] == PLANE], rows[sc['label'] == OFF_PLANE]
    th2 = 4.0
    for order in (np.arange(7), np.array([5, 0, 1, 6, 2, 3, 4]), np.array([0, 5, 1, 2, 6, 3, 4])):
        sample = np.concatenate([plane[:5], off[:2]])[order]          # 5 coplanar points, anywhere in the sample
        k, H = D.degeneracy(sc['F'], sample, T, th2)
        assert k >= 0 and (V.errors(1, H, plane[:5])[0] < th2).all()
        if k == 0 and (order[:3] < 5).all():            # the first triplet is coplanar: its H is the plane's
            assert np.abs(H - sc['H']).max() < 1e-6 * np.abs(sc['H']).max()
    for s in range(5):
        assert D.degeneracy(sc['F'], off[7 * s:7 * s + 7], T, th2) == (-1, None)   # 7 points in general position
    # two off-plane points and the true H give the true F
    far = off[V.errors(1, sc['H'], off)[0] > 100.0]                 # clear parallax
    F, ok = D.parallax_hypotheses(far[:2], sc['H'], np.arange(4), 0, th2)
    assert ok.all()
    for f in F:
        assert min(np.abs(f - sc['F']).max(), np.abs(f + sc['F']).max()) < 1e-9


def _dominant(seed):
    sc = synthetic_dominant_plane(seed, 1000, 0.3, 0.08, 0.5)
    return sc, _rows(sc)


def test_recovers_off_plane_inliers_on_dominant_plane_scenes():
    """Measured: model 2 reaches a median off-plane recall of 0.95 with no scene below 0.875; model 0 (plain F RANSAC +
    LO) 0.58 with 15 / 20 scenes below 0.8."""
    rec, rec0 = [], []
    for seed in range(20):
        sc, rows = _dominant(seed)
        off = sc['label'] == OFF_PLANE
        F, mask, c = D.find_model(rows, 1.0)
        assert F is not None and c == int(mask.sum())
        assert mask[sc['label'] == PLANE].mean() >= 0.9
        rec.append(mask[off].mean())
        rec0.append(V.find_model(0, rows, 1.0)[1][off].mean())
    assert np.median(rec) >= 0.9 and min(rec) >= 0.8, rec
    assert np.median(rec0) < 0.8                   # the scenes do defeat plain RANSAC


def test_costs_nothing_on_general_scenes():
    """General scenes (50 % outliers): the degeneracy test rarely fires, and a parallax model is only adopted with more
    support.  Such an adoption raises the inlier ratio the stopping bound reads, so later rounds may not run and LO may
    end a little lower: measured over these 20 scenes, the mean count is 0.03 % below model 0's and the worst scene
    1.03 % below."""
    c0, c2 = [], []
    for seed in range(20):
        sc = synthetic_two_view(seed, 1000, 0.5, 0.5)
        rows = _rows(sc)
        c0.append(V.find_model(0, rows, 1.0)[2])
        c2.append(D.find_model(rows, 1.0)[2])
    c0, c2 = np.array(c0), np.array(c2)
    assert c2.mean() >= 0.999 * c0.mean(), (c0, c2)
    assert (c2 >= 0.985 * c0).all(), (c0, c2)


def test_count_matches_opencv_on_dominant_plane_scenes():
    cv2 = pytest.importorskip('cv2')
    ours, ref = [], []
    for seed in range(20):
        sc, rows = _dominant(seed)
        ours.append(D.find_model(rows, 1.0)[2])
        _, cm = cv2.findFundamentalMat(sc['pts1'], sc['pts2'], cv2.USAC_ACCURATE, 1.0, 0.999, 10000)
        ref.append(int(cm.sum()))
    assert np.mean(ours) >= 0.97 * np.mean(ref), (ours, ref)
