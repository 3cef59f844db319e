"""CPU checks of relative pose: the numpy oracle of p2p_find_essential / p2p_recover_pose (oracle/pose_oracle.py) against
OpenCV's 5-point solver, RANSAC and recoverPose on synthetic scenes; the host helpers of the reference's pose evaluation;
pose.cu compiles for sm_90a without register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import pose_oracle as P
from oracle import verify_oracle as V
from patch2pix_b200 import pose as PP
from patch2pix_b200.synth import synthetic_two_view

INTR = [500.0, 500.0, 320.0, 240.0, 500.0, 500.0, 320.0, 240.0]     # synthetic_two_view's cameras


def _rows(sc):
    return np.concatenate([sc['pts1'], sc['pts2']], 1)


def _canon(M):
    M = np.asarray(M, dtype=np.float64).reshape(9)
    M = M / np.linalg.norm(M)
    return M * np.sign(M[np.argmax(np.abs(M))])


def _angle(R1, R2):
    return np.degrees(np.arccos(np.clip((np.trace(R1.T @ R2) - 1) / 2, -1, 1)))


def _t_angle(t, t_gt):
    return np.degrees(np.arccos(np.clip(np.dot(np.ravel(t), t_gt / np.linalg.norm(t_gt)), -1, 1)))


def test_pose_kernels_compile_without_spills(tmp_path):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'pose.cu'), '-o', str(tmp_path / 'p.o')]
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
    assert len(spills) == 7, sorted(spills)     # prep, round, select, lo, decompose, count, pose select
    assert not {k: v for k, v in spills.items() if v}, spills


def _residual(E):
    """Largest violation of det E = 0 and 2 E E^T E - tr(E E^T) E = 0 at unit Frobenius norm."""
    E = np.asarray(E, dtype=np.float64).reshape(3, 3)
    E = E / np.linalg.norm(E)
    return max(abs(np.linalg.det(E)), np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max())


def test_five_point_solutions_match_opencv():
    cv2 = pytest.importorskip('cv2')
    sc = synthetic_two_view(3, 300, 0.0, 0.0)
    cam = P.to_camera(_rows(sc), INTR)
    idx = np.arange(300).reshape(60, 5)
    models, valid = P.solve_e5(cam[idx])
    t = sc['t']
    truth = _canon(np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ sc['R'])
    compared = 0
    for s in range(len(idx)):
        ours = [models[s, k] for k in range(P.SLOTS) if valid[s, k]]
        Ec, _ = cv2.findEssentialMat(sc['pts1'][idx[s]], sc['pts2'][idx[s]], sc['K1'], cv2.RANSAC, 0.999, 1.0)
        theirs = [Ec[3 * i:3 * i + 3] for i in range(Ec.shape[0] // 3)]       # 5 points: every solution, stacked
        assert len(ours) == len(theirs), (s, len(ours), len(theirs))
        assert min(np.abs(_canon(E) - truth).max() for E in ours) < 1e-8, s
        # Both solvers lose digits on roots that nearly coincide; the comparison holds where both sets satisfy the
        # cubic constraints to 1e-11 (the solvers then agree to ~1e-12): 41 of these 60 samples.
        if max(_residual(E) for E in ours + theirs) > 1e-11:
            continue
        compared += 1
        for E in ours:
            assert min(np.abs(_canon(E) - _canon(F)).max() for F in theirs) < 1e-8, s
    assert compared >= 35, compared


@pytest.mark.parametrize('n', [5, 6, 50, 100000])
def test_generator_never_repeats_an_index_for_five_point_samples(n):
    idx, ok = V.draw_samples(11, np.arange(20000), n, P.SAMPLE)
    assert idx.min() >= 0 and idx.max() < n
    srt = np.sort(idx[ok], 1)
    assert not (srt[:, 1:] == srt[:, :-1]).any()
    assert ok.mean() > (0.5 if n == P.SAMPLE else 0.999)


@pytest.mark.parametrize('seed, ratio', [(0, 0.2), (1, 0.5), (2, 0.7)])
def test_recover_pose_matches_opencv(seed, ratio):
    cv2 = pytest.importorskip('cv2')
    sc = synthetic_two_view(seed, 400, ratio, 0.5)
    rows = _rows(sc)
    E, mask, _ = P.find_essential(rows, INTR, 1.5, seed=seed)
    n, R, t, good = P.recover_pose(E, rows, INTR, mask)
    nc, Rc, tc, mc = cv2.recoverPose(E, sc['pts1'], sc['pts2'], sc['K1'], mask=mask.astype(np.uint8).copy())
    assert n == nc and np.array_equal(good, mc.ravel() > 0)
    assert np.abs(R - Rc).max() < 1e-9 and np.abs(t - tc.ravel()).max() < 1e-9
    assert not (good & ~mask).any()
    # a zero E: no pose
    n0, R0, t0, g0 = P.recover_pose(np.zeros((3, 3)), rows, INTR, mask)
    assert n0 == 0 and not R0.any() and not t0.any() and not g0.any()


# Threshold 1.5 px at sigma = 0.5 px per coordinate: the Sampson error of a true correspondence is ~ sigma^2 chi2(1), so
# the true E keeps P(chi2(1) < 9) = 0.997 of the inliers; an estimated E keeps a few percent fewer at 70 % outliers
# (0.96-0.98 measured), hence recall >= 0.95.  A uniformly random outlier falls inside the +-1.5 px epipolar band with
# probability ~ 3 px * 600 px / (640 * 480 px^2) ~ 0.6 %: at 70 % outliers ~2 of 350 against ~145 inliers, hence
# precision >= 0.95.  Rotation and translation-direction errors were at most 0.53 and 2.84 degrees over the seeds 0-3
# of these scenes (500 rows); the bounds are 1 and 4 degrees.
E_CASES = [(0.2, 0), (0.5, 0), (0.7, 1)]
E_TH = 1.5


def _solve(ratio, seed):
    sc = synthetic_two_view(seed, 500, ratio, 0.5)
    E, mask, c = P.find_essential(_rows(sc), INTR, E_TH, max_iters=5000, seed=seed)
    return sc, E, mask, c


@pytest.mark.parametrize('ratio, seed', E_CASES)
def test_oracle_essential_separates_inliers_and_recovers_the_pose(ratio, seed):
    sc, E, mask, c = _solve(ratio, seed)
    lab = sc['inlier']
    tp = int((mask & lab).sum())
    assert E is not None and c == int(mask.sum())
    assert tp / lab.sum() >= 0.95, (tp, lab.sum())
    assert tp / mask.sum() >= 0.95, (tp, mask.sum())
    sv = np.linalg.svd(E, compute_uv=False)
    assert abs(np.linalg.norm(E) - 1) < 1e-12 and abs(sv[0] - sv[1]) < 1e-12 and sv[2] < 1e-12
    _, R, t, _ = P.recover_pose(E, _rows(sc), INTR, mask)
    assert _angle(R, sc['R']) < 1.0 and _t_angle(t, sc['t']) < 4.0


@pytest.mark.parametrize('ratio, seed', E_CASES)
def test_oracle_essential_count_matches_opencv(ratio, seed):
    cv2 = pytest.importorskip('cv2')
    sc, E, mask, c = _solve(ratio, seed)
    # USAC_ACCURATE refits on the inliers as find_essential does; plain RANSAC keeps the best minimal-sample model
    _, cm = cv2.findEssentialMat(sc['pts1'], sc['pts2'], sc['K1'], cv2.USAC_ACCURATE, 0.999, E_TH, maxIters=5000)
    ref = int(cm.sum())
    assert abs(c - ref) <= 0.05 * ref, (c, ref)


def test_quaternion_helpers():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(0)
    for _ in range(20):
        v = rng.normal(size=3)
        R, _ = cv2.Rodrigues(v)
        q = PP.mat2quat(R)
        th = np.linalg.norm(v)
        ref = np.array([np.cos(th / 2), *(np.sin(th / 2) * v / th)])
        assert q[0] >= 0 and (np.allclose(q, ref, atol=1e-12) or np.allclose(q, -ref, atol=1e-12))
        assert np.allclose(PP.quat2mat(q), R, atol=1e-12)
        assert np.allclose(PP.quat2mat(-q), R, atol=1e-12)
    assert np.array_equal(PP.quat2mat([0, 0, 0, 0]), np.eye(3))


def test_pose_helpers_are_consistent_with_the_synthetic_scene():
    sc = synthetic_two_view(4, 50, 0.0, 0.0, focal2=650.0)
    F = PP.pose2fund(sc['K1'], sc['K2'], sc['R'], sc['t'])
    F = F / np.linalg.norm(F)
    assert min(np.abs(F - sc['F']).max(), np.abs(F + sc['F']).max()) < 1e-9
    # absolute poses (world -> camera: X_cam = R_i (X - c_i)) of the scene's cameras give back its relative pose
    rng = np.random.default_rng(1)
    R1, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    R1 *= np.sign(np.linalg.det(R1))
    c1 = rng.normal(size=3)
    R2 = sc['R'] @ R1
    c2 = c1 - R2.T @ sc['t']
    t12, q12 = PP.abs2relapose(c1, c2, PP.mat2quat(R1), PP.mat2quat(R2))
    assert np.allclose(t12, sc['t'], atol=1e-12) and np.allclose(PP.quat2mat(q12), sc['R'], atol=1e-12)


def test_angle_errors_on_constructed_cases():
    assert PP.cal_vec_angle_error(np.array([1.0, 0, 0]), np.array([0, 2.0, 0])) == pytest.approx(90.0)
    assert PP.cal_vec_angle_error(np.array([1.0, 0, 0]), np.array([-3.0, 0, 0])) == pytest.approx(180.0)
    assert PP.cal_vec_angle_error(np.array([1.0, 1, 0]), np.array([1.0, 0, 0])) == pytest.approx(45.0)
    q = np.array([1.0, 0, 0, 0])
    th = np.radians(30)
    qz = np.array([np.cos(th / 2), 0, 0, np.sin(th / 2)])
    assert PP.cal_quat_angle_error(q, qz) == pytest.approx(30.0)
    assert PP.cal_quat_angle_error(q, -qz) == pytest.approx(30.0)        # q and -q are the same rotation
    # the reference's formula: arccos of a dot product one ulp-ish below 1 after the eps normalisation, ~2e-5 degrees
    assert PP.cal_quat_angle_error(qz, qz) == pytest.approx(0.0, abs=1e-4)
