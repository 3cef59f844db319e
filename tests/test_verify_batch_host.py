"""Argument checks of the batched verification and pose functions: every one raises before any CUDA work, so these run
without a GPU."""
import numpy as np
import pytest
import torch

from patch2pix_b200 import pose as P
from patch2pix_b200 import verify as V

K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])


def _pts(n, seed=0):
    return np.random.default_rng(seed).uniform(0, 400, (n, 2))


@pytest.fixture(autouse=True)
def no_cuda(monkeypatch):
    """Any CUDA call fails the test: the checks must come first."""
    def boom(*a, **k):
        raise AssertionError('CUDA was touched before the arguments were checked')
    monkeypatch.setattr(torch.cuda, 'current_device', boom)
    monkeypatch.setattr(torch.Tensor, 'to', boom)


def test_mismatched_list_lengths():
    with pytest.raises(ValueError, match='same length'):
        V.find_fundamental_matrices([_pts(9)], [_pts(9), _pts(9)], 1.0)
    with pytest.raises(ValueError, match='same length'):
        V.find_homographies([_pts(9)] * 3, [_pts(9)] * 2, 2.0)
    with pytest.raises(ValueError, match='same length'):
        P.find_essential_matrices([_pts(9)], [], [K], [K], 1.0)


def test_bad_shapes():
    with pytest.raises(ValueError, match='pair 1'):
        V.find_fundamental_matrices([_pts(9), _pts(9)], [_pts(9), _pts(8)], 1.0)
    with pytest.raises(ValueError):
        V.find_homographies([np.zeros(7)], [np.zeros(7)], 2.0)          # 3.5 points
    with pytest.raises(TypeError, match='list'):
        V.find_fundamental_matrices(_pts(9), _pts(9), 1.0)            # an array, not a list of arrays
    with pytest.raises(ValueError, match='pair 0'):
        P.matches2relapose_batch([np.zeros((5, 3))], [K], [K])
    with pytest.raises(ValueError, match='pair 1: E'):
        P.recover_poses([np.eye(3), np.eye(2)], [_pts(9)] * 2, [_pts(9)] * 2, [K] * 2, [K] * 2)
    with pytest.raises(ValueError, match='pair 0: mask'):
        P.recover_poses([np.eye(3)], [_pts(9)], [_pts(9)], [K], [K], [np.ones(8)])


def test_intrinsics_lists():
    with pytest.raises(ValueError, match='one matrix per pair'):
        P.find_essential_matrices([_pts(9)] * 2, [_pts(9)] * 2, [K], [K, K], 1.0)
    with pytest.raises(ValueError, match='one matrix per pair'):
        P.matches2relapose_degensac_batch([np.zeros((9, 4))] * 2, [K] * 3, [K] * 2)
    with pytest.raises(ValueError, match='one matrix per pair'):
        P.recover_poses([np.eye(3)], [_pts(9)], [_pts(9)], [], [K])
    with pytest.raises(ValueError, match='pair 1: intrinsics'):
        P.find_essential_matrices([_pts(9)] * 2, [_pts(9)] * 2, [K, np.eye(2)], [K, K], 1.0)
    bad = K.copy()
    bad[0, 0] = -1.0                  # the reference cameras use K[0, 0] on both axes
    with pytest.raises(ValueError, match='positive focal'):
        P.matches2relapose_batch([np.zeros((9, 4))], [bad], [K])
