"""The CPU restatement of SuperPoint + nearest-neighbour matching (oracle/superpoint_oracle.py) on hand-built cases,
and the host side of patch2pix_b200/superpoint.py (state_dict names, argument checks)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import superpoint_oracle as O


def _torch_nms(s, r):
    """The max-pool NMS written with torch's max_pool2d (padding -inf), as SuperGlue publishes it."""
    s = torch.as_tensor(s)[None, None]

    def mp(x):
        return F.max_pool2d(x, 2 * r + 1, 1, r)
    M = s == mp(s)
    for _ in range(2):
        S = mp(M.float()) > 0
        s2 = torch.where(S, torch.zeros_like(s), s)
        M = M | ((s2 == mp(s2)) & ~S)
    return torch.where(M, s, torch.zeros_like(s))[0, 0].numpy()


@pytest.mark.parametrize('r', [0, 1, 2, 4])
def test_nms_matches_max_pool_statement_on_random_and_quantised_maps(r):
    rng = np.random.default_rng(r)
    for s in (rng.random((37, 53), dtype=np.float32), (rng.integers(0, 4, (40, 33)) / 4).astype(np.float32)):
        assert np.array_equal(O.nms(s, r), _torch_nms(s, r))


def test_nms_plateau_keeps_every_equal_maximum():
    s = np.zeros((20, 20), np.float32)
    s[5, 5] = s[5, 6] = 0.5
    kept = O.nms(s, 4)
    assert kept[5, 5] == 0.5 and kept[5, 6] == 0.5


@pytest.mark.parametrize('d, both', [(4, False), (5, True)])
def test_nms_neighbours_at_radius_and_one_past(d, both):
    s = np.zeros((16, 30), np.float32)
    s[8, 5], s[8, 5 + d] = 0.9, 0.6
    kept = O.nms(s, 4)
    assert kept[8, 5] == np.float32(0.9)
    assert (kept[8, 5 + d] != 0) == both


def test_nms_second_iteration_recovers_a_pixel_only_a_suppressed_pixel_dominated():
    r = 4
    s = np.zeros((12, 40), np.float32)
    s[6, 2], s[6, 2 + r], s[6, 2 + 2 * r] = 0.9, 0.8, 0.5     # A keeps, B is suppressed by A, C only by B
    first = (s == O.maxpool(s, r))
    assert first[6, 2] and not first[6, 2 + r] and not first[6, 2 + 2 * r]
    kept = O.nms(s, r)
    assert kept[6, 2] == np.float32(0.9) and kept[6, 2 + r] == 0 and kept[6, 2 + 2 * r] == np.float32(0.5)


def test_border_and_threshold_are_strict_where_stated():
    s = np.zeros((32, 32), np.float32)
    for (y, x, v) in ((4, 10, 0.5), (3, 20, 0.5), (27, 12, 0.5), (28, 22, 0.5), (16, 16, 0.005), (16, 27, 0.0051),
                      (10, 27, 0.5), (10, 28, 0.5)):
        s[y, x] = v
    kp, sc = O.keypoints(s, 4, 0.005, 4)
    got = {(int(x), int(y)) for x, y in kp}
    # y = 4 and y = 27 (H - border - 1) are inside, y = 3 and y = 28 are not; 0.005 is not > 0.005; x = 28 is outside
    assert got == {(10, 4), (12, 27), (27, 16), (27, 10)}
    assert [tuple(k) for k in kp] == sorted([tuple(k) for k in kp], key=lambda t: (t[1], t[0]))   # row-major


def test_top_k_orders_by_score_then_lowest_flat_index():
    s = np.zeros((40, 40), np.float32)
    pts = [(30, 30, 0.5), (10, 30, 0.5), (30, 10, 0.7), (10, 10, 0.5), (20, 20, 0.6)]
    for y, x, v in pts:
        s[y, x] = v
    kp, sc = O.keypoints(s, 4, 0.005, 4, max_keypoints=4)
    assert [tuple(int(v) for v in k) for k in kp] == [(10, 30), (20, 20), (10, 10), (30, 10)]
    assert np.array_equal(sc, np.float32([0.7, 0.6, 0.5, 0.5]))
    assert len(O.keypoints(s, 4, 0.005, 4, max_keypoints=0)[0]) == 0
    assert len(O.keypoints(s, 4, 0.005, 4, max_keypoints=100)[0]) == 5


def test_sampling_convention_equals_grid_sample():
    rng = np.random.default_rng(3)
    D, hc, wc = 16, 6, 9
    desc = rng.standard_normal((D, hc, wc)).astype(np.float32)
    kps = np.stack([rng.integers(-4, 8 * wc + 4, 50), rng.integers(-4, 8 * hc + 4, 50)], 1).astype(np.float32)
    kps[:4] = [[0, 0], [8 * wc - 1, 8 * hc - 1], [3.5, 3.5], [8 * wc - 4.5, 8 * hc - 4.5]]
    got = O.sample_descriptors(desc, kps)
    t = F.normalize(torch.from_numpy(desc).double()[None], p=2, dim=1)
    k = torch.from_numpy(kps).double() - 8 / 2 + 0.5
    k = k / torch.tensor([8 * wc - 8 / 2 - 0.5, 8 * hc - 8 / 2 - 0.5], dtype=torch.float64)
    k = k * 2 - 1
    ref = F.grid_sample(t, k.view(1, 1, -1, 2), mode='bilinear', align_corners=True)
    ref = F.normalize(ref.reshape(1, D, -1), p=2, dim=1)[0].T.numpy()
    assert np.abs(got - ref).max() < 1e-13


def test_similarity_is_the_sequential_float64_sum():
    rng = np.random.default_rng(5)
    a = rng.standard_normal((7, 32)).astype(np.float32)
    b = rng.standard_normal((5, 32)).astype(np.float32)
    a[0, :3], b[0, :3] = [2.0 ** 20, 1.0, -(2.0 ** 20)], [2.0 ** 20, 2.0 ** -40, 2.0 ** 20]
    S = O.similarity(a, b)
    for i in range(7):
        for j in range(5):
            acc = 0.0
            for k in range(32):
                acc += float(a[i, k]) * float(b[j, k])
            assert S[i, j] == acc
    # the order matters: 2^40 + 2^-40 - 2^40 keeps nothing of 2^-40 in fp64, a pairwise sum could
    assert O.similarity(a[:1, :3], b[:1, :3])[0, 0] == 0.0


def _sets():
    d0 = np.float32([[1, 0], [0.8, 0.6], [0, 1], [0.6, 0.8]])
    d1 = np.float32([[1, 0], [0, 1], [1, 0]])
    return d0, d1


def test_rules_mutual_min_sim_ratio_and_ties():
    d0, d1 = _sets()
    S = O.similarity(d0, d1)
    m, s = O.match(d0, d1, mutual=False)
    assert m.tolist() == [0, 0, 1, 1]                        # column 0 and 2 tie: the lowest index wins
    m, s = O.match(d0, d1, mutual=True)
    assert m.tolist() == [0, -1, 1, -1] and s.tolist() == [S[0, 0], 0.0, S[2, 1], 0.0]
    m, _ = O.match(d0, d1, mutual=False, min_sim=S[1, 0])
    assert m.tolist() == [0, -1, 1, -1]                      # s1 == min_sim is rejected
    m, _ = O.match(d0, d1, mutual=False, ratio=0.99)
    assert m.tolist() == [-1, -1, 1, 1]                      # row 0 ties its second neighbour: 0 < 0 fails
    m, _ = O.match(d0[:1], d1[:1], mutual=False, ratio=0.0)
    assert m.tolist() == [0]                                 # no second neighbour: the ratio test passes
    assert O.match(d0[:0], d1)[0].shape == (0,) and O.match(d0, d1[:0])[0].tolist() == [-1] * 4


def test_state_dict_names_and_argument_checks():
    from patch2pix_b200.superpoint import SuperPoint
    sp = SuperPoint()
    want = [f'{n}.{p}' for n, *_ in O.CONVS for p in ('weight', 'bias')]
    assert sorted(sp.state_dict()) == sorted(want)
    sd = O.seeded_state_dict(0)
    assert all(sp.state_dict()[k].shape == v.shape for k, v in sd.items())
    with pytest.raises(RuntimeError, match='no weights'):
        sp({'image': torch.zeros(1, 1, 16, 16)})
    sp.load_state_dict(sd)
    with pytest.raises(ValueError, match='CUDA'):
        sp({'image': torch.zeros(1, 1, 16, 16)})
    for kw in ({'nms_radius': -1}, {'nms_radius': 17}, {'nms_radius': 2.0}, {'remove_borders': -1},
               {'keypoint_threshold': float('nan')}, {'max_keypoints': True}):
        with pytest.raises(ValueError):
            SuperPoint(**kw)
    with pytest.raises(NotImplementedError):
        sp.train()


def test_oracle_network_shapes():
    sd = O.seeded_state_dict(1)
    logits, desc = O.heads(sd, torch.rand(1, 1, 35, 50))
    assert logits.shape == (1, 65, 4, 6) and desc.shape == (1, 256, 4, 6)
    assert O.score_map(logits[0]).shape == (32, 48)
