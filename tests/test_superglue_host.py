"""SuperGlue's module (patch2pix_b200/superglue.py) on the CPU: its state_dict, its argument checks, and its GNN score
path in float64 against the numpy restatement (oracle/superglue_oracle.py); the oracle's Sinkhorn and extraction."""
import numpy as np
import pytest
import torch

from oracle import superglue_oracle as O
from patch2pix_b200 import superglue as SG


def test_state_dict_names_and_shapes():
    sd = SG.SuperGlue().state_dict()
    ref = O.seeded_state_dict(0)
    assert sorted(sd) == sorted(ref)
    for k, v in ref.items():
        assert tuple(sd[k].shape) == tuple(v.shape), k
    assert tuple(sd['kenc.encoder.0.weight'].shape) == (32, 3, 1)
    assert tuple(sd['kenc.encoder.12.weight'].shape) == (256, 256, 1)
    assert tuple(sd['gnn.layers.17.attn.proj.2.weight'].shape) == (256, 256, 1)
    assert tuple(sd['gnn.layers.0.mlp.0.weight'].shape) == (512, 512, 1)
    assert tuple(sd['gnn.layers.0.mlp.3.weight'].shape) == (256, 512, 1)
    assert tuple(sd['gnn.layers.5.mlp.1.running_var'].shape) == (512,)
    assert sd['bin_score'].shape == () and float(sd['bin_score']) == 1.0
    assert len({k.split('.')[2] for k in sd if k.startswith('gnn.layers.')}) == 18


@pytest.mark.parametrize('cfg', [{'descriptor_dim': 30}, {'descriptor_dim': True}, {'GNN_layers': ['self', 'other']},
                                 {'GNN_layers': 'self'}, {'sinkhorn_iterations': -1},
                                 {'sinkhorn_iterations': 1.5}, {'match_threshold': float('nan')},
                                 {'keypoint_encoder': [32, 0]}, {'no_such_key': 1}])
def test_config_is_checked(cfg):
    with pytest.raises(ValueError):
        SG.SuperGlue(cfg)


def test_config_defaults_and_modes():
    sg = SG.SuperGlue({'weights': 'outdoor'})
    assert sg.config['weights'] == 'outdoor' and sg.config['sinkhorn_iterations'] == 100
    assert sg.config['match_threshold'] == 0.2 and sg.config['GNN_layers'] == ['self', 'cross'] * 9
    assert not sg.training
    with pytest.raises(NotImplementedError):
        sg.train()
    sg.eval()
    data = _data(torch.Generator().manual_seed(0), 1, 5, 6, 256, torch.float32)
    with pytest.raises(RuntimeError, match='load_state_dict'):
        sg(data)
    sg.load_state_dict(O.seeded_state_dict(0))
    with pytest.raises(ValueError, match='CUDA'):
        sg(data)


def test_empty_sets_return_no_matches_without_a_launch():
    sg = SG.SuperGlue()
    sg.load_state_dict(O.seeded_state_dict(0))
    for n, m in ((0, 7), (4, 0), (0, 0)):
        data = _data(torch.Generator().manual_seed(1), 2, n, m, 256, torch.float32)
        out = sg(data)                                   # CPU tensors: nothing runs, so no CUDA is needed
        assert out['matches0'].shape == (2, n) and out['matches1'].shape == (2, m)
        assert out['matches0'].dtype == torch.int64 and (out['matches0'] == -1).all() and (out['matches1'] == -1).all()
        assert out['matching_scores0'].dtype == torch.float32 and not out['matching_scores0'].any()
        assert not out['matching_scores1'].any()


def test_sinkhorn_arguments_are_checked():
    with pytest.raises(ValueError, match='CUDA'):
        SG.log_optimal_transport(torch.zeros(1, 3, 4), 1.0, 10)
    with pytest.raises(ValueError):
        SG.log_optimal_transport(torch.zeros(3, 4), 1.0, 10)


def _data(g, B, n, m, dim, dtype, H=(120, 96), W=(160, 128)):
    def kp(k, h, w):
        return torch.stack([torch.rand(B, k, generator=g) * (w - 1), torch.rand(B, k, generator=g) * (h - 1)], 2)

    def desc(k):
        d = torch.randn(B, dim, k, generator=g)
        return d / d.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return {'image0': torch.zeros(B, 1, H[0], W[0]), 'image1': torch.zeros(B, 1, H[1], W[1]),
            'keypoints0': kp(n, H[0], W[0]).to(dtype), 'keypoints1': kp(m, H[1], W[1]).to(dtype),
            'scores0': torch.rand(B, n, generator=g).to(dtype), 'scores1': torch.rand(B, m, generator=g).to(dtype),
            'descriptors0': desc(n).to(dtype), 'descriptors1': desc(m).to(dtype)}


@pytest.mark.parametrize('dim, enc, layers', [(256, [32, 64, 128, 256], ['self', 'cross'] * 9),
                                              (64, [16, 32], ['cross', 'self', 'cross'])])
def test_gnn_scores_equal_float64_oracle(dim, enc, layers):
    sd = O.seeded_state_dict(3, dim, enc, len(layers), bin_score=0.7)
    sg = SG.SuperGlue({'descriptor_dim': dim, 'keypoint_encoder': enc, 'GNN_layers': layers})
    sg.load_state_dict(sd)
    sg = sg.double()
    data = _data(torch.Generator().manual_seed(5), 2, 37, 29, dim, torch.float64)
    with torch.no_grad():
        got = sg.score_matrix(data).numpy()
    npd = O.to_numpy(sd)
    for b in range(2):
        ref = O.scores(npd, data['keypoints0'][b].numpy(), data['keypoints1'][b].numpy(), data['scores0'][b].numpy(),
                       data['scores1'][b].numpy(), data['descriptors0'][b].numpy(), data['descriptors1'][b].numpy(),
                       (120, 160), (96, 128), layers, len(enc) + 1)
        assert np.abs(got[b] - ref).max() < 1e-10 * max(1.0, np.abs(ref).max())
        assert np.abs(ref).max() > 1e-2                  # the scores are not trivially small


def test_heads_are_interleaved_and_cross_sources_swapped():
    # the oracle with head-blocked channels, or with self sources in the cross layers, must not match the module
    sd = O.seeded_state_dict(4, 64, [16], 2)
    sg = SG.SuperGlue({'descriptor_dim': 64, 'keypoint_encoder': [16], 'GNN_layers': ['self', 'cross']})
    sg.load_state_dict(sd)
    sg = sg.double()
    data = _data(torch.Generator().manual_seed(6), 1, 11, 13, 64, torch.float64)
    with torch.no_grad():
        got = sg.score_matrix(data)[0].numpy()
    npd = O.to_numpy(sd)
    args = [data[k][0].numpy() for k in ('keypoints0', 'keypoints1', 'scores0', 'scores1', 'descriptors0',
                                          'descriptors1')] + [(120, 160), (96, 128)]
    assert np.abs(got - O.scores(npd, *args, ['self', 'cross'], 2)).max() < 1e-10
    assert np.abs(got - O.scores(npd, *args, ['self', 'self'], 2)).max() > 1e-6
    perm = np.arange(64).reshape(4, 16).T.ravel()        # channel c -> head c // 16 instead of c % 4
    blocked = dict(npd)
    for k in range(2):
        for p in range(3):
            blocked[f'gnn.layers.{k}.attn.proj.{p}.weight'] = npd[f'gnn.layers.{k}.attn.proj.{p}.weight'][perm]
            blocked[f'gnn.layers.{k}.attn.proj.{p}.bias'] = npd[f'gnn.layers.{k}.attn.proj.{p}.bias'][perm]
        blocked[f'gnn.layers.{k}.attn.merge.weight'] = npd[f'gnn.layers.{k}.attn.merge.weight'][:, perm]
    assert np.abs(got - O.scores(blocked, *args, ['self', 'cross'], 2)).max() > 1e-6


@pytest.mark.parametrize('n, m, alpha', [(7, 5, 1.0), (1, 9, -0.5), (12, 12, 2.5)])
def test_oracle_sinkhorn_converges_to_the_marginals(n, m, alpha):
    s = np.random.default_rng(n * 100 + m).normal(0, 2, (n, m))
    la, vmax = O.log_optimal_transport(s, alpha, 3000)
    norm = -np.log(n + m)
    log_mu = np.concatenate([np.full(n, norm), [np.log(m) + norm]])
    log_nu = np.concatenate([np.full(m, norm), [np.log(n) + norm]])
    lse_r = np.log(np.exp(la).sum(1))
    lse_c = np.log(np.exp(la).sum(0))
    assert np.abs(lse_r - (log_mu - norm)).max() < 1e-6
    assert np.abs(lse_c - (log_nu - norm)).max() < 1e-9   # the last half-iteration fits the columns exactly
    assert vmax > 0


def test_oracle_extraction_rules():
    z = np.array([[0.0, -1.5, -2.0],      # row 0 -> col 0, mutual
                  [-3.0, -3.0, -9.0],     # row 1: tie -> col 0 (lowest index), not mutual
                  [-9.0, -1.0, -1.0]])    # row 2: tie -> col 1, mutual; exp(-1) > 0.2
    la = np.full((4, 4), -50.0)
    la[:3, :3] = z
    e = O.extract(la, 0.2)
    assert e['matches0'].tolist() == [0, -1, 1] and e['matches1'].tolist() == [0, 2, -1]
    assert e['mutual0'].tolist() == [True, False, True] and e['mutual1'].tolist() == [True, True, False]
    assert np.allclose(e['mscores0'], [1.0, 0.0, np.exp(-1.0)]) and np.allclose(e['mscores1'], [1.0, np.exp(-1.0), 0])
    e = O.extract(la, 0.5)                # row 2 is mutual but fails the threshold: mscores keep exp(max)
    assert e['matches0'].tolist() == [0, -1, -1] and e['matches1'].tolist() == [0, -1, -1]
    assert np.isclose(e['mscores0'][2], np.exp(-1.0)) and np.isclose(e['mscores1'][1], np.exp(-1.0))
    rows, cols = O.decidable(la, 0.2, 0.1)
    assert rows.tolist() == [True, False, False] and cols.tolist() == [True, False, False]


def test_error_bound_grows_with_iterations_and_magnitudes():
    b0 = O.sinkhorn_bound(100, 100, 10.0, 0.0, 0)
    assert 0 < b0 < 1e-5
    assert O.sinkhorn_bound(100, 100, 10.0, 5.0, 100) > O.sinkhorn_bound(100, 100, 10.0, 5.0, 10) > b0
    assert O.sinkhorn_bound(4000, 3000, 10.0, 5.0, 100) > O.sinkhorn_bound(100, 100, 10.0, 5.0, 100)
