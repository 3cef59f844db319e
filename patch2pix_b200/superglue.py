"""SuperGlue's matcher on SuperPoint keypoints, as the coarse matcher in front of Patch2Pix's refiner
("SuperPoint + SuperGlue, refined by Patch2Pix").

The keypoint encoder and the attentional GNN are dense 1x1 convolutions and attention; they run in PyTorch (cuBLAS)
and follow torch's TF32 flags, as SuperPoint's encoder does.  For fp32 set
``torch.backends.cuda.matmul.allow_tf32 = False`` and ``torch.backends.cudnn.allow_tf32 = False``.  The optimal
transport step, 100 log-domain Sinkhorn iterations over an (N+1) x (M+1) matrix with a dustbin row and column,
followed by the mutual-argmax extraction, runs as one cooperative launch of csrc/superglue.cu (p2p_sg_sinkhorn, whose
semantics include/p2p_b200.h states).

Conventions.  These are recalled from SuperGlue's published code and were not checked against that code or its released
weights; oracle/superglue_oracle.py restates them in float64:
  - keypoints are normalised by (kpts - [W/2, H/2]) / (0.7 max(W, H)) for an image of H x W pixels;
  - the keypoint encoder is MLP([3, 32, 64, 128, 256, 256]) of Conv1d(k=1) + BatchNorm1d + ReLU with no BN / ReLU after
    the last layer; its input is cat(normalised kpts^T, scores) and its output is added to the descriptors;
  - 18 AttentionalPropagation layers ('self', 'cross' x 9).  Each is 4-head attention whose q / k / v projections are
    viewed as [B, 64, 4, N], so channel c belongs to head c % 4; logits are scaled by 1/8 (1/sqrt(64)).  A layer
    applies merge, then MLP([512, 512, 256]) to cat(x, message), and adds the result to x.  Cross layers take their
    source from the other image;
  - final_proj is Conv1d(256, 256, 1), and the scores are mdesc0^T mdesc1 / sqrt(descriptor_dim) (/ 16);
  - bin_score is a scalar parameter (1.0 before loading);
  - state_dict names: kenc.encoder.{0,1,3,4,6,7,9,10,12}.*, gnn.layers.{k}.attn.proj.{0,1,2}.*,
    gnn.layers.{k}.attn.merge.*, gnn.layers.{k}.mlp.{0,1,3}.*, final_proj.*, bin_score.
"""
import math

import torch
from torch import nn

from . import _lib

DEFAULT_CONFIG = {
    'descriptor_dim': 256,
    'weights': 'indoor',
    'keypoint_encoder': [32, 64, 128, 256],
    'GNN_layers': ['self', 'cross'] * 9,
    'sinkhorn_iterations': 100,
    'match_threshold': 0.2,
}
NUM_HEADS = 4
MAX_ITERS = 100000


def _mlp(channels):
    """Conv1d(k=1) + BatchNorm1d + ReLU per layer, with no BN / ReLU after the last one."""
    layers = []
    for i in range(1, len(channels)):
        layers.append(nn.Conv1d(channels[i - 1], channels[i], 1, bias=True))
        if i < len(channels) - 1:
            layers += [nn.BatchNorm1d(channels[i]), nn.ReLU()]
    return nn.Sequential(*layers)


class _KeypointEncoder(nn.Module):
    def __init__(self, dim, layers):
        super().__init__()
        self.encoder = _mlp([3] + list(layers) + [dim])
        nn.init.constant_(self.encoder[-1].bias, 0.0)

    def forward(self, kpts, scores):
        return self.encoder(torch.cat([kpts.transpose(1, 2), scores.unsqueeze(1)], 1))


class _Attention(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.heads, self.head_dim = heads, dim // heads
        self.merge = nn.Conv1d(dim, dim, 1)
        self.proj = nn.ModuleList([nn.Conv1d(dim, dim, 1) for _ in range(3)])

    def forward(self, x, source):
        b = x.shape[0]
        q, k, v = (p(t).view(b, self.head_dim, self.heads, -1) for p, t in zip(self.proj, (x, source, source)))
        prob = torch.softmax(torch.einsum('bdhn,bdhm->bhnm', q, k) / self.head_dim ** 0.5, dim=-1)
        msg = torch.einsum('bhnm,bdhm->bdhn', prob, v)
        return self.merge(msg.reshape(b, self.head_dim * self.heads, -1))


class _Propagation(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.attn = _Attention(dim, heads)
        self.mlp = _mlp([2 * dim, 2 * dim, dim])
        nn.init.constant_(self.mlp[-1].bias, 0.0)

    def forward(self, x, source):
        return self.mlp(torch.cat([x, self.attn(x, source)], 1))


class _GNN(nn.Module):
    def __init__(self, dim, names):
        super().__init__()
        self.names = list(names)
        self.layers = nn.ModuleList([_Propagation(dim, NUM_HEADS) for _ in self.names])

    def forward(self, d0, d1):
        for layer, name in zip(self.layers, self.names):
            s0, s1 = (d1, d0) if name == 'cross' else (d0, d1)
            d0, d1 = d0 + layer(d0, s0), d1 + layer(d1, s1)
        return d0, d1


def normalize_keypoints(kpts, image_shape):
    """(kpts - [W/2, H/2]) / (0.7 max(W, H)) for keypoints [B, N, 2] (x, y) of images of shape [..., H, W]."""
    h, w = int(image_shape[-2]), int(image_shape[-1])
    center = torch.stack([kpts.new_full((), w / 2), kpts.new_full((), h / 2)])   # filled on the device: no copy
    return (kpts - center) / (0.7 * max(w, h))


def _check_config(cfg):
    d = cfg['descriptor_dim']
    if isinstance(d, bool) or not isinstance(d, int) or d < NUM_HEADS or d % NUM_HEADS:
        raise ValueError(f'descriptor_dim must be a positive multiple of {NUM_HEADS}, got {d!r}')
    enc = cfg['keypoint_encoder']
    if not all(isinstance(c, int) and not isinstance(c, bool) and c > 0 for c in enc):
        raise ValueError(f'keypoint_encoder must be a list of positive ints, got {enc!r}')
    names = cfg['GNN_layers']
    if isinstance(names, str) or not all(n in ('self', 'cross') for n in names):
        raise ValueError(f"GNN_layers must be a list of 'self' / 'cross', got {names!r}")
    it = cfg['sinkhorn_iterations']
    if isinstance(it, bool) or not isinstance(it, int) or not 0 <= it <= MAX_ITERS:
        raise ValueError(f'sinkhorn_iterations must be an int in 0..{MAX_ITERS}, got {it!r}')
    thr = cfg['match_threshold']
    if isinstance(thr, bool) or not isinstance(thr, (int, float)) or not math.isfinite(thr):
        raise ValueError(f'match_threshold must be a finite number, got {thr!r}')


def _sinkhorn(scores, alpha, iters, threshold, log_assign=False, matches=True):
    """p2p_sg_sinkhorn on scores [B, N, M] (fp32 CUDA) and alpha (a CUDA scalar tensor) -> dict of the requested
    outputs: 'log_assign' [B, N+1, M+1]; 'matches0' [B, N] / 'matches1' [B, M] int32, 'mscores0' / 'mscores1' fp32.
    No host sync."""
    if not (isinstance(scores, torch.Tensor) and scores.is_cuda and scores.dim() == 3):
        raise ValueError('scores must be a [B, N, M] CUDA tensor')
    B, n, m = scores.shape
    if B < 1 or n < 1 or m < 1:
        raise ValueError(f'scores must be non-empty, got {tuple(scores.shape)}')
    if isinstance(iters, bool) or not isinstance(iters, int) or not 0 <= iters <= MAX_ITERS:
        raise ValueError(f'iters must be an int in 0..{MAX_ITERS}, got {iters!r}')
    dev = scores.device
    scores = scores.float().contiguous()
    if isinstance(alpha, torch.Tensor):
        if alpha.numel() != 1:
            raise ValueError('alpha must hold one value')
        alpha = alpha.detach().to(device=dev, dtype=torch.float32).reshape(1).contiguous()
    else:
        alpha = torch.full((1,), float(alpha), dtype=torch.float32, device=dev)
    out = {}
    if log_assign:
        out['log_assign'] = torch.empty(B, n + 1, m + 1, dtype=torch.float32, device=dev)
    if matches:
        out['matches0'] = torch.empty(B, n, dtype=torch.int32, device=dev)
        out['matches1'] = torch.empty(B, m, dtype=torch.int32, device=dev)
        out['mscores0'] = torch.empty(B, n, dtype=torch.float32, device=dev)
        out['mscores1'] = torch.empty(B, m, dtype=torch.float32, device=dev)
    h = _lib.default_handle(dev)
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_sg_sinkhorn(
            h.h, _lib.ptr(scores), B, n, m, _lib.ptr(alpha), iters, float(threshold), _lib.ptr(out.get('log_assign')),
            *(_lib.ptr(out.get(k)) for k in ('matches0', 'matches1', 'mscores0', 'mscores1')), h.stream()))
    return out


def log_optimal_transport(scores, alpha, iters):
    """SuperGlue's log_optimal_transport on p2p_sg_sinkhorn: scores [B, N, M] fp32 CUDA, alpha the bin score (a CUDA
    scalar tensor or a number) -> log assignment [B, N+1, M+1] fp32.  No host sync."""
    return _sinkhorn(scores, alpha, iters, 0.0, log_assign=True, matches=False)['log_assign']


class SuperGlue(nn.Module):
    """SuperGlue (inference, CUDA): forward(data) with SuperGlue's keys image0/1, keypoints0/1 [B, N, 2], scores0/1
    [B, N], descriptors0/1 [B, D, N] -> {'matches0' [B, N], 'matches1' [B, M] int64 (-1: no match),
    'matching_scores0', 'matching_scores1' fp32}, with no host sync.  `config['weights']` is recorded only: nothing is
    downloaded, and forward raises until load_state_dict has been called."""

    def __init__(self, config=None):
        super().__init__()
        config = dict(config or {})
        unknown = set(config) - set(DEFAULT_CONFIG)
        if unknown:
            raise ValueError(f'unknown SuperGlue config keys: {sorted(unknown)}')
        self.config = {**DEFAULT_CONFIG, **config}
        _check_config(self.config)
        dim = self.config['descriptor_dim']
        self.kenc = _KeypointEncoder(dim, self.config['keypoint_encoder'])
        self.gnn = _GNN(dim, self.config['GNN_layers'])
        self.final_proj = nn.Conv1d(dim, dim, 1, bias=True)
        self.register_parameter('bin_score', nn.Parameter(torch.tensor(1.0)))
        self._loaded = False
        super().train(False)

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._loaded = True
        return r

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('SuperGlue is inference-only here')
        return super().train(False)

    def score_matrix(self, data):
        """The network up to the optimal transport: scores [B, N, M] = mdesc0^T mdesc1 / sqrt(descriptor_dim), on the
        module's device and dtype (the CPU in float64 works too)."""
        k0, k1 = data['keypoints0'], data['keypoints1']
        d0, d1 = data['descriptors0'], data['descriptors1']
        s0, s1 = data['scores0'], data['scores1']
        dim = self.config['descriptor_dim']
        for k, d, s, i in ((k0, d0, s0, 0), (k1, d1, s1, 1)):
            if k.dim() != 3 or k.shape[2] != 2 or d.dim() != 3 or d.shape[1] != dim or s.dim() != 2:
                raise ValueError(f'keypoints{i} must be [B, N, 2], descriptors{i} [B, {dim}, N] and scores{i} [B, N]')
            if d.shape[0] != k.shape[0] or d.shape[2] != k.shape[1] or tuple(s.shape) != tuple(k.shape[:2]):
                raise ValueError(f'keypoints{i}, descriptors{i} and scores{i} disagree on B or N')
        if k0.shape[0] != k1.shape[0]:
            raise ValueError('both images need the same batch size')
        k0 = normalize_keypoints(k0, data['image0'].shape)
        k1 = normalize_keypoints(k1, data['image1'].shape)
        d0 = d0 + self.kenc(k0, s0)
        d1 = d1 + self.kenc(k1, s1)
        d0, d1 = self.gnn(d0, d1)
        m0, m1 = self.final_proj(d0), self.final_proj(d1)
        return torch.einsum('bdn,bdm->bnm', m0, m1) / dim ** 0.5

    @torch.no_grad()
    def forward(self, data):
        if not self._loaded:
            raise RuntimeError('SuperGlue has no weights: call load_state_dict (nothing is downloaded)')
        k0, k1 = data['keypoints0'], data['keypoints1']
        if not (isinstance(k0, torch.Tensor) and isinstance(k1, torch.Tensor) and k0.dim() == 3 and k1.dim() == 3):
            raise ValueError('keypoints0 / keypoints1 must be [B, N, 2] tensors')
        if k0.shape[1] == 0 or k1.shape[1] == 0:     # nothing to match: no launch, as SuperGlue returns early
            s0, s1 = k0.shape[:-1], k1.shape[:-1]
            return {'matches0': k0.new_full(s0, -1, dtype=torch.int64),
                    'matches1': k1.new_full(s1, -1, dtype=torch.int64),
                    'matching_scores0': k0.new_zeros(s0, dtype=torch.float32),
                    'matching_scores1': k1.new_zeros(s1, dtype=torch.float32)}
        if not (k0.is_cuda and k1.is_cuda):
            raise ValueError('SuperGlue runs on CUDA tensors only')
        scores = self.score_matrix(data)
        out = _sinkhorn(scores, self.bin_score, self.config['sinkhorn_iterations'], self.config['match_threshold'])
        return {'matches0': out['matches0'].long(), 'matches1': out['matches1'].long(),
                'matching_scores0': out['mscores0'], 'matching_scores1': out['mscores1']}


def superglue_matcher(sp, sg):
    """The coarse_matcher(grey1, grey2) -> [N, 4] float32 (x1, y1, x2, y2) rows that eval_helper.refine_matches takes:
    SuperPoint `sp` on both grey images, then SuperGlue `sg` on its keypoints; one row per valid matches0 entry."""
    def matcher(grey1, grey2):
        if grey1.shape == grey2.shape:
            out = sp({'image': torch.cat([grey1, grey2])})
            k0, k1 = out['keypoints']
            s0, s1 = out['scores']
            e0, e1 = out['descriptors']
        else:
            a, b = sp({'image': grey1}), sp({'image': grey2})
            k0, k1 = a['keypoints'][0], b['keypoints'][0]
            s0, s1 = a['scores'][0], b['scores'][0]
            e0, e1 = a['descriptors'][0], b['descriptors'][0]
        m = sg({'image0': grey1, 'image1': grey2, 'keypoints0': k0[None], 'keypoints1': k1[None],
                'scores0': s0[None], 'scores1': s1[None], 'descriptors0': e0[None], 'descriptors1': e1[None]})
        m = m['matches0'][0]
        keep = m >= 0
        return torch.cat([k0[keep], k1[m[keep]]], 1)
    return matcher
