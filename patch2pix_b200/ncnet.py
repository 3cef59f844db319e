"""NCNet's matcher (the reference's networks/ncn/model.py: ImMatchNet, NeighConsensus, and
networks/ncn/extract_ncmatches.py: corr_to_matches, corr_to_matches_topk) on the tensor-core library.

    -from networks.ncn.model import ImMatchNet
    +from patch2pix_b200.ncnet import ImMatchNet

The ResNet101 layer3 backbone is plain PyTorch (torchvision, no weights are ever downloaded), like backbone.py.
Everything after it -- L2 normalisation, correlation, 4D max-pool relocalisation, both MutualMatchings and the
NeighConsensus stack -- runs as CUDA kernels of libp2p_b200.so (p2p_ncnet_coarse, p2p_nc_stack).  Inference only.
"""
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib

__all__ = ['ImMatchNet', 'NeighConsensus', 'corr_to_matches', 'corr_to_matches_topk']


def _as_ints(v, name):
    try:
        return [int(x) for x in v]
    except TypeError:
        raise ValueError(f'{name} must be a list of ints, got {v!r}') from None


class _Conv4dParams(nn.Module):
    """Parameters of the reference's Conv4d (pre-permuted weight [k, Cout, Cin, k, k, k], bias [Cout])."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(k, cout, cin, k, k, k))
        self.bias = nn.Parameter(torch.zeros(cout))


class NeighConsensus(nn.Module):
    """networks/ncn/model.py:124-155.  State-dict names are the reference's (conv.0.weight, conv.0.bias, conv.2...);
    forward runs the stack on the tensor cores (p2p_nc_stack) on a [b, 1, hA, wA, hB, wB] fp32 CUDA volume."""

    def __init__(self, use_cuda=True, kernel_sizes=[3, 3, 3], channels=[10, 10, 1], symmetric_mode=True):
        super().__init__()
        if not use_cuda:
            raise ValueError('NeighConsensus runs on CUDA only (use_cuda=False is not supported)')
        ks, ch = _as_ints(kernel_sizes, 'kernel_sizes'), _as_ints(channels, 'channels')
        if len(ks) != len(ch) or not ks:
            raise ValueError('kernel_sizes and channels must be non-empty lists of the same length')
        if any(k not in (3, 5) for k in ks):
            raise ValueError(f'kernel sizes must be 3 or 5, got {ks}')
        if any(c < 1 or c > 16 for c in ch):
            raise ValueError(f'channels must be in 1..16, got {ch}')
        if ch[-1] != 1:
            raise ValueError(f'the last layer must have 1 output channel, got {ch}')
        self.symmetric_mode = bool(symmetric_mode)
        self.kernel_sizes, self.channels = ks, ch
        mods = []
        for i, (k, c) in enumerate(zip(ks, ch)):
            mods += [_Conv4dParams(1 if i == 0 else ch[i - 1], c, k), nn.ReLU(inplace=True)]
        self.conv = nn.Sequential(*mods)
        self._handles = {}

    def _handle(self, device):
        """Per-device handle with the current weights packed (re-packed when a parameter changed)."""
        key = device.index
        stamp = tuple((p.data_ptr(), p._version) for p in self.parameters())
        hs = self._handles.get(key)
        if hs is None or hs[1] != stamp:
            h = hs[0] if hs is not None else _lib.Handle(device)
            import ctypes as C
            n = len(self.kernel_sizes)
            ws = [m.weight.detach().float().cpu().contiguous() for m in self.conv if isinstance(m, _Conv4dParams)]
            bs = [m.bias.detach().float().cpu().contiguous() for m in self.conv if isinstance(m, _Conv4dParams)]
            wp = (C.c_void_p * n)(*[w.data_ptr() for w in ws])
            bp = (C.c_void_p * n)(*[b.data_ptr() for b in bs])
            _lib.check(h.lib.p2p_set_nc_stack_weights(h.h, n, (C.c_int * n)(*self.kernel_sizes),
                                                      (C.c_int * n)(*self.channels), wp, bp,
                                                      int(self.symmetric_mode)))
            hs = (h, stamp)
            self._handles[key] = hs
        return hs[0]

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('NeighConsensus is inference-only (no Conv4d backward)')
        return super().train(False)

    @torch.no_grad()
    def forward(self, x):
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 6 and x.shape[1] == 1):
            raise ValueError('NeighConsensus expects a [b, 1, hA, wA, hB, wB] float32 CUDA tensor')
        x = x.contiguous()
        b, _, hA, wA, hB, wB = x.shape
        out = torch.empty_like(x)
        h = self._handle(x.device)
        with torch.cuda.device(x.device):
            for i in range(b):
                _lib.check(h.lib.p2p_nc_stack(h.h, _lib.ptr(x[i]), hA, wA, hB, wB, _lib.ptr(out[i]), h.stream()))
        return out


class FeatureExtraction(nn.Module):
    """ResNet101 cut after layer3 (networks/ncn/model.py:21-96, resnet101 branch); state-dict names model.{0,1,4,5,6}.*"""

    def __init__(self):
        super().__init__()
        import torchvision
        r = torchvision.models.resnet101(weights=None)
        self.model = nn.Sequential(r.conv1, r.bn1, r.relu, r.maxpool, r.layer1, r.layer2, r.layer3)

    def forward(self, x):
        return self.model(x)


class ImMatchNet(nn.Module):
    """networks/ncn/model.py:205-331 (inference).  Outputs keep the reference's shapes and dtypes: corr4d
    [b, 1, hA, wA, hB, wB] float32, and with relocalization_k_size 2 delta4d = (max_i, max_j, max_k float32, max_l int64)
    as maxpool4d's true division yields them on torch 2.x."""

    def __init__(self, feature_extraction_cnn='resnet101', feature_extraction_last_layer='',
                 feature_extraction_model_file=None, return_correlation=False, ncons_kernel_sizes=[3, 3, 3],
                 ncons_channels=[10, 10, 1], normalize_features=True, train_fe=False, use_cuda=True,
                 relocalization_k_size=0, half_precision=False, checkpoint=None):
        super().__init__()
        if feature_extraction_cnn != 'resnet101':
            raise ValueError(f"only feature_extraction_cnn='resnet101' is supported, got {feature_extraction_cnn!r}")
        if feature_extraction_last_layer not in ('', 'layer3'):
            raise ValueError('only the layer3 features of ResNet101 are supported')
        if half_precision:
            raise ValueError('half_precision=True is not supported (the stack computes fp32-grade results)')
        if not use_cuda:
            raise ValueError('ImMatchNet runs on CUDA only (use_cuda=False is not supported)')
        if train_fe:
            raise ValueError('training is not supported')
        if not normalize_features:
            raise ValueError('normalize_features=False is not supported (the correlation kernel L2-normalises)')
        if relocalization_k_size not in (0, 1, 2):
            raise ValueError(f'relocalization_k_size must be 0, 1 or 2, got {relocalization_k_size}')
        sd = None
        if checkpoint is not None and checkpoint != '':
            ck = torch.load(checkpoint, map_location='cpu', weights_only=False)
            sd = OrderedDict((k.replace('vgg', 'model'), v) for k, v in ck['state_dict'].items())
            ncons_channels = ck['args'].ncons_channels
            ncons_kernel_sizes = ck['args'].ncons_kernel_sizes
        self.normalize_features = normalize_features
        self.return_correlation = return_correlation
        self.relocalization_k_size = relocalization_k_size
        self.half_precision = False
        self.FeatureExtraction = FeatureExtraction()
        if torch.cuda.is_available():          # the reference's use_cuda=True: the backbone lives on the current GPU
            self.FeatureExtraction.to(torch.device('cuda', torch.cuda.current_device()))
        self.NeighConsensus = NeighConsensus(kernel_sizes=ncons_kernel_sizes, channels=ncons_channels)
        self._loaded = False
        if sd is not None:
            own = self.state_dict()
            missing = [k for k in own if 'num_batches_tracked' not in k and k not in sd]
            if missing:
                raise KeyError(f'checkpoint lacks {missing[:4]}{" ..." if len(missing) > 4 else ""}')
            self.load_state_dict(OrderedDict((k, sd[k]) for k in own if k in sd), strict=False)
        super().train(False)

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._loaded = True
        return r

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('ImMatchNet is inference-only here')
        return super().train(False)

    def _require_weights(self):
        if not self._loaded:
            raise RuntimeError('ImMatchNet has no weights: pass checkpoint=... or call load_state_dict (nothing is '
                               'downloaded)')

    @torch.no_grad()
    def forward_feat(self, featA, featB, normalize=True):
        """networks/ncn/model.py:314-331 on layer3 features [b, C, h, w] (C % 64 == 0)."""
        self._require_weights()
        if not normalize:
            raise ValueError('forward_feat runs with normalize=True only (the correlation kernel L2-normalises)')
        for t, n in ((featA, 'featA'), (featB, 'featB')):
            if not (t.is_cuda and t.dim() == 4):
                raise ValueError(f'{n} must be a [b, C, h, w] CUDA tensor')
        from .model import _coarse_per_pair, _unpack_delta
        featA, featB = featA.float().contiguous(), featB.float().contiguous()
        k = max(1, self.relocalization_k_size)
        h = self.NeighConsensus._handle(featA.device)
        corr4d, code = _coarse_per_pair(h, h.lib.p2p_ncnet_coarse, featA, featB, k)
        if k == 1:
            return corr4d
        ds = _unpack_delta(code, k, h)
        return corr4d, (ds[0].float(), ds[1].float(), ds[2].float(), ds[3])

    @torch.no_grad()
    def forward(self, tnf_batch):
        """networks/ncn/model.py:281-312: tnf_batch['source_image'], tnf_batch['target_image'] [b, 3, H, W]."""
        self._require_weights()
        fa = self.FeatureExtraction(tnf_batch['source_image'])
        fb = self.FeatureExtraction(tnf_batch['target_image'])
        return self.forward_feat(fa, fb, normalize=True)


def _grid(n, lo):
    return torch.linspace(lo, 1.0, n, dtype=torch.float64).float()


@torch.no_grad()
def corr_to_matches(corr4d, delta4d=None, ksize=1, do_softmax=True, scale='positive', invert_matching_direction=False,
                    return_indices=True):
    """networks/ncn/extract_ncmatches.py:6-94 on the GPU (p2p_proposals).  corr4d [b, 1, hA, wA, hB, wB] fp32 CUDA;
    delta4d: the reference's (max_i, max_j, max_k, max_l) tuple (float or int64 tensors) or ImMatchNet's.
    -> (jA, iA, jB, iB, score) int64 indices, or (xA, yA, xB, yB, score) float32 coordinates for return_indices=False;
    score float32 [b, N] (N = hB*wB, or hA*wA with invert_matching_direction)."""
    from .model import cal_coarse_matches
    if scale not in ('positive', 'centered'):
        raise ValueError(f"scale must be 'positive' or 'centered', got {scale!r}")
    if not (corr4d.is_cuda and corr4d.dtype == torch.float32 and corr4d.dim() == 6):
        raise ValueError('corr_to_matches expects a [b, 1, hA, wA, hB, wB] float32 CUDA tensor')
    b, _, hA, wA, hB, wB = corr4d.shape
    if delta4d is not None:
        if ksize not in (1, 2, 3):
            raise ValueError('ksize must be 1, 2 or 3 with delta4d')
        delta4d = tuple(d.to(device=corr4d.device, dtype=torch.int64).contiguous() for d in delta4d)
    # rows: the best A cell of every B cell, then the best B cell of every A cell, as (jA, iA, jB, iB) in indices
    m, sc = cal_coarse_matches(corr4d.contiguous(), delta4d, ksize if delta4d is not None else 1, do_softmax,
                               upsample=1, center=False)
    n = hA * wA if invert_matching_direction else hB * wB
    rows = m[:, hB * wB:] if invert_matching_direction else m[:, :n]
    score = (sc[:, hB * wB:] if invert_matching_direction else sc[:, :n]).contiguous()
    jA, iA, jB, iB = [rows[..., c].contiguous() for c in range(4)]
    if return_indices:
        return jA, iA, jB, iB, score
    lo = -1.0 if scale == 'centered' else 0.0
    dev = corr4d.device
    xa, ya = _grid(wA * ksize, lo).to(dev), _grid(hA * ksize, lo).to(dev)
    xb, yb = _grid(wB * ksize, lo).to(dev), _grid(hB * ksize, lo).to(dev)
    return xa[jA], ya[iA], xb[jB], yb[iB], score


TOPK_MAX_SLICE = 32768      # longest slice p2p_proposals_topk stages (kTopkMaxSlice in csrc/kernels.h)


@torch.no_grad()
def corr_to_matches_topk(corr4d, delta4d=None, topk=1, ksize=1, do_softmax=True, invert_matching_direction=False):
    """networks/ncn/extract_ncmatches.py:96-158 on the GPU (p2p_proposals_topk, one launch for the batch).
    corr4d [b, 1, hA, wA, hB, wB] fp32 CUDA; delta4d as for corr_to_matches (ksize is ignored without it).
    -> (jA, iA, jB, iB, score): int64 indices and float32 scores, each [b, topk * N].  Forward, for each of the
    N = hB*wB B cells the topk best A cells, rank-major (rank r of B cell s at r * N + s); inverted, for each of the
    N = hA*wA A cells the topk best B cells, cell-major (s * topk + r).  Ranks follow the raw value, descending, and
    exact ties go to the lowest flat cell index (the reference leaves their order to torch.topk)."""
    if not (isinstance(corr4d, torch.Tensor) and corr4d.is_cuda and corr4d.dtype == torch.float32
            and corr4d.dim() == 6 and corr4d.shape[1] == 1):
        raise ValueError('corr_to_matches_topk expects a [b, 1, hA, wA, hB, wB] float32 CUDA tensor')
    b, _, hA, wA, hB, wB = corr4d.shape
    n_slice, n = (hB * wB, hA * wA) if invert_matching_direction else (hA * wA, hB * wB)
    topk = int(topk)
    if not 1 <= topk <= n_slice:
        raise ValueError(f'topk must be in 1..{n_slice} (the cells of the other image), got {topk}')
    if n_slice > TOPK_MAX_SLICE:
        raise ValueError(f'slices of at most {TOPK_MAX_SLICE} cells are supported, got {n_slice}')
    if b > 65535:
        raise ValueError(f'batches of at most 65535 volumes are supported, got {b}')
    from .model import _pack_delta
    dev = corr4d.device
    h = _lib.default_handle(dev)
    code = None
    if delta4d is not None:
        if ksize not in (1, 2, 3):
            raise ValueError('ksize must be 1, 2 or 3 with delta4d')
        if len(delta4d) != 4 or any(tuple(d.shape) != tuple(corr4d.shape) for d in delta4d):
            raise ValueError('delta4d must be four tensors shaped like corr4d')
        delta4d = tuple(d.to(device=dev, dtype=torch.int64).contiguous() for d in delta4d)
    corr4d = corr4d.contiguous()
    out = [torch.empty(b, topk * n, dtype=torch.int64, device=dev) for _ in range(4)]
    score = torch.empty(b, topk * n, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        if delta4d is not None:
            code = _pack_delta(delta4d, ksize, h)
        _lib.check(h.lib.p2p_proposals_topk(h.h, _lib.ptr(corr4d), _lib.ptr(code), b, hA, wA, hB, wB, topk,
                                            ksize if code is not None else 1, int(bool(do_softmax)),
                                            int(bool(invert_matching_direction)), *[_lib.ptr(t) for t in out],
                                            _lib.ptr(score), h.stream()))
    return (*out, score)
