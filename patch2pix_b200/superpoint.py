"""SuperPoint keypoints and descriptors with exact nearest-neighbour matching, as the coarse matcher in front of
Patch2Pix's refiner ("SuperPoint + NN, refined by Patch2Pix").

The VGG-style encoder and the two heads run in PyTorch (cuDNN).  Everything after them runs in csrc/keypoints.cu:
softmax + depth-to-space, max-pool NMS, border and threshold, top-k and compaction (p2p_sp_keypoints), descriptor
sampling (p2p_sp_descriptors), and mutual nearest-neighbour matching of many descriptor-set pairs in one launch chain
(p2p_match_descriptors_batch), whose similarities are float64 sums in a fixed order, so its result is exact.

The conventions are those of SuperGlue's published SuperPoint (state_dict names, NMS, the descriptor sampling
coordinates); include/p2p_b200.h states them and oracle/superpoint_oracle.py restates them on the CPU.
"""
import ctypes as C
import math

import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from . import _lib

_CONVS = [('conv1a', 1, 64, 3), ('conv1b', 64, 64, 3), ('conv2a', 64, 64, 3), ('conv2b', 64, 64, 3),
          ('conv3a', 64, 128, 3), ('conv3b', 128, 128, 3), ('conv4a', 128, 128, 3), ('conv4b', 128, 128, 3),
          ('convPa', 128, 256, 3), ('convPb', 256, 65, 1), ('convDa', 128, 256, 3), ('convDb', 256, 256, 1)]


def _handle(device):
    return _lib.default_handle(device)


def _host_offsets(sizes):
    return np.concatenate([[0], np.cumsum(np.asarray(sizes, dtype=np.int64))]).astype(np.int64)


def _device_offsets(off, device):
    """int64 offsets on `device` without a host sync (pinned staging, asynchronous copy)."""
    return torch.from_numpy(off).pin_memory().to(device, non_blocking=True)


def detect_keypoints(logits, nms_radius=4, keypoint_threshold=0.005, max_keypoints=-1, remove_borders=4,
                     return_score_map=False):
    """p2p_sp_keypoints on the detector head's logits [B, 65, Hc, Wc] (fp32 CUDA) -> (keypoints: list of [N_b, 2]
    float32 (x, y), scores: list of [N_b] float32[, score map [B, 8Hc, 8Wc] float32]).  One host sync (the counts)."""
    if not (isinstance(logits, torch.Tensor) and logits.is_cuda and logits.dim() == 4 and logits.shape[1] == 65):
        raise ValueError('logits must be a [B, 65, Hc, Wc] CUDA tensor')
    _check_config(nms_radius, keypoint_threshold, max_keypoints, remove_borders)
    logits = logits.float().contiguous()
    B, _, hc, wc = logits.shape
    dev = logits.device
    hw = 64 * hc * wc
    cap = B * (hw if max_keypoints < 0 else min(max_keypoints, hw))
    kp = torch.empty(max(cap, 1), 2, dtype=torch.float32, device=dev)
    sc = torch.empty(max(cap, 1), dtype=torch.float32, device=dev)
    off = torch.empty(B + 1, dtype=torch.int64, device=dev)
    smap = torch.empty(B, 8 * hc, 8 * wc, dtype=torch.float32, device=dev) if return_score_map else None
    h = _handle(dev)
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_sp_keypoints(h.h, _lib.ptr(logits), B, hc, wc, int(nms_radius), float(keypoint_threshold),
                                          int(remove_borders), int(max_keypoints), _lib.ptr(smap), _lib.ptr(kp),
                                          _lib.ptr(sc), _lib.ptr(off), h.stream()))
    o = off.cpu().tolist()
    kps = [kp[o[b]:o[b + 1]] for b in range(B)]
    scs = [sc[o[b]:o[b + 1]] for b in range(B)]
    return (kps, scs, smap) if return_score_map else (kps, scs)


def sample_descriptors(desc, keypoints):
    """p2p_sp_descriptors: the raw descriptor head [B, D, Hc, Wc] (fp32 CUDA) sampled at each image's keypoints (a list
    of B [N_b, 2] (x, y) tensors) -> list of [N_b, D] float32, unit rows."""
    if not (isinstance(desc, torch.Tensor) and desc.is_cuda and desc.dim() == 4):
        raise ValueError('desc must be a [B, D, Hc, Wc] CUDA tensor')
    B, D, hc, wc = desc.shape
    if len(keypoints) != B:
        raise ValueError(f'need one keypoint tensor per image: {B} images, {len(keypoints)} keypoint sets')
    dev = desc.device
    sizes = [int(k.shape[0]) for k in keypoints]
    kp = torch.cat([k.to(device=dev, dtype=torch.float32).reshape(-1, 2) for k in keypoints]).contiguous()
    off = _device_offsets(_host_offsets(sizes), dev)
    n = sum(sizes)
    out = torch.empty(max(n, 1), D, dtype=torch.float32, device=dev)
    desc = desc.float().contiguous()
    h = _handle(dev)
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_sp_descriptors(h.h, _lib.ptr(desc), B, D, hc, wc, _lib.ptr(kp), _lib.ptr(off), n,
                                            _lib.ptr(out), h.stream()))
    o = _host_offsets(sizes)
    return [out[o[b]:o[b + 1]] for b in range(B)]


def _check_config(nms_radius, keypoint_threshold, max_keypoints, remove_borders):
    for v, n in ((nms_radius, 'nms_radius'), (max_keypoints, 'max_keypoints'), (remove_borders, 'remove_borders')):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError(f'{n} must be an int, got {v!r}')
    if not 0 <= nms_radius <= 16:
        raise ValueError(f'nms_radius must be in 0..16, got {nms_radius}')
    if remove_borders < 0:
        raise ValueError(f'remove_borders must be >= 0, got {remove_borders}')
    if not math.isfinite(float(keypoint_threshold)):
        raise ValueError(f'keypoint_threshold must be finite, got {keypoint_threshold}')


class SuperPoint(nn.Module):
    """SuperGlue's SuperPoint (inference, CUDA): forward({'image': grey [B, 1, H, W] in [0, 1]}) -> {'keypoints':
    [N, 2] float32 (x, y) integer pixels, 'scores': [N], 'descriptors': [256, N]} lists, one entry per image.
    Loads the state_dict names of SuperGlue's superpoint_v1.pth (conv1a.weight ... convDb.bias); nothing is downloaded,
    and forward raises until load_state_dict has been called."""

    def __init__(self, nms_radius=4, keypoint_threshold=0.005, max_keypoints=-1, remove_borders=4):
        super().__init__()
        _check_config(nms_radius, keypoint_threshold, max_keypoints, remove_borders)
        self.nms_radius, self.keypoint_threshold = int(nms_radius), float(keypoint_threshold)
        self.max_keypoints, self.remove_borders = int(max_keypoints), int(remove_borders)
        for name, cin, cout, k in _CONVS:
            setattr(self, name, nn.Conv2d(cin, cout, k, 1, k // 2))
        self._loaded = False
        super().train(False)

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._loaded = True
        return r

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('SuperPoint is inference-only here')
        return super().train(False)

    def heads(self, image):
        """The network on grey [B, 1, H, W] -> (detector logits [B, 65, H/8, W/8], raw descriptors [B, 256, ...])."""
        relu = F.relu
        x = image
        for i, stage in enumerate(('1', '2', '3', '4')):
            x = relu(getattr(self, f'conv{stage}a')(x))
            x = relu(getattr(self, f'conv{stage}b')(x))
            if i < 3:
                x = F.max_pool2d(x, 2, 2)
        return self.convPb(relu(self.convPa(x))), self.convDb(relu(self.convDa(x)))

    @torch.no_grad()
    def forward(self, data):
        if not self._loaded:
            raise RuntimeError('SuperPoint has no weights: call load_state_dict (nothing is downloaded)')
        image = data['image']
        if not (isinstance(image, torch.Tensor) and image.is_cuda and image.dim() == 4 and image.shape[1] == 1):
            raise ValueError('image must be a grey [B, 1, H, W] CUDA tensor')
        if image.shape[2] < 8 or image.shape[3] < 8:
            raise ValueError(f'image must be at least 8 x 8, got {tuple(image.shape[2:])}')
        logits, desc = self.heads(image.float())
        kps, scores = detect_keypoints(logits, self.nms_radius, self.keypoint_threshold, self.max_keypoints,
                                       self.remove_borders)
        descs = sample_descriptors(desc, kps)
        return {'keypoints': kps, 'scores': scores, 'descriptors': [d.t() for d in descs]}


def _check_sets(sets, what):
    out = []
    for t in sets:
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 2 and t.dtype == torch.float32):
            raise ValueError(f'{what} must be [N, D] float32 CUDA tensors')
        out.append(t.contiguous())
    return out


def _opt(v, name):
    if v is None:
        return math.nan
    v = float(v)
    if not math.isfinite(v):
        raise ValueError(f'{name} must be finite or None, got {v}')
    return v


def match_descriptors_batch(list0, list1, mutual=True, min_sim=None, ratio=None):
    """Nearest neighbours of each row of list0[k] among the rows of list1[k], for all k in one launch chain (semantics
    in include/p2p_b200.h, p2p_match_descriptors_batch).  -> list of (matches0 [N_k] int64, the index in list1[k] or
    -1, sim0 [N_k] float64, the similarity of an accepted row or 0), SuperGlue's matches0 / matching_scores0.  The
    similarity is a float64 sum in a fixed order, so the result is exact and element k equals
    match_descriptors(list0[k], list1[k]) bit for bit.  No host sync."""
    return _match_batch(list0, list1, mutual, min_sim, ratio)


def _match_batch(list0, list1, mutual, min_sim, ratio, probe=None):
    """match_descriptors_batch; with a dict `probe`, also fills it with the tensor-core pass's own numbers:
    'tc_sim' / 'tc_idx' (each row's best similarity and column before the float64 fix-up), 'eps' (the per-pair bound
    of |s_tc - s_fp64|) and 'n_fixed' (rows, columns redone in float64)."""
    if len(list0) != len(list1) or len(list0) == 0:
        raise ValueError('need the same, non-zero number of sets on both sides')
    list0, list1 = _check_sets(list0, 'list0'), _check_sets(list1, 'list1')
    dims = {int(t.shape[1]) for t in list0 + list1}
    devs = {t.device for t in list0 + list1}
    if len(dims) != 1 or len(devs) != 1:
        raise ValueError('all descriptor sets must share one dimension and one device')
    D, dev = dims.pop(), devs.pop()
    if ratio is not None and not float(ratio) >= 0:
        raise ValueError(f'ratio must be >= 0, got {ratio}')
    ms, rt = _opt(min_sim, 'min_sim'), _opt(ratio, 'ratio')
    n0, n1 = [int(t.shape[0]) for t in list0], [int(t.shape[0]) for t in list1]
    o0, o1 = _host_offsets(n0), _host_offsets(n1)
    d0, d1 = torch.cat(list0), torch.cat(list1)
    match = torch.empty(max(int(o0[-1]), 1), dtype=torch.int32, device=dev)
    sim = torch.empty(max(int(o0[-1]), 1), dtype=torch.float64, device=dev)
    h = _handle(dev)
    pr = [None] * 4
    if probe is not None:
        n = max(int(o0[-1]), 1)
        pr = [torch.zeros(n, dtype=torch.float64, device=dev), torch.zeros(n, dtype=torch.int32, device=dev),
              torch.zeros(len(list0), dtype=torch.float64, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)]
        probe.update(zip(('tc_sim', 'tc_idx', 'eps', 'n_fixed'), pr))
    with torch.cuda.device(dev):
        g0, g1 = _device_offsets(o0, dev), _device_offsets(o1, dev)
        _lib.check(h.lib.p2p_match_descriptors_batch(
            h.h, _lib.ptr(d0), _lib.ptr(d1), _lib.ptr(g0), _lib.ptr(g1), o0.ctypes.data_as(C.POINTER(C.c_int64)),
            o1.ctypes.data_as(C.POINTER(C.c_int64)), len(list0), D, int(bool(mutual)), ms, rt, _lib.ptr(match),
            _lib.ptr(sim), *(_lib.ptr(t) for t in pr), h.stream()))
    m64 = match.long()
    return [(m64[o0[k]:o0[k + 1]], sim[o0[k]:o0[k + 1]]) for k in range(len(list0))]


def match_descriptors(d0, d1, mutual=True, min_sim=None, ratio=None):
    """match_descriptors_batch for one pair: d0 [N, D], d1 [M, D] float32 CUDA -> (matches0 [N] int64, sim0 [N]
    float64)."""
    return match_descriptors_batch([d0], [d1], mutual, min_sim, ratio)[0]


def superpoint_nn_matcher(sp, **match_opts):
    """The coarse_matcher(grey1, grey2) -> [N, 4] float32 (x1, y1, x2, y2) rows that eval_helper.refine_matches takes:
    SuperPoint `sp` on both grey images, then match_descriptors(**match_opts) (mutual nearest neighbours by default)."""
    def matcher(grey1, grey2):
        if grey1.shape == grey2.shape:
            out = sp({'image': torch.cat([grey1, grey2])})
            k0, k1 = out['keypoints']
            e0, e1 = (d.t() for d in out['descriptors'])
        else:
            a, b = sp({'image': grey1}), sp({'image': grey2})
            k0, k1 = a['keypoints'][0], b['keypoints'][0]
            e0, e1 = a['descriptors'][0].t(), b['descriptors'][0].t()
        m, _ = match_descriptors(e0.contiguous(), e1.contiguous(), **match_opts)
        keep = m >= 0
        return torch.cat([k0[keep], k1[m[keep]]], 1)
    return matcher


def sp_patch2pix_matcher(net, sp, io_thres=0.0, imsize=None, sg=None):
    """The (path0, path1) -> [N, 4] float64 rows callable that eval_hpatches / eval_relpose / localize_* take:
    SuperPoint + mutual nearest-neighbour matches refined by the Patch2Pix `net` (eval_helper.refine_matches).  With a
    SuperGlue `sg`, SuperGlue's matches (superglue.superglue_matcher) are refined instead."""
    from .eval_helper import refine_matches
    if sg is None:
        coarse = superpoint_nn_matcher(sp)
    else:
        from .superglue import superglue_matcher
        coarse = superglue_matcher(sp, sg)

    def matcher(path0, path1):
        return refine_matches(path0, path1, net, coarse, io_thres, imsize)[0]
    return matcher
