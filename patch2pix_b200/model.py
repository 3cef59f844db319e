"""Host-side mirror of the reference's `Patch2Pix` model object for the hot path.

Same constructor config, same method names, same argument meaning and return shapes as
`networks/patch2pix.py` (reference file:line cited per method), with the computation done by
libp2p_b200.so (hand-written sm_90a kernels) instead of eager PyTorch:

    forward_coarse_match   networks/patch2pix.py:120-136
    cal_coarse_matches     networks/patch2pix.py:340-375
    filter_coarse          networks/utils.py:38-72          (module-level function, as in the reference)
    shift_to_anchors       networks/patch2pix.py:377-402
    forward_fine_match     networks/patch2pix.py:186-218
    forward / predict_coarse / predict_fine / refine_matches   networks/patch2pix.py:220-318

PyTorch tensors in, PyTorch tensors out.  The ResNet34 pyramid that feeds the path stays
PyTorch/cuDNN (backbone.py).  There is no CPU or eager fallback: a missing CUDA library or a
non-CUDA device raises.
"""
import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .backbone import ResNet34Features

BN_EPS = 1e-5


# ----------------------------------------------------------------------------------------------
# stateless ops (weight-free kernels)
# ----------------------------------------------------------------------------------------------
def _check_cuda_f32(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        raise RuntimeError(f'{name} must be a CUDA float32 tensor (no CPU fallback)')
    return t.contiguous()


def _feat_format(t, name):
    """0: contiguous NCHW fp32 (the reference's layout); 1: channels-last fp16 (the fast backbone of the end-to-end path)."""
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError(f'{name} must be a CUDA tensor (no CPU fallback)')
    if t.dtype == torch.float32:
        return 0
    if t.dtype == torch.float16 and t.dim() >= 3 and t.permute(*range(t.dim() - 3), -2, -1, -3).is_contiguous():
        return 1
    raise RuntimeError(f'{name} must be float32 NCHW or channels-last float16')


class _PinnedPool:
    """Recycled pinned int32 staging buffers.  A per-step `torch.empty(pin_memory=True)` can fall through PyTorch's
    caching host allocator to cudaHostAlloc (page locking: anything from hundreds of microseconds to hundreds of
    milliseconds on a loaded host, and serialising) whenever the cached block is still marked in use; here a buffer
    returns to the pool with the event after which it may be rewritten, and the pool grows eight buffers at a time
    from ONE pinned allocation, so a steady-state loop never page-locks memory."""

    def __init__(self):
        self._free = {}
        self._slabs = []

    def get(self, n):
        lst = self._free.setdefault(n, [])
        for i, (t, ev) in enumerate(lst):
            if ev is None or ev.query():
                lst.pop(i)
                if ev is not None:
                    _events.put(ev)
                return t
        slab = torch.empty(8 * n, dtype=torch.int32).pin_memory()
        self._slabs.append(slab)
        views = list(slab.view(8, n).unbind(0))
        lst.extend((v, None) for v in views[1:])
        return views[0]

    def put(self, t, ev=None):
        self._free.setdefault(t.numel(), []).append((t, ev))


class _EventPool:
    """Recycled CUDA events (one per ticket / staging copy), per device: no event creation in a steady-state loop."""

    def __init__(self):
        self._free = {}

    def get(self, device):
        ev = None
        lst = self._free.get(torch.device(device).index)
        if lst:
            ev = lst.pop()
        if ev is None:
            ev = torch.cuda.Event()
        ev._p2p_dev = torch.device(device).index
        return ev

    def put(self, ev):
        lst = self._free.setdefault(getattr(ev, '_p2p_dev', None), [])
        if len(lst) < 256:
            lst.append(ev)


_pinned = _PinnedPool()
_events = _EventPool()


class _UniqueTicket:
    """unique_rows in flight: ids buffer on the device, counters on their way to pinned host memory.
    Every ticket owns its pinned counter buffer (taken from / returned to a pool), so any number of tickets can be
    outstanding."""

    def __init__(self, ids, cnt_host, event, thres):
        self.ids, self.cnt_host, self.event, self.thres = ids, cnt_host, event, thres
        self.n = self.n_pass_selected = self.n_pass_all = None

    def wait_count(self):
        """-> number of ids (the one host sync of filter_coarse; the reference syncs here too: utils.py:42)."""
        if self.n is None:
            self.event.synchronize()
            self.n, bad, self.n_pass_selected, self.n_pass_all = self.cnt_host.tolist()
            _pinned.put(self.cnt_host)           # the copy has completed: the buffer may be reused at once
            _events.put(self.event)
            self.cnt_host = self.event = None
            if bad:
                raise RuntimeError('filter_coarse: match coordinates must lie in [0, 65535]')
        return self.n

    def wait(self):
        return self.ids[:self.wait_count()].long()


def unique_rows_submit(rows, mutual=True, handle=None, scores=None, thres=0.0):
    if not (rows.is_cuda and rows.dtype == torch.int64 and rows.dim() == 2 and rows.shape[1] == 4):
        raise RuntimeError('unique_rows expects a CUDA int64 [n,4] tensor')
    rows = rows.contiguous()
    n = rows.shape[0]
    h = handle or _lib.default_handle(rows.device)
    ids = torch.empty(max(n, 1), dtype=torch.int32, device=rows.device)
    cnt = torch.empty(4, dtype=torch.int32, device=rows.device)
    cnt_host = _pinned.get(4)
    if scores is not None:
        scores = _check_cuda_f32(scores.flatten(), 'scores')
    with torch.cuda.device(rows.device):
        _lib.check(h.lib.p2p_unique_rows(h.h, _lib.ptr(rows), n, int(bool(mutual)), _lib.ptr(scores), float(thres),
                                         _lib.ptr(ids), _lib.ptr(cnt), h.stream()))
        cnt_host.copy_(cnt, non_blocking=True)
        ev = _events.get(rows.device)
        ev.record(torch.cuda.current_stream(rows.device))
    return _UniqueTicket(ids, cnt_host, ev, float(thres) if scores is not None else None)


def unique_rows(rows, mutual=True, handle=None):
    """Device-side np.unique(rows, axis=0, return_index, return_counts): lexicographically ordered
    first-occurrence indices of distinct rows (mutual: rows seen more than once)."""
    return unique_rows_submit(rows, mutual, handle).wait()


def _select_anchor(rows, scores, ids, sel, m, panc, pshift, handle=None):
    """One launch: out row r <- rows[ids[sel[r]]] (+ scores) and, for panc 8, the 8-anchor expansion
    (networks/utils.py:51-69 index arithmetic + networks/patch2pix.py:377-402)."""
    h = handle or _lib.default_handle(rows.device)
    dev = rows.device
    out_m = torch.empty(m, 4, dtype=torch.int64, device=dev)
    out_s = torch.empty(m, dtype=torch.float32, device=dev) if scores is not None else None
    anch = torch.empty(m * 8, 4, dtype=torch.int64, device=dev) if panc == 8 else None
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_select_anchor(h.h, _lib.ptr(rows), _lib.ptr(scores), _lib.ptr(ids), _lib.ptr(sel), m, panc,
                                           int(pshift), _lib.ptr(out_m), _lib.ptr(out_s), _lib.ptr(anch), h.stream()))
    return out_m, out_s, anch


def _filter_coarse_core(coarse_matches, match_scores, ncn_thres, mutual, ptmax, tickets, anchor):
    """filter_coarse (networks/utils.py:38-72) with np.unique on the device; `anchor` = (panc, pshift) additionally
    returns shift_to_anchors of the result from the same launch.  Quirks kept: lexicographic output order,
    first-occurrence scores, 'skip a filter that would empty the set', degenerate [0,0,0,0] ids and the
    global-numpy-RNG shuffle/tile for ptmax (drawn on the host from the same count as the reference)."""
    matches, scores, anchors = [], [], []
    panc, pshift = anchor if anchor is not None else (1, 0)
    for ib, (imatches, iscores) in enumerate(zip(coarse_matches, match_scores)):
        if not (isinstance(imatches, torch.Tensor) and imatches.is_cuda):
            raise RuntimeError('filter_coarse expects CUDA tensors (no CPU fallback)')
        tk = tickets[ib] if tickets is not None else unique_rows_submit(imatches, mutual, None, iscores, ncn_thres)
        n = tk.wait_count()
        n_rows = n if n > 0 else imatches.shape[0]            # rows left after the (possibly skipped) mutual step
        n_pass = tk.n_pass_selected if n > 0 else tk.n_pass_all
        fast = tk.thres == float(ncn_thres) and n_pass == n_rows and n_rows > 0 and imatches.dtype == torch.int64
        if fast:
            # every row passes the score threshold (the normal case: softmax scores > 0): the second index list is
            # arange(n_rows) and the whole selection is one gather launch
            ids = tk.ids if n > 0 else None
            sel, m = None, n_rows
            if ptmax:
                iids = np.arange(n_rows)
                np.random.shuffle(iids)
                iids = np.tile(iids, (ptmax // n_rows + 1))[:ptmax]
                stage = _pinned.get(int(ptmax))
                stage.numpy()[:] = iids
                sel, m = stage.to(imatches.device, non_blocking=True), int(ptmax)
                ev = _events.get(imatches.device)
                ev.record(torch.cuda.current_stream(imatches.device))
                _pinned.put(stage, ev)           # reusable once the host-to-device copy has executed
            if ids is None and sel is None and panc == 1:
                om, osc, an = imatches, iscores, None       # nothing filtered: the input passes unchanged
            else:
                om, osc, an = _select_anchor(imatches.contiguous(), _check_cuda_f32(iscores.flatten(), 'scores'), ids, sel, m,
                                             panc, pshift)
        else:
            ids = tk.ids[:n].long()
            if len(ids) > 0:
                iscores = iscores[ids]
                imatches = imatches[ids]
            ids = torch.nonzero(iscores.flatten() > ncn_thres, as_tuple=False).flatten()
            if ptmax:
                if len(ids) == 0:
                    ids = torch.tensor([0, 0, 0, 0]).long()
                iids = np.arange(len(ids))
                np.random.shuffle(iids)
                iids = np.tile(iids, (ptmax // len(ids) + 1))[:ptmax]
                ids = ids.to(imatches.device)[torch.from_numpy(iids).to(imatches.device)]
            if len(ids) > 0:
                iscores = iscores[ids]
                imatches = imatches[ids]
            om, osc, an = imatches, iscores, None
            if panc == 8:
                an = (om.unsqueeze(1) + _anchor_template(om.device, pshift)).reshape(-1, 4)
        matches.append(om)
        scores.append(osc)
        anchors.append(an if panc == 8 else om)
    return matches, scores, anchors


_tmpl_cache = {}


def _anchor_template(device, p):
    key = (str(device), int(p))
    if key not in _tmpl_cache:
        _tmpl_cache[key] = torch.tensor([[-p, -p, 0, 0], [p, -p, 0, 0], [-p, p, 0, 0], [p, p, 0, 0],
                                         [0, 0, -p, -p], [0, 0, p, -p], [0, 0, -p, p], [0, 0, p, p]], device=device)
    return _tmpl_cache[key]


def filter_coarse(coarse_matches, match_scores, ncn_thres=0.0, mutual=True, ptmax=None, _tickets=None):
    """networks/utils.py:38-72 with the np.unique step and the index arithmetic on the device."""
    m, s, _ = _filter_coarse_core(coarse_matches, match_scores, ncn_thres, mutual, ptmax, _tickets, None)
    return m, s


def mutual_matching(corr4d, handle=None):
    """MutualMatching, networks/ncn/model.py:157-176.  corr4d [b,1,hA,wA,hB,wB]."""
    corr4d = _check_cuda_f32(corr4d, 'corr4d')
    b, _, hA, wA, hB, wB = corr4d.shape
    h = handle or _lib.default_handle(corr4d.device)
    out = torch.empty_like(corr4d)
    with torch.cuda.device(corr4d.device):
        for i in range(b):
            _lib.check(h.lib.p2p_mutual_matching(h.h, _lib.ptr(corr4d[i]), hA * wA, hB * wB, _lib.ptr(out[i]), h.stream()))
    return out


def _pack_delta(delta4d, ksize, h):
    di, dj, dk, dl = [d.contiguous() for d in delta4d]
    code = torch.empty(di.shape, dtype=torch.uint8, device=di.device)
    _lib.check(h.lib.p2p_delta_pack(h.h, _lib.ptr(di), _lib.ptr(dj), _lib.ptr(dk), _lib.ptr(dl), di.numel(), ksize,
                                    _lib.ptr(code), h.stream()))
    return code


class _FeatList(list):
    """Feature pyramid list that remembers the CUDA-graph instance whose static buffers it views."""
    graph_inst = None


class _DeltaTuple(tuple):
    """The reference's (max_i, max_j, max_k, max_l) int64 tuple; also carries the packed code so
    that cal_coarse_matches does not have to re-pack it."""
    code = None


def cal_coarse_matches(corr4d, delta4d, ksize=1, do_softmax=True, upsample=16, sort=False, center=True, pshift=0,
                       handle=None):
    """Patch2Pix.cal_coarse_matches, networks/patch2pix.py:340-375 -> (matches [b,N,4] int64, scores [b,N])."""
    corr4d = _check_cuda_f32(corr4d, 'corr4d')
    b, _, hA, wA, hB, wB = corr4d.shape
    h = handle or _lib.default_handle(corr4d.device)
    n = hA * wA + hB * wB
    matches = torch.empty(b, n, 4, dtype=torch.int64, device=corr4d.device)
    scores = torch.empty(b, n, dtype=torch.float32, device=corr4d.device)
    with torch.cuda.device(corr4d.device):
        code = None
        if delta4d is not None:
            code = getattr(delta4d, 'code', None)
            if code is None:
                code = _pack_delta(delta4d, ksize, h)
        for i in range(b):
            _lib.check(h.lib.p2p_proposals(h.h, _lib.ptr(corr4d[i]), _lib.ptr(code[i]) if code is not None else None,
                                           hA, wA, hB, wB, ksize if code is not None else 1, int(upsample),
                                           int(bool(center)), int(bool(do_softmax)), _lib.ptr(matches[i]),
                                           _lib.ptr(scores[i]), h.stream()))
    if sort:
        order = torch.sort(-scores)[1]
        matches = torch.gather(matches, 1, order.unsqueeze(-1).expand(-1, -1, 4))
        scores = torch.gather(scores, 1, order)
    return matches, scores


# ----------------------------------------------------------------------------------------------
# parameter containers with the reference's state_dict names (never called in the product path)
# ----------------------------------------------------------------------------------------------
class _Conv4dParams(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(3, cout, cin, 3, 3, 3))   # pre-permuted [k1,Cout,Cin,k2,k3,k4]
        self.bias = nn.Parameter(torch.zeros(cout))


class _NcnParams(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.ModuleDict({'0': _Conv4dParams(1, 16), '2': _Conv4dParams(16, 1)})


class _RegressorParams(nn.Module):
    def __init__(self, feat_dim=518):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(feat_dim, 512, 3, 2, 1, bias=False), nn.BatchNorm2d(512),
                                  nn.Conv2d(512, 512, 3, 1, 1, bias=False), nn.BatchNorm2d(512),
                                  nn.ReLU(), nn.MaxPool2d(8))
        self.fc = nn.Sequential(nn.Linear(512, 512), nn.BatchNorm1d(512), nn.ReLU(),
                                nn.Linear(512, 256), nn.BatchNorm1d(256), nn.ReLU(), nn.Linear(256, 5))

    def forward(self, *a, **k):
        raise RuntimeError('regressor parameters are consumed by libp2p_b200; there is no eager path')


def refine_level_shapes(H, W):
    """Shapes of the pyramid levels 0..3 the refine stage reads for an H x W image, as the backbone produces them:
    the image [3,H,W], then each stride-2 layer rounds up (h1 = ceil(H/2), h2 = ceil(h1/2), h3 = ceil(h2/2)).
    Below 8 px the reference's level-3 clamp bound W // 8 - 1 is negative and its index wraps around, so such
    sizes are refused."""
    H, W = int(H), int(W)
    if H < 8 or W < 8:
        raise RuntimeError(f'the refine stage needs images of at least 8 x 8 pixels, got {H} x {W}')
    shapes = [(3, H, W)]
    for c in (64, 64, 128):
        H, W = (H + 1) // 2, (W + 1) // 2
        shapes.append((c, H, W))
    return shapes


def _host_f32(t):
    return t.detach().to('cpu', torch.float32).contiguous()


class Patch2PixB200(nn.Module):
    """Drop-in for `networks.patch2pix.Patch2Pix` (inference). Config fields as in
    utils/eval/model_helper.py:32-46: training(False), device, regr_batch, backbone('ResNet34'),
    feat_idx([0,1,2,3]), weights_dict, regressor_config(Namespace|None), change_stride(True)."""

    def __init__(self, config):
        super().__init__()
        if getattr(config, 'training', False):
            raise RuntimeError('Patch2PixB200 implements the inference path only (config.training must be False)')
        self.device = torch.device(config.device)
        if self.device.type != 'cuda':
            raise RuntimeError('Patch2PixB200 needs a CUDA (sm_90a) device; there is no CPU fallback')
        if config.backbone != 'ResNet34':
            raise RuntimeError('only the ResNet34 backbone of the released model is supported')
        self.backbone = config.backbone
        self.change_stride = config.change_stride
        self.upsample = 8 if self.change_stride else 16
        self.feats_downsample = [1, 2, 2, 2, 1 if self.change_stride else 2]
        self.extract = ResNet34Features(change_stride=self.change_stride)
        self.ncn = _NcnParams()
        self.regressor_config = config.regressor_config
        if not self.regressor_config:
            self.regress_mid = None
            self.regress_fine = None
        else:
            rc = self.regressor_config
            if list(config.feat_idx) != [0, 1, 2, 3] or list(rc.psize) != [16, 16] or rc.feat_comb != 'pre' \
                    or list(rc.conv_dims) != [512, 512] or list(rc.conv_kers) != [3, 3] or list(rc.conv_strs) != [2, 1] \
                    or list(rc.fc_dims) != [512, 256] or not self.change_stride:
                raise RuntimeError('the CUDA path is specialised to the released regressor configuration '
                                   '(feat_idx [0,1,2,3], psize 16, conv 512-512 k3 s2/s1, fc 512-256, feat_comb pre)')
            self.regr_batch = config.regr_batch
            self.feat_idx = list(config.feat_idx)
            self.ptype = ['center', 'center']
            self.psize = list(rc.psize)
            self.pshift = rc.pshift
            self.panc = rc.panc
            self.shared = rc.shared
            self.regress_mid = _RegressorParams()
            self.regress_fine = self.regress_mid if self.shared else _RegressorParams()
        self.to(self.device)
        self.eval()
        self._handle = _lib.Handle(self.device)
        self._packed = False
        if getattr(config, 'weights_dict', None):
            sd = config.weights_dict
            missing, unexpected = self.load_state_dict(sd, strict=False)
            missing = [k for k in missing if 'num_batches_tracked' not in k]
            if missing:
                raise RuntimeError(f'weights_dict lacks {len(missing)} parameters, e.g. {missing[:3]}')

    # -- weights -------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._packed = False
        object.__setattr__(self, '_extract_half', None)
        return r

    def train(self, mode=True):
        if mode:
            raise RuntimeError('Patch2PixB200 is inference-only (BatchNorm is folded in eval mode)')
        return super().train(False)

    def set_option(self, key, value):
        self._handle.set_option(key, value)

    def pack_weights(self):
        """Push ncn / regressor parameters into the C library (BN folding, fp16 hi/lo split, re-layout)."""
        h = self._handle
        keep = [_host_f32(self.ncn.conv['0'].weight), _host_f32(self.ncn.conv['0'].bias),
                _host_f32(self.ncn.conv['2'].weight), _host_f32(self.ncn.conv['2'].bias)]
        _lib.check(h.lib.p2p_set_ncn_weights(h.h, *[_lib.ptr(t) for t in keep]))
        if self.regress_mid is not None:
            for which, reg in enumerate((self.regress_mid, self.regress_fine)):
                hold = []

                def hp(t):
                    t = _host_f32(t)
                    hold.append(t)
                    return t.data_ptr()

                def bn(m):
                    return _lib.BN(hp(m.weight), hp(m.bias), hp(m.running_mean), hp(m.running_var))
                w = _lib.RegressorWeights(hp(reg.conv[0].weight), bn(reg.conv[1]), hp(reg.conv[2].weight), bn(reg.conv[3]),
                                          hp(reg.fc[0].weight), hp(reg.fc[0].bias), bn(reg.fc[1]),
                                          hp(reg.fc[3].weight), hp(reg.fc[3].bias), bn(reg.fc[4]),
                                          hp(reg.fc[6].weight), hp(reg.fc[6].bias), BN_EPS)
                _lib.check(h.lib.p2p_set_regressor_weights(h.h, which, C.byref(w)))
        self._packed = True

    def _ready(self):
        if not self._packed:
            self.pack_weights()
        return self._handle

    # -- coarse --------------------------------------------------------------------------------
    def _coarse_raw(self, feat1, feat2, ksize, return_stages=False):
        h = self._ready()
        fmt = _feat_format(feat1, 'feat1')
        if _feat_format(feat2, 'feat2') != fmt:
            raise RuntimeError('feat1 and feat2 must share dtype / memory format')
        if fmt == 0:
            feat1, feat2 = feat1.contiguous(), feat2.contiguous()
        entry = h.lib.p2p_coarse if fmt == 0 else h.lib.p2p_coarse_nhwc16
        b, c, h1, w1 = feat1.shape
        _, _, h2, w2 = feat2.shape
        hA, wA, hB, wB = h1 // ksize, w1 // ksize, h2 // ksize, w2 // ksize
        dev = feat1.device
        corr4d = torch.empty(b, 1, hA, wA, hB, wB, dtype=torch.float32, device=dev)
        code = torch.empty(b, 1, hA, wA, hB, wB, dtype=torch.uint8, device=dev) if ksize > 1 else None
        pooled = torch.empty_like(corr4d) if return_stages else None
        ncn = torch.empty_like(corr4d) if return_stages else None
        with torch.cuda.device(dev):
            for i in range(b):
                _lib.check(entry(h.h, _lib.ptr(feat1[i]), _lib.ptr(feat2[i]), c, h1, w1, h2, w2, ksize,
                                            _lib.ptr(corr4d[i]), _lib.ptr(code[i]) if code is not None else None,
                                            _lib.ptr(pooled[i]) if pooled is not None else None,
                                            _lib.ptr(ncn[i]) if ncn is not None else None, h.stream()))
        if return_stages:
            return corr4d, code, {'pooled': pooled, 'ncn': ncn}
        return corr4d, code

    def forward_coarse_match(self, feat1, feat2, ksize=1, return_stages=False):
        """networks/patch2pix.py:120-136 -> (corr4d [b,1,hA,wA,hB,wB] f32, delta4d 4 x int64 | None)."""
        r = self._coarse_raw(feat1, feat2, ksize, return_stages)
        corr4d, code = r[0], r[1]
        h = self._handle
        delta4d = None
        if ksize > 1:
            with torch.cuda.device(corr4d.device):
                ds = [torch.empty(code.shape, dtype=torch.int64, device=code.device) for _ in range(4)]
                _lib.check(h.lib.p2p_delta_unpack(h.h, _lib.ptr(code), code.numel(), ksize, *[_lib.ptr(d) for d in ds],
                                                  h.stream()))
            delta4d = _DeltaTuple(ds)
            delta4d.code = code
        if return_stages:
            return corr4d, delta4d, r[2]
        return corr4d, delta4d

    def cal_coarse_matches(self, corr4d, delta4d, ksize=1, do_softmax=True, upsample=16, sort=False, center=True,
                           pshift=0):
        return cal_coarse_matches(corr4d, delta4d, ksize, do_softmax, upsample, sort, center, pshift, self._handle)

    def shift_to_anchors(self, matches):
        """networks/patch2pix.py:377-402 (8-row template)."""
        if self.panc == 1:
            return matches
        out = []
        for m in matches:
            if m.is_cuda and m.dtype == torch.int64 and m.dim() == 2 and m.shape[1] == 4:
                out.append(_select_anchor(m.contiguous(), None, None, None, m.shape[0], 8, self.pshift, self._handle)[2])
            else:
                out.append((m.unsqueeze(1) + _anchor_template(m.device, self.pshift)).reshape(-1, 4))
        return out

    # -- refine --------------------------------------------------------------------------------
    def _which(self, regressor):
        if regressor is self.regress_mid:
            return 0
        if regressor is self.regress_fine:
            return 1
        raise RuntimeError('regressor must be self.regress_mid or self.regress_fine')

    def _prepare_pair(self, feats1, feats2, ibatch):
        h = self._handle
        fmt = _feat_format(feats1[1], 'feats1[1]')
        lvs = []
        for feats, nm in ((feats1, 'feats1'), (feats2, 'feats2')):
            lv = [_check_cuda_f32(feats[0][ibatch], f'{nm}[0]')]
            for l in range(1, 4):
                if _feat_format(feats[l], f'{nm}[{l}]') != fmt:
                    raise RuntimeError('all pyramid levels must share dtype / memory format')
                t = feats[l][ibatch]
                lv.append(t.contiguous() if fmt == 0 else t)     # a channels-last fp16 item is dense as [h][w][C]
            lvs.append(lv)
        lv1, lv2 = lvs
        _, H1, W1 = lv1[0].shape
        _, H2, W2 = lv2[0].shape
        for lv, H, W in ((lv1, H1, W1), (lv2, H2, W2)):
            exp = refine_level_shapes(H, W)
            if [tuple(t.shape) for t in lv] != exp:
                raise RuntimeError(f'feature pyramid shapes {[tuple(t.shape) for t in lv]} do not match {exp}')
        a1 = (C.c_void_p * 4)(*[t.data_ptr() for t in lv1])
        a2 = (C.c_void_p * 4)(*[t.data_ptr() for t in lv2])
        entry = h.lib.p2p_refine_prepare if fmt == 0 else h.lib.p2p_refine_prepare_nhwc16
        _lib.check(entry(h.h, a1, a2, H1, W1, H2, W2, h.stream()))
        return lv1, lv2   # keep alive until the refine kernels have been enqueued

    def forward_fine_match(self, feats1, feats2, coarse_matches, psize=16, ptype='center', regressor=None,
                           _prepared=None):
        """networks/patch2pix.py:186-218 -> (list of [N,4] f32, list of [N] f32).  The reference's
        regr_batch chunking is numerically neutral in eval mode and is not needed here; its
        `.squeeze()` of multi-chunk results is reproduced."""
        if psize != 16 or ptype != 'center':
            raise RuntimeError('the CUDA path is specialised to psize 16, ptype center')
        h = self._ready()
        which = self._which(regressor)
        fine, probs = [], []
        with torch.cuda.device(self.device):
            for ib, im in enumerate(coarse_matches):
                if not im.is_cuda:
                    raise RuntimeError('coarse matches must be CUDA tensors')
                if im.dtype == torch.int64:
                    is_float = 0
                elif im.dtype == torch.float32:
                    is_float = 1
                else:
                    raise RuntimeError('coarse matches must be int64 or float32')
                im = im.contiguous()
                n = im.shape[0]
                keep = None
                if _prepared is None or _prepared != ib:
                    keep = self._prepare_pair(feats1, feats2, ib)
                out = torch.empty(n, 4, dtype=torch.float32, device=self.device)
                pr = torch.empty(n, dtype=torch.float32, device=self.device)
                _lib.check(h.lib.p2p_refine(h.h, which, _lib.ptr(im), is_float, n, _lib.ptr(out), _lib.ptr(pr),
                                            h.stream()))
                del keep
                if n > self.regr_batch:
                    out, pr = out.squeeze(), pr.squeeze()
                fine.append(out)
                probs.append(pr)
        return fine, probs

    # -- orchestration -------------------------------------------------------------------------
    def forward(self, im1, im2, ksize=1, return_feats=False):
        """networks/patch2pix.py:220-237."""
        feat1s = self.extract.forward_all(im1, [], early_feat=True)
        feat2s = self.extract.forward_all(im2, [], early_feat=True)
        corr4d, delta4d = self.forward_coarse_match(feat1s[-1], feat2s[-1], ksize=ksize)
        if return_feats:
            return corr4d, delta4d, feat1s, feat2s
        return corr4d, delta4d

    def predict_coarse(self, im1, im2, ksize=2, ncn_thres=0.0, mutual=False, center=True):
        """networks/patch2pix.py:240-248."""
        corr4d, delta4d = self.forward(im1, im2, ksize)
        cm, sc = self.cal_coarse_matches(corr4d, delta4d, ksize=ksize, upsample=self.upsample, center=center)
        return filter_coarse(cm, sc, ncn_thres, mutual)

    def submit_coarse(self, feats1, feats2, ksize=2, mutual=True, ncn_thres=0.0):
        """First half of match_from_feats: enqueue correlation .. proposals and the device-side
        unique/mutual pass, start the asynchronous read-back of the mutual-match count and return a
        ticket.  Nothing here waits for the GPU, so the caller can keep a second pair in flight."""
        corr4d, code = self._coarse_raw(feats1[-1], feats2[-1], ksize)
        delta = None
        if code is not None:
            delta = _DeltaTuple(())
            delta.code = code
        cm, sc = self.cal_coarse_matches(corr4d, delta, ksize=ksize, upsample=self.upsample, center=True)
        tickets = [unique_rows_submit(m, mutual, self._handle, sc_i, ncn_thres) for m, sc_i in zip(cm, sc)]
        inst = getattr(feats1, 'graph_inst', None)
        if inst is not None:
            inst['pending'] += 1          # the ticket reads the graph instance's static output buffers until finish_match
        return {'feats1': feats1, 'feats2': feats2, 'cm': cm, 'sc': sc, 'tickets': tickets, 'mutual': mutual, 'inst': inst}

    @staticmethod
    def _release(ticket):
        inst = ticket.get('inst')
        if inst is not None:
            inst['pending'] -= 1
            ticket['inst'] = None
            if inst['pending'] == 0:
                # every kernel that reads this instance's pyramids is enqueued on the current stream: a replay on the
                # side stream (overlap mode) may overwrite them once this point has executed
                dev = inst['inp'].device
                old = inst.get('free')
                ev = _events.get(dev)
                ev.record(torch.cuda.current_stream(dev))
                inst['free'] = ev
                if old is not None:
                    _events.put(old)

    def finish_match(self, ticket, ncn_thres=0.0, ptmax=None, return_all=False):
        """Second half: wait for the count, run filter_coarse's host logic (numpy RNG sampling for
        ptmax exactly as the reference), shift to anchors, mid and fine refine."""
        feats1, feats2, cm, sc = ticket['feats1'], ticket['feats2'], ticket['cm'], ticket['sc']
        anchor = (self.panc, self.pshift)
        if ptmax:
            if self.panc > 1 and ptmax > 0:
                _, _, cm = _filter_coarse_core(cm, sc, 0.0, True, ptmax, ticket['tickets'] if ticket['mutual'] else None, anchor)
            else:
                cm = self.shift_to_anchors(cm)
        else:
            _, _, cm = _filter_coarse_core(cm, sc, ncn_thres, ticket['mutual'], None, ticket['tickets'], anchor)
        single = len(cm) == 1
        if single:
            self._ready()
            with torch.cuda.device(self.device):
                keep = self._prepare_pair(feats1, feats2, 0)
        mid, mid_p = self.forward_fine_match(feats1, feats2, cm, self.psize[0], self.ptype[0], self.regress_mid,
                                             _prepared=0 if single else None)
        fine, fine_p = self.forward_fine_match(feats1, feats2, mid, self.psize[1], self.ptype[1], self.regress_fine,
                                               _prepared=0 if single else None)
        if single:
            del keep
        self._release(ticket)          # everything that reads the pyramids has been enqueued (stream order protects it)
        if return_all:
            return fine, fine_p, mid, mid_p, cm
        return fine, fine_p, cm

    def match_from_feats(self, feats1, feats2, ksize=2, ncn_thres=0.0, mutual=True, ptmax=None, return_all=False):
        """Everything after the backbone.  ptmax=None: the predict_fine sequence
        (networks/patch2pix.py:250-276); ptmax>0 with panc>1: the training-loop forward sequence
        (train_patch2pix.py:97-118), i.e. the 'ptmax=400 panc=8' benchmark configuration (which always
        filters with mutual=True, train_patch2pix.py:100-101)."""
        ticket = self.submit_coarse(feats1, feats2, ksize, True if ptmax else mutual, 0.0 if ptmax else ncn_thres)
        return self.finish_match(ticket, ncn_thres, ptmax, return_all)

    def predict_fine(self, im1, im2, ksize=2, ncn_thres=0.0, mutual=True, return_all=False):
        """networks/patch2pix.py:250-276."""
        feats1, feats2 = self.extract_pair(im1, im2)
        return self.match_from_feats(feats1, feats2, ksize, ncn_thres, mutual, None, return_all)

    # -- backbone (feeds the path) ---------------------------------------------------------------
    def extract_pair(self, im1, im2, slot=None):
        """ResNet34 pyramids of both images (networks/patch2pix.py:222-226).  Equal-sized images go
        through the extractor as one batch of 2; with `enable_backbone_graphs` the batch runs as a
        captured CUDA graph (one of two alternating instances, so two pairs can be in flight)."""
        if im1.shape != im2.shape:
            return (self.extract.forward_all(im1, [], early_feat=True), self.extract.forward_all(im2, [], early_feat=True))
        g = getattr(self, '_bb_graphs', None)
        if g is not None and tuple(im1.shape) == g['shape'] and im1.shape[0] == 1:
            if slot is None:                      # rotate through the instances
                slot = g['next']
                g['next'] = (slot + 1) % len(g['inst'])
            inst = g['inst'][slot % len(g['inst'])]
            if inst['pending'] > 0:
                raise RuntimeError('extract_pair: this backbone-graph instance still backs a pending submit_coarse ticket '
                                   '(its static output buffers would be overwritten); call finish_match first or capture '
                                   'more instances with enable_backbone_graphs(..., instances=n)')
            main = torch.cuda.current_stream(self.device)
            if im1.is_cuda:
                inst['inp'][0:1].copy_(im1, non_blocking=True)
                inst['inp'][1:2].copy_(im2, non_blocking=True)
            else:
                # host images: H2D on a side stream so that the copy overlaps the kernels still queued on the
                # main stream; the instance's input buffer is free once its previous replay has finished
                cs = g['copy_stream']
                cs.wait_event(inst['consumed'])
                if g.get('overlap'):
                    # the whole backbone runs on the side stream and fills the SMs the main stream's small kernels and
                    # kernel tails leave idle; its outputs are protected by the ticket protocol (inst['free'])
                    if inst.get('free') is not None:
                        cs.wait_event(inst['free'])
                    with torch.cuda.stream(cs):
                        inst['inp'][0:1].copy_(im1, non_blocking=True)
                        inst['inp'][1:2].copy_(im2, non_blocking=True)
                        inst['graph'].replay()
                        done = cs.record_event()
                    main.wait_event(done)
                    inst['consumed'] = done
                    feats = inst['out']
                    f1, f2 = _FeatList(f[:1] for f in feats), _FeatList(f[1:] for f in feats)
                    f1.graph_inst = f2.graph_inst = inst
                    return f1, f2
                with torch.cuda.stream(cs):
                    inst['inp'][0:1].copy_(im1, non_blocking=True)
                    inst['inp'][1:2].copy_(im2, non_blocking=True)
                    ready = cs.record_event()
                main.wait_event(ready)
            inst['graph'].replay()
            inst['consumed'] = main.record_event()
            feats = inst['out']
            f1, f2 = _FeatList(f[:1] for f in feats), _FeatList(f[1:] for f in feats)
            f1.graph_inst = f2.graph_inst = inst
            return f1, f2
        feats = self.extract.forward_all(torch.cat([im1, im2], 0), [], early_feat=True)
        b = im1.shape[0]
        return [f[:b] for f in feats], [f[b:] for f in feats]

    def _extract16(self):
        """fp16 / channels_last copy of the backbone (same weights): cuDNN's tensor-core NHWC kernels, and pyramids born
        in the layouts the path wants (levels 1..4 channels-last fp16; the K-major re-layout and the NCHW->NHWC prep
        transposes disappear).  fp16 carries the same 10-bit mantissa as the TF32 convolutions PyTorch runs by default."""
        net = getattr(self, '_extract_half', None)
        if net is None:
            import copy
            net = copy.deepcopy(self.extract).half().to(memory_format=torch.channels_last).eval()
            object.__setattr__(self, '_extract_half', net)      # not a registered sub-module: state_dict stays the reference's
        return net

    def _forward_all_fast(self, x32):
        """x32 [b,3,H,W] fp32 -> [x32, fp16 channels-last levels 1..4]."""
        feats = self._extract16().forward_all(x32.to(dtype=torch.float16, memory_format=torch.channels_last), [], early_feat=True)
        return [x32] + feats[1:]

    def enable_backbone_graphs(self, height, width, instances=2, fast=False, overlap=False):
        """Capture the (launch-bound) backbone for a fixed image size into CUDA graphs.  fast=True: the fp16 /
        channels_last backbone (levels 1..4 come out channels-last fp16, consumed directly by the C ABI's *_nhwc16 entries).
        overlap=True: for host images, extract_pair replays the graph on a side stream (after the H2D copy), so the
        backbone of the next pair overlaps the hot path of the pairs in flight; the pyramids of an instance must then be
        consumed through submit_coarse / finish_match tickets (which record when the instance may be overwritten)."""
        shape = (1, 3, height, width)
        insts = []
        fwd = self._forward_all_fast if fast else (lambda x: self.extract.forward_all(x, [], early_feat=True))
        with torch.no_grad(), torch.cuda.device(self.device):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(instances):
                    inp = torch.zeros(2, 3, height, width, device=self.device)
                    for _ in range(3):
                        fwd(inp)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=side):
                        out = fwd(inp)
                    insts.append({'inp': inp, 'graph': graph, 'out': out, 'pending': 0})
            torch.cuda.current_stream().wait_stream(side)
            for inst in insts:
                inst['consumed'] = torch.cuda.current_stream().record_event()
            copy_stream = torch.cuda.Stream()
        self._bb_graphs = {'shape': shape, 'inst': insts, 'copy_stream': copy_stream, 'next': 0, 'overlap': bool(overlap)}

    def predict_train_sequence(self, im1, im2, ksize=2, ptmax=400, return_all=False):
        """train_patch2pix.py:97-118 under eval()/no_grad: forward -> cal_coarse_matches ->
        filter_coarse(ptmax) -> shift_to_anchors -> mid -> fine (the benchmark configuration)."""
        feats1, feats2 = self.extract_pair(im1, im2)
        return self.match_from_feats(feats1, feats2, ksize, 0.0, True, ptmax, return_all)

    def refine_matches(self, im1, im2, coarse_matches, io_thres):
        """networks/patch2pix.py:278-318.  coarse_matches [N,4] numpy or torch (any device), int64 or float; float64
        rows are refined as float32, which is what the reference's parse_regressor_out computes in (`.float()`).
        The refined rows, their scores and (for a device tensor) the coarse rows come back in one device->host copy."""
        if len(coarse_matches) == 0:
            return np.empty((0, 4)), np.empty((0,)), np.empty((0, 4))
        host_cm = None
        if isinstance(coarse_matches, np.ndarray):
            host_cm = coarse_matches
            cm_ = torch.from_numpy(coarse_matches).to(self.device)
        elif isinstance(coarse_matches, torch.Tensor):
            if not coarse_matches.is_cuda:
                host_cm = coarse_matches.data.numpy()
            cm_ = coarse_matches.to(self.device)
        else:
            raise RuntimeError('coarse_matches must be a numpy array or a torch tensor')
        cm_k = cm_
        if cm_k.dtype not in (torch.int64, torch.float32):
            cm_k = cm_k.float() if cm_k.is_floating_point() else cm_k.long()
        feats1 = self.extract.forward_all(im1, [], early_feat=True)
        feats2 = self.extract.forward_all(im2, [], early_feat=True)
        mid, _ = self.forward_fine_match(feats1, feats2, [cm_k], self.psize[0], self.ptype[0], self.regress_mid)
        fine, fine_p = self.forward_fine_match(feats1, feats2, mid, self.psize[1], self.ptype[1], self.regress_fine)
        # float64 holds fp32 and the coarse rows (int64 below 2^53, fp32, fp64) exactly
        cols = [fine[0].reshape(-1, 4).double(), fine_p[0].reshape(-1, 1).double()]
        if host_cm is None:
            cols.append(cm_.reshape(-1, 4).double())
        both = torch.cat(cols, 1).cpu().numpy()          # one device->host copy
        refined, scores = both[:, :4].astype(np.float32), both[:, 4].astype(np.float32)
        if host_cm is None:
            host_cm = both[:, 5:].astype(torch.empty(0, dtype=cm_.dtype).numpy().dtype)
        coarse_matches = host_cm
        if io_thres > 0:
            pos = np.where(scores > io_thres)[0]
            if len(pos) > 0:
                coarse_matches, refined, scores = coarse_matches[pos], refined[pos], scores[pos]
        return refined, scores, coarse_matches
