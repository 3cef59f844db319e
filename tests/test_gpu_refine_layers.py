"""Each layer of the refine regressor against float64, on every arithmetic path.

`p2p_refine_taps` hands out the intermediate buffers of the last `p2p_refine` call.  Every layer's float64 reference
takes as its input the GPU's own input to that layer (the features and match rows for conv1, the dequantised conv1
output for conv2, the pooled / h1 / h2 taps for the FC layers, the raw tap for the parse), so each comparison measures
one layer's arithmetic.

Two checks per layer:

1. A hard element bound, derived from the arithmetic (not fitted):

       |gpu - ref| <= (e_op + e_acc + e_epi) * sum_k |a_k w_k|  +  e_out * |gpu|  +  floors

   - e_op, operand rounding: 1-pass conv1 reads fp16 operands, the activation rounded twice on the window-map path
     (fp16 feature map, then the normalised window map) and the weight once: 3 * 2^-11, plus 2^-20 for the fp32
     normalisation.  1-pass conv2 reads the conv1 tap itself (exact) and fp16 weights: 2^-11.  3-pass operands are
     hi + lo splits (2^-22 each), the dropped lo * lo term (2^-22) and the fp32 normalisation: 2^-20 in all.
   - e_acc, accumulation: the tensor core is taken to truncate (not round) once per wgmma k16 instruction, with an
     error of at most 2^-22 of the magnitudes it adds, so a chain of N instructions contributes N * 2^-22 (N = K / 16
     times the passes; the segmented 3-pass launches drain shorter chains, so the whole-K chain bounds every seg_len).
     The CUDA-core paths (gemm_impl 1, fc_impl 0, the Linear(256, 5) tail) round each fma: K * 2^-24 per pass.
   - e_epi: the epilogue's fmaf and scale: 2^-22, of sum |a w| and of |bias|.  The fp32 BatchNorm fold rounds the
     bias: 2^-21 of |beta| + |mean * gain| (+ |linear bias * gain| for the FC layers), a term of the bound and of the
     gate's scale.
   - e_out: the fp16 output of conv1 (2^-11 on 1-pass, which writes hi only; 2^-22 for hi + lo) and of the FC layers
     (2^-22).  Floors: half the smallest fp16 subnormal, 2^-25, divided by the buffer's power-of-two scale, for the
     output and for each operand (weights are scaled so that each row's largest lies in [512, 1024), activations by
     their reported scales).
   - conv2's max-pool: a max of values moves by no more than the largest error of the values it takes, so the pooled
     bound is the largest bound over its 8 x 8 window.

   `test_bound_holds_on_emulated_arithmetic` emulates this arithmetic in numpy at conv1's K (truncating fp32
   accumulation per k16 group included) and shows the bound is never exceeded.

2. A statistical gate: the RMS of the error over the RMS of the operand-rounding scale u * sqrt(sum_k (a_k w_k)^2)
   (with the output rounding and floors added in quadrature), per output channel and per row.  A defect confined to
   one channel among 512, or one row, moves its ratio far past the limit.  Limits: GATE below.
"""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p_oracle as O

U11, U22, U24 = 2.0 ** -11, 2.0 ** -22, 2.0 ** -24
FLOOR = 2.0 ** -25                    # half the smallest fp16 subnormal
K1, K2 = 73 * 64, 72 * 64             # conv1 / conv2 GEMM K (rgb chunk included)

# Statistical gate limits (largest per-channel ratio, largest per-row ratio) per layer and conv pass count: twice the
# largest ratio measured over every path, input and weight set of this file on one H100 80GB HBM3 (power limit 700 W);
# the measured values are in the comments.  The FC layers run 3-pass on every tensor-core path.
GATE = {
    ('conv1', 1): (3.0, 1.3),     # measured 1.49, 0.64
    ('conv1', 3): (8.0, 3.8),     # measured 3.94, 1.89
    ('conv2', 1): (2.7, 1.3),     # measured 1.34, 0.62
    ('conv2', 3): (23., 9.6),     # measured 11.2, 4.76
    'fc1': (10., 2.1),            # measured 4.95, 1.04
    'fc2': (5.3, 1.4),            # measured 2.64, 0.70
    'fc3': (5.6, 6.3),            # measured 2.76, 3.12
}
REPORT = os.environ.get('P2P_LAYER_REPORT')    # optional path: the measured ratios are appended there as JSON lines


def op_units(layer, passes, simt=False):
    """(e_op + e_acc + e_epi, e_out, u) of one layer on one arithmetic path; u is the gate's operand unit."""
    if layer == 'conv1':
        op = 3 * U11 + 2.0 ** -20 if passes == 1 else 2.0 ** -20
        k = K1
    elif layer == 'conv2':
        op = U11 if passes == 1 else 2.0 ** -20
        k = K2
    else:                              # fc1 / fc2: 3-pass on the tensor cores or fp32 on the CUDA cores
        op = 4 * U22
        k = 512
    acc = passes * k * U24 if simt else passes * (k // 16) * U22
    out = {'conv1': U11 if passes == 1 else U22, 'conv2': 0.0}.get(layer, U22)
    u = U11 if passes == 1 else U22
    return op + acc + U22, out, u


def hard_bound(S, gpu, alpha, e_out, floor):
    return alpha * S + e_out * (1 + 2 * U11) * gpu.abs() + floor


# ------------------------------------------------------------------------------------------------------------------
# the bound on emulated arithmetic (no GPU)
# ------------------------------------------------------------------------------------------------------------------
def _trunc_f32(x):
    """Round float64 values toward zero to float32."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def test_bound_holds_on_emulated_arithmetic():
    """1-pass and 3-pass dot products of conv1's K = 4672 in emulated tensor-core arithmetic: fp16 operands (the
    activation rounded twice, as on the window-map path), each k16 group's exact sum added to an fp32 accumulator that
    truncates, fp16 output.  Inputs span 2^-12 .. 2^4 in magnitude with either sign, so cancellation, subnormal operands
    and subnormal outputs all occur.  The error against float64 never exceeds the bound, and reaches a visible part of
    it (the bound is not vacuous)."""
    rng = np.random.default_rng(0)
    n = 2048
    a = rng.standard_normal((n, K1)) * np.exp2(rng.uniform(-12, 4, (n, 1)))
    a[:, ::7] *= 2.0 ** -14                                                   # subnormal operands
    w = rng.standard_normal((n, K1)) * np.exp2(rng.uniform(-6, 0, (n, 1)))
    sw = np.exp2(9 - np.floor(np.log2(np.abs(w).max(1, keepdims=True))))      # row max in [512, 1024)
    exact = (a * w).sum(1)
    S = np.abs(a * w).sum(1)
    worst = {}
    for passes in (1, 3):
        c = 1.3717                                    # a per-level norm: fp16(f / c), then fp16 of that times c
        a16 = (a / c).astype(np.float16).astype(np.float64)
        a16 = (a16.astype(np.float32) * np.float32(c)).astype(np.float16).astype(np.float64)
        w_hi = (w * sw).astype(np.float16).astype(np.float64)
        if passes == 1:
            prods = [a16 * w_hi]
        else:
            a_hi = a.astype(np.float16).astype(np.float64)
            a_lo = (a - a_hi).astype(np.float16).astype(np.float64)
            w_lo = (w * sw - w_hi).astype(np.float16).astype(np.float64)
            prods = [a_lo * w_hi, a_hi * w_lo, a_hi * w_hi]
        acc = np.zeros(n, dtype=np.float32)
        for g in range(K1 // 16):
            for p in prods:
                acc = _trunc_f32(acc.astype(np.float64) + p[:, 16 * g:16 * g + 16].sum(1))
        y = acc.astype(np.float64) / sw[:, 0]
        y_out = y.astype(np.float16).astype(np.float64) if passes == 1 else y
        alpha, e_out, _ = op_units('conv1', passes)
        # floors: both activation roundings and the weight's (relative to its row scale), and the output's
        floor = FLOOR * (2 * c * np.abs(w).sum(1) + np.abs(a).sum(1) / sw[:, 0] + 1)
        bound = alpha * S + e_out * (1 + 2 * U11) * np.abs(y_out) + floor
        err = np.abs(y_out - exact)
        assert (err <= bound).all(), (passes, float((err / bound).max()))
        worst[passes] = float((err / bound).max())
    assert worst[1] > 0.01, worst      # independent roundings add like sqrt(K); the bound adds them like K


# ------------------------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------------------------
def _fold(sd, pre, bn):
    g = sd[pre + bn + '.weight'].double() / torch.sqrt(sd[pre + bn + '.running_var'].double() + O.BN_EPS)
    return g, sd[pre + bn + '.bias'].double() - sd[pre + bn + '.running_mean'].double() * g


class Ref:
    """The regressor's layers in float64 on the GPU, BatchNorm folded."""

    def __init__(self, sd, pre):
        d = lambda k: sd[pre + k].double().cuda()
        g1, self.b1 = (t.cuda() for t in _fold(sd, pre, 'conv.1'))
        g2, self.b2 = (t.cuda() for t in _fold(sd, pre, 'conv.3'))
        gf1, bf1 = (t.cuda() for t in _fold(sd, pre, 'fc.1'))
        gf2, bf2 = (t.cuda() for t in _fold(sd, pre, 'fc.4'))
        self.w1 = d('conv.0.weight') * g1[:, None, None, None]
        self.w2 = d('conv.2.weight') * g2[:, None, None, None]
        self.f1 = d('fc.0.weight') * gf1[:, None]
        self.c1 = d('fc.0.bias') * gf1 + bf1
        self.f2 = d('fc.3.weight') * gf2[:, None]
        self.c2 = d('fc.3.bias') * gf2 + bf2
        self.f3, self.c3 = d('fc.6.weight'), d('fc.6.bias')
        # magnitudes of the terms of each folded bias: its fp32 fold is good to 2^-21 of them
        mag = lambda bn, lin=None: ((d(bn + '.bias').abs() + (d(bn + '.running_mean') * d(bn + '.weight')).abs()
                                     / torch.sqrt(d(bn + '.running_var') + O.BN_EPS) +
                                     (0 if lin is None else (d(lin) * d(bn + '.weight')).abs()
                                      / torch.sqrt(d(bn + '.running_var') + O.BN_EPS))) * 2.0 ** -21)
        self.eb = {'conv1': mag('conv.1'), 'conv2': mag('conv.3'), 'fc1': mag('fc.1', 'fc.0.bias'),
                   'fc2': mag('fc.4', 'fc.3.bias')}
        # each weight row's largest magnitude: its fp16 image is scaled to [512, 1024), so a subnormal weight is off by
        # at most 2^-25 / scale <= rowmax * 2^-34
        self.wsub = {k: v.abs().flatten(1).max(1).values * 2.0 ** -34 for k, v in
                     (('conv1', self.w1), ('conv2', self.w2), ('fc1', self.f1), ('fc2', self.f2))}

    def conv1_input(self, feats1, feats2, rows):
        f1 = [f.double().cpu() for f in feats1]
        f2 = [f.double().cpu() for f in feats2]
        n = rows.shape[0]
        a, b = O.select_local_patch_feats(f1, f2, 0, rows.cpu(), 16)
        a = O.l2_normalize(a.cuda(), 0).view(-1, n, 16, 16).permute(1, 0, 2, 3)
        b = O.l2_normalize(b.cuda(), 0).view(-1, n, 16, 16).permute(1, 0, 2, 3)
        return torch.cat([a, b], 1)

    @staticmethod
    def _conv(x, w, stride):
        return (F.conv2d(x, w, None, stride, 1), F.conv2d(x.abs(), w.abs(), None, stride, 1),
                F.conv2d(x * x, w * w, None, stride, 1).sqrt(), F.conv2d(x.abs(), torch.ones_like(w[:1]), None, stride, 1))

    def conv1(self, x):
        """-> y [m][512][8][8], sum |a w|, sqrt(sum (a w)^2), sum |a|."""
        y, S, Q, A = self._conv(x, self.w1, 2)
        return y + self.b1[:, None, None], S, Q, A

    def conv2(self, y):
        z, S, Q, A = self._conv(y, self.w2, 1)
        return z + self.b2[:, None, None], S, Q, A


def _dq(hi, lo, scale):
    v = hi.double()
    if lo is not None:
        v = v + lo.double()
    return v / scale


def taps(net):
    """The last p2p_refine call's buffers (p2p_refine_taps) as float64 tensors, and its info."""
    import ctypes as C
    from patch2pix_b200 import _lib
    h = net._handle
    info = (C.c_int32 * 4)()
    sc = (C.c_float * 4)()
    _lib.check(h.lib.p2p_refine_taps(h.h, info, sc, *([None] * 10), h.stream()))
    m, passes, band, fc_tc = list(info)
    y_scale, s0, s1, s2 = list(sc)
    dev = net.device
    e16 = lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)
    rows = torch.empty(m, dtype=torch.int32, device=dev)
    y_hi, y_lo = e16(m, 64, 512), (e16(m, 64, 512) if passes == 3 else None)
    pooled = torch.empty(m, 512, dtype=torch.float32, device=dev)
    h1 = (e16(m, 512), e16(m, 512)) if fc_tc else (None, None)
    h2 = (e16(m, 256), e16(m, 256)) if fc_tc else (None, None)
    n_all = net._last_n
    raw = torch.empty(n_all, 5, dtype=torch.float32, device=dev)
    P = _lib.ptr
    _lib.check(h.lib.p2p_refine_taps(h.h, info, sc, P(rows), P(y_hi), P(y_lo), P(pooled), P(h1[0]), P(h1[1]), P(h2[0]),
                                     P(h2[1]), P(raw), h.stream()))
    torch.cuda.synchronize()
    t = dict(m=m, passes=passes, band=band, fc_tc=fc_tc, scales=(y_scale, s0, s1, s2), rows=rows.long(),
             y_hi=y_hi, y_lo=y_lo, pooled=pooled.double(), raw=raw.double())
    t['y'] = _dq(y_hi, y_lo, y_scale).view(m, 8, 8, 512).permute(0, 3, 1, 2)
    if fc_tc:
        t['h1'] = _dq(h1[0], h1[1], s1)
        t['h2'] = _dq(h2[0], h2[1], s2)
        t['h_raw'] = (h1, h2)
    return t


def _gate(name, err, scale, stats):
    """RMS ratios per output channel (dim 1) and per row (dim 0) of err / scale [m][C][...]."""
    e2 = err.pow(2).flatten(2).sum(2)
    s2 = scale.pow(2).flatten(2).sum(2)
    ch = (e2.sum(0) / s2.sum(0).clamp_min(1e-300)).sqrt()
    rw = (e2.sum(1) / s2.sum(1).clamp_min(1e-300)).sqrt()
    stats[name] = (float(ch.max()), float(rw.max()))
    return ch, rw


def _check(name, gpu, ref, bound, gate_scale, stats, limit):
    err = (gpu - ref).abs()
    bad = err > bound
    assert not bad.any(), (name, int(bad.sum()), float((err / bound).max()), float(err.max()))
    ch, rw = _gate(name, err.view(err.shape[0], err.shape[1], -1), gate_scale.view(err.shape[0], err.shape[1], -1),
                   stats)
    assert float(ch.max()) <= limit[0], (name, 'channel', int(ch.argmax()), float(ch.max()))
    assert float(rw.max()) <= limit[1], (name, 'row', int(rw.argmax()), float(rw.max()))


def check_layers(net, ref, feats1, feats2, matches, W, H, simt=False):
    """All float64 layer comparisons of the last refine call on `matches`; returns the gate ratios and the taps."""
    t = taps(net)
    stats = {'m': t['m'], 'passes': t['passes'], 'band': t['band']}
    m, passes = t['m'], t['passes']
    y_scale, s0, s1, s2 = t['scales']
    rows = t['rows'].cpu()
    W1_, H1_, W2_, H2_ = W[0], H[0], W[1], H[1]
    if m > 0:
        # conv1 + BN
        x = ref.conv1_input(feats1, feats2, matches[rows])
        y64, S, Q, A = ref.conv1(x)
        alpha, e_out, u = op_units('conv1', passes, simt)
        fl = FLOOR / y_scale + ref.wsub['conv1'][:, None, None] * A + 2.0 ** -37 * ref.w1.abs().sum((1, 2, 3))[:, None, None]
        eb = ref.eb['conv1'][:, None, None]
        bnd = hard_bound(S, t['y'], alpha, e_out, fl) + U22 * ref.b1.abs()[:, None, None] + eb
        gs = ((u * Q) ** 2 + (e_out * y64) ** 2 + (FLOOR / y_scale) ** 2 + eb ** 2).sqrt()
        _check('conv1', t['y'], y64, bnd, gs, stats, GATE['conv1', passes])
        # conv2 + BN + ReLU + 8x8 max-pool, from the dequantised conv1 tap
        z64, S, Q, A = ref.conv2(t['y'])
        alpha, _, u = op_units('conv2', passes, simt)
        eb = ref.eb['conv2'][:, None, None]
        b = alpha * S + U22 * ref.b2.abs()[:, None, None] + eb + ref.wsub['conv2'][:, None, None] * A
        p64 = z64.clamp_min(0).flatten(2).max(2).values
        pb = b.flatten(2).max(2).values
        idx = z64.flatten(2).argmax(2, keepdim=True)
        gs = ((u * Q.flatten(2).gather(2, idx)[..., 0]) ** 2 + ref.eb['conv2'] ** 2).sqrt()
        _check('conv2', t['pooled'], p64, pb, gs[..., None].clamp_min(1e-30), stats,
               GATE['conv2', passes])
        if t['fc_tc']:
            for name, a_in, wt, c, s_in, s_out, out in (('fc1', t['pooled'], ref.f1, ref.c1, s0, s1, t['h1']),
                                                        ('fc2', t['h1'], ref.f2, ref.c2, s1, s2, t['h2'])):
                r = (a_in @ wt.T + c).clamp_min(0)
                S = a_in.abs() @ wt.abs().T
                Q = ((a_in * a_in) @ (wt * wt).T).sqrt()
                alpha, e_out, u = op_units(name, 3)
                fl = (FLOOR / s_in) * wt.abs().sum(1) + ref.wsub[name] * a_in.abs().sum(1, keepdim=True) + FLOOR / s_out
                eb = ref.eb[name]
                bnd = alpha * S + U22 * c.abs() + eb + e_out * (1 + U11) * out.abs() + fl
                gs = ((u * Q) ** 2 + (FLOOR / s_out) ** 2 + ((FLOOR / s_in) * wt.abs().sum(1)) ** 2 + eb ** 2).sqrt()
                _check(name, out[..., None], r[..., None], bnd[..., None], gs[..., None], stats,
                       GATE[name])
            # Linear(256, 5) on the CUDA cores, from h2
            h2 = t['h2']
            r = h2 @ ref.f3.T + ref.c3
            S = h2.abs() @ ref.f3.abs().T + ref.c3.abs()
            Q = ((h2 * h2) @ (ref.f3 * ref.f3).T).sqrt()
            bnd = 16 * U24 * S + 2.0 ** -30
            raw_rows = t['raw'][t['rows']]
            _check('fc3', raw_rows[..., None], r[..., None], bnd[..., None], (U24 * Q + 2.0 ** -30)[..., None], stats,
                   GATE['fc3'])
        else:
            # CUDA-core FC (fp32 fma chains), raw only: the three layers' chains, propagated through the magnitudes
            p = t['pooled']
            h1 = (p @ ref.f1.T + ref.c1).clamp_min(0)
            h2 = (h1 @ ref.f2.T + ref.c2).clamp_min(0)
            r = h2 @ ref.f3.T + ref.c3
            m1 = p @ ref.f1.abs().T + ref.c1.abs()
            m2 = m1 @ ref.f2.abs().T + ref.c2.abs()
            m3 = m2 @ ref.f3.abs().T + ref.c3.abs()
            bnd = 3 * 520 * U24 * m3 + 2.0 ** -30
            err = (t['raw'][t['rows']] - r).abs()
            assert (err <= bnd).all(), ('fc_cuda_core', float((err / bnd).max()))
            stats['fc_cuda_core'] = float((err / bnd).max())
    # parse_regressor_out from the raw tap, every row
    raw = t['raw']
    mt = net._last_out
    mi = matches.double().cuda() if not matches.is_floating_point() else matches.float().double().cuda()
    lim = torch.tensor([W1_, H1_, W2_, H2_], dtype=torch.float64, device=raw.device)
    un = mi + 16 * torch.tanh(raw[:, :4].clamp_min(0)) - 8
    c64 = torch.minimum(un.clamp_min(0), lim)
    err = (mt[0].double() - c64).abs()
    bnd = 16 * 4 * U24 + 2 * U24 * (mi.abs() + 8) + 1e-12
    assert (err <= bnd).all(), ('parse coords', float((err / bnd).max()))
    p64 = torch.sigmoid(raw[:, 4])
    assert ((mt[1].double() - p64).abs() <= 8 * U24).all(), ('parse probs', float((mt[1].double() - p64).abs().max()))
    if REPORT:
        with open(REPORT, 'a') as f:
            f.write(json.dumps(stats) + '\n')
    return stats, t


# ------------------------------------------------------------------------------------------------------------------
# fixtures and inputs
# ------------------------------------------------------------------------------------------------------------------
def _make_net(sd):
    from patch2pix_b200.model import Patch2PixB200
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    cfg = Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=sd, change_stride=True, regressor_config=rc)
    net = Patch2PixB200(cfg)
    _instrument(net)
    return net


def _instrument(net):
    """Remember the last call's n and outputs (the taps' raw is [n][5]; the parse check reads the outputs)."""
    inner = net.forward_fine_match

    def wrapped(f1, f2, cm, psize=16, ptype='center', regressor=None, _prepared=None):
        out = inner(f1, f2, cm, psize, ptype, regressor, _prepared)
        net._last_n = cm[0].shape[0]
        net._last_out = (out[0][0].reshape(-1, 4), out[1][0].reshape(-1))
        return out
    net.forward_fine_match = wrapped


DEFAULTS = dict(mid_passes=3, fine_passes=1, mid_band=26, fuse_gather=3, share_windows=1, epi_async=1, fc_impl=1,
                gemm_impl=0)


def run(net, f1, f2, m, which='mid', **opts):
    for k, v in opts.items():
        net.set_option(k, v)
    try:
        with torch.no_grad():
            reg = net.regress_mid if which == 'mid' else net.regress_fine
            net.forward_fine_match(f1, f2, [m.cuda()], 16, 'center', reg)
        torch.cuda.synchronize()
        shared = net._handle.get_option('shared_rows')
    finally:
        for k in opts:
            net.set_option(k, DEFAULTS[k])
    return shared


@pytest.fixture(scope='module')
def sd0(consensus_sd):
    return {k: v.clone() for k, v in consensus_sd.items()}


@pytest.fixture(scope='module')
def net0(sd0):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _make_net(sd0)


def _feats(net, size1, size2, seed=9):
    from patch2pix_b200.synth import synthetic_pair_sized
    im1, im2 = synthetic_pair_sized(seed, size1, size2)
    with torch.no_grad():
        return (net.extract.forward_all(im1.cuda(), [], early_feat=True),
                net.extract.forward_all(im2.cuda(), [], early_feat=True))


def anchor_rows(n_groups, W, H, seed, frac):
    """shift_to_anchors groups (rows 8g..8g+3 move point 1 by (+-8, +-8), rows 8g+4..8g+7 point 2), so that window
    sharing engages, then rows whose windows clip every border and rows outside both images."""
    g = torch.Generator().manual_seed(seed)
    base = (torch.rand(n_groups, 4, generator=g) * torch.tensor([W[0], H[0], W[1], H[1]], dtype=torch.float32)).floor()
    m = O.shift_to_anchors([base.long()], 8)[0].float()
    if frac:
        m = m + torch.rand(m.shape, generator=g) * 0.9
    edge = torch.tensor([[0.0, 0.0, W[1] - 1, H[1] - 1], [W[0] - 1, H[0] - 1, 0.0, 0.0], [0.0, H[0] - 1, W[1] - 1, 0.0],
                         [-25.0, -30.5, W[1] + 25, H[1] + 40], [W[0] + 33, H[0] + 17.5, -40.0, -9.0]])
    m = torch.cat([m, edge])
    return m if frac else m.long()


EQ = ((128, 160), (128, 160))
UNEQ = ((96, 224), (128, 160))
ODD = ((97, 133), (120, 161))


def _wh(sizes):
    return [sizes[0][1], sizes[1][1]], [sizes[0][0], sizes[1][0]]


@pytest.fixture(scope='module')
def eq_case(net0):
    f1, f2 = _feats(net0, *EQ)
    W, H = _wh(EQ)
    return f1, f2, W, H


PATHS = {
    # name: (which, options, CUDA-core conv)
    'mid_shipped': ('mid', {}, False),
    'mid_1pass_share': ('mid', dict(mid_passes=1), False),
    'mid_1pass_noshare': ('mid', dict(mid_passes=1, share_windows=0), False),
    'fine_shipped': ('fine', {}, False),
    'fine_fuse_gather0': ('fine', dict(fuse_gather=0), False),
    'mid_3pass_all': ('mid', dict(mid_band=0), False),
    'fine_3pass': ('fine', dict(fine_passes=3), False),
    'mid_fc_cuda_core': ('mid', dict(mid_passes=1, fc_impl=0), False),
    'fine_gemm_impl1': ('fine', dict(gemm_impl=1), True),
}


@pytest.mark.gpu
@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('frac', [False, True])
def test_layers_against_float64(net0, sd0, eq_case, path, frac):
    """16 anchor groups (128 rows) + 5 border / outside rows = 133 rows, int64 and float, on each arithmetic path."""
    f1, f2, W, H = eq_case
    which, opts, simt = PATHS[path]
    m = anchor_rows(16, W, H, 5, frac)
    shared = run(net0, f1, f2, m, which, **opts)
    if path == 'mid_1pass_share':
        assert shared > 0
    ref = Ref(sd0, 'regress_mid.' if which == 'mid' else 'regress_fine.')
    stats, t = check_layers(net0, ref, f1, f2, m, W, H, simt)
    if path == 'mid_shipped':
        assert t['band'] == 1 and t['m'] > 0, stats
    print(path, frac, stats)


@pytest.mark.gpu
@pytest.mark.parametrize('sizes', [UNEQ, ODD], ids=['96x224_128x160', '97x133_120x161'])
@pytest.mark.parametrize('path', ['mid_shipped', 'mid_1pass_share', 'fine_shipped'])
def test_layers_unequal_and_odd_sizes(net0, sd0, sizes, path):
    f1, f2 = _feats(net0, *sizes, seed=4)
    W, H = _wh(sizes)
    which, opts, simt = PATHS[path]
    m = anchor_rows(9, W, H, 7, True)          # 72 anchor rows + 5 edge rows
    run(net0, f1, f2, m, which, **opts)
    check_layers(net0, Ref(sd0, 'regress_mid.' if which == 'mid' else 'regress_fine.'), f1, f2, m, W, H, simt)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 3, 131, 8 * 17 + 3])
def test_layers_row_counts(net0, sd0, eq_case, n):
    """n = 1, 3, 131 and 17 anchor groups plus a partial one (139 rows; the sharing classifier's last group is
    incomplete)."""
    f1, f2, W, H = eq_case
    m = anchor_rows(18, W, H, 11 + n, True)[:n]
    ref = Ref(sd0, 'regress_mid.')
    for opts in (dict(mid_passes=1), {}):
        run(net0, f1, f2, m, 'mid', **opts)
        check_layers(net0, ref, f1, f2, m, W, H)


def _tap_arrays(net):
    t = taps(net)
    out = [t['y_hi'], t['pooled'], t['raw']]
    if t['y_lo'] is not None:
        out.append(t['y_lo'])
    if t['fc_tc']:
        out += [x for pair in t['h_raw'] for x in pair]
    return out


@pytest.mark.gpu
def test_bit_identical_paths_have_equal_taps(net0, eq_case):
    """fuse_gather 1 and 2 (gathering producers) against 3 (window map), and epi_async 0 against 1, are documented
    as bit-identical: every tap must be equal, not just the outputs."""
    f1, f2, W, H = eq_case
    m = anchor_rows(16, W, H, 5, True)
    run(net0, f1, f2, m, 'fine')
    base = _tap_arrays(net0)
    for opts in (dict(fuse_gather=1), dict(fuse_gather=2), dict(epi_async=0)):
        run(net0, f1, f2, m, 'fine', **opts)
        for a, b in zip(base, _tap_arrays(net0)):
            assert torch.equal(a, b), opts
    run(net0, f1, f2, m, 'mid', mid_passes=1)
    base = _tap_arrays(net0)
    run(net0, f1, f2, m, 'mid', mid_passes=1, epi_async=0)
    for a, b in zip(base, _tap_arrays(net0)):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------
# weights beyond the seeded ones
# ------------------------------------------------------------------------------------------------------------------
REGRESSORS = ('regress_mid.', 'regress_fine.')


def weights_w1(sd0):
    """Per-channel BN gains spread over 2^-12 .. 2^4 (either sign) in both convs: per-channel weight scales and the
    fp16 subnormal floors of conv1's output."""
    sd = {k: v.clone() for k, v in sd0.items()}
    g = torch.Generator().manual_seed(21)
    for pre in REGRESSORS:
        for bn in ('conv.1', 'conv.3'):
            e = torch.empty(512).uniform_(-12, 4, generator=g)
            s = torch.where(torch.rand(512, generator=g) < 0.2, -1.0, 1.0)
            sd[pre + bn + '.weight'] = sd[pre + bn + '.weight'].abs() * torch.exp2(e) * s
    return sd


W2_POOLED = list(range(3, 512, 61))
W2_H1 = list(range(5, 512, 73))
W2_F = 2.0 ** 13


def weights_w2(sd0):
    """Large activations: pooled channels W2_POOLED and h1 channels W2_H1 scaled by 2^13 through their BatchNorm, and
    the next layer's weights on those channels by 2^-13.  In exact arithmetic the network computes what the seeded one
    computes; its pooled and h1 activations reach about 1e4, past what a fixed FC operand scale of 16 can hold."""
    sd = {k: v.clone() for k, v in sd0.items()}
    for pre in REGRESSORS:
        for bn, nxt, chans in (('conv.3', 'fc.0', W2_POOLED), ('fc.1', 'fc.3', W2_H1)):
            for k in ('.weight', '.bias'):
                sd[pre + bn + k][chans] *= W2_F
            sd[pre + nxt + '.weight'][:, chans] /= W2_F
    return sd


def weights_w3(sd0):
    """Degenerate channels: all-zero conv1 / conv2 / FC weight rows, and conv2 channels whose bias ReLU-zeroes them,
    so that pooled is exactly 0 there."""
    sd = {k: v.clone() for k, v in sd0.items()}
    for pre in REGRESSORS:
        sd[pre + 'conv.0.weight'][7::50] = 0
        sd[pre + 'conv.2.weight'][11::50] = 0
        z = list(range(13, 512, 50))
        sd[pre + 'conv.2.weight'][z] = 0
        sd[pre + 'conv.3.bias'][z] = -1.0
        sd[pre + 'conv.3.running_mean'][z] = 0.0
        sd[pre + 'fc.0.weight'][17::60] = 0
        sd[pre + 'fc.3.weight'][19::40] = 0
    return sd


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['w1', 'w2', 'w3'])
def test_layers_weight_variants(sd0, eq_case, variant):
    sd = {'w1': weights_w1, 'w2': weights_w2, 'w3': weights_w3}[variant](sd0)
    net = _make_net(sd)
    f1, f2, W, H = eq_case
    m = anchor_rows(16, W, H, 5, True)
    for path in ('mid_shipped', 'mid_1pass_share', 'fine_shipped'):
        which, opts, simt = PATHS[path]
        run(net, f1, f2, m, which, **opts)
        stats, t = check_layers(net, Ref(sd, 'regress_mid.' if which == 'mid' else 'regress_fine.'), f1, f2, m, W, H)
        if variant == 'w2':
            assert float(t['pooled'][:, W2_POOLED].max()) > 4096 and float(t['h1'][:, W2_H1].max()) > 4096, stats
        if variant == 'w3':
            assert (t['pooled'][:, 13::50] == 0).all()


@pytest.mark.gpu
def test_large_activations_end_to_end_against_oracle(sd0, eq_case):
    """W2 through the shipped mid and fine stages against the fp32 oracle: the outputs stay as close as the seeded
    weights' do.  With a fixed FC operand scale of 16, activations above 4094 were clipped silently."""
    sd = weights_w2(sd0)
    net = _make_net(sd)
    f1, f2, W, H = eq_case
    m = anchor_rows(16, W, H, 5, False)
    fo1 = [f.cpu() for f in f1]
    fo2 = [f.cpu() for f in f2]
    for which, pre in (('mid', 'regress_mid.'), ('fine', 'regress_fine.')):
        run(net, f1, f2, m, which)
        c, p = net._last_out
        cr, pr = O.forward_fine_match(fo1, fo2, [m], {k: v.cpu() for k, v in sd.items()}, pre)
        dc = (c.cpu() - cr[0]).abs().max().item()
        dp = (p.cpu() - pr[0]).abs().max().item()
        assert dc < 0.05 and dp < 1e-3, (which, dc, dp)


# ------------------------------------------------------------------------------------------------------------------
# sensitivity of the gates
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gate_catches_one_conv1_channel_off_by_2_pow_minus_6(sd0, eq_case):
    """The GPU runs with one conv1 output channel's weights scaled by 1 + 2^-6, the reference with the true weights:
    the conv1 channel gate fails (the hard bound alone, at 3 * 2^-11 of sum |a w|, may not)."""
    sd = {k: v.clone() for k, v in sd0.items()}
    sd['regress_mid.conv.0.weight'][123] *= 1 + 2.0 ** -6
    net = _make_net(sd)
    f1, f2, W, H = eq_case
    m = anchor_rows(16, W, H, 5, True)
    run(net, f1, f2, m, 'mid', mid_passes=1)
    t = taps(net)
    x = Ref(sd0, 'regress_mid.').conv1_input(f1, f2, m[t['rows'].cpu()])
    y64, S, Q, A = Ref(sd0, 'regress_mid.').conv1(x)
    alpha, e_out, u = op_units('conv1', 1)
    gs = ((u * Q) ** 2 + (e_out * y64) ** 2).sqrt()
    ch, rw = _gate('conv1', (t['y'] - y64).abs().flatten(2), gs.flatten(2), {})
    lim = GATE['conv1', 1][0]
    assert int(ch.argmax()) == 123 and float(ch[123]) > lim, float(ch[123])
    others = torch.cat([ch[:123], ch[124:]])
    assert float(others.max()) <= lim


@pytest.mark.gpu
def test_gate_catches_a_row_shifted_by_one_pixel(net0, sd0, eq_case):
    """The reference is given one row shifted by 1 px: that row's conv1 gate fails."""
    f1, f2, W, H = eq_case
    m = anchor_rows(16, W, H, 5, False)
    run(net0, f1, f2, m, 'mid', mid_passes=1)
    t = taps(net0)
    shifted = m.clone()
    shifted[40, 0] += 1
    ref = Ref(sd0, 'regress_mid.')
    y64, S, Q, A = ref.conv1(ref.conv1_input(f1, f2, shifted[t['rows'].cpu()]))
    alpha, e_out, u = op_units('conv1', 1)
    gs = ((u * Q) ** 2 + (e_out * y64) ** 2).sqrt()
    ch, rw = _gate('conv1', (t['y'] - y64).abs().flatten(2), gs.flatten(2), {})
    assert int(rw.argmax()) == 40 and float(rw[40]) > GATE['conv1', 1][1], float(rw[40])


# ------------------------------------------------------------------------------------------------------------------
# the risk band's premise
# ------------------------------------------------------------------------------------------------------------------
def _band(o, tau):
    th = torch.tanh(o.clamp_min(0))
    return torch.minimum(torch.full_like(o, tau), tau * (1 - th * th) + 3e-4)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['eq_int', 'eq_float', 'uneq', 'odd'])
def test_risk_band_covers_the_1pass_error(net0, sd0, case):
    """Every coordinate the band lets through on its 1-pass value (not flagged) is within band(o) (+ the 2e-4 tie
    slack) of the float64 forward's, and a raw output <= -eps_o (the exact -8 offset) is <= 0 in float64 too."""
    sizes = {'eq_int': EQ, 'eq_float': EQ, 'uneq': UNEQ, 'odd': ODD}[case]
    f1, f2 = _feats(net0, *sizes, seed=13)
    W, H = _wh(sizes)
    m = anchor_rows(48, W, H, 29, case != 'eq_int')
    tau = DEFAULTS['mid_band'] * 1e-3
    run(net0, f1, f2, m, 'mid', mid_passes=1)
    t = taps(net0)
    c1 = net0._last_out[0].double()
    o = t['raw']
    ref = Ref(sd0, 'regress_mid.')
    y, _, _, _ = ref.conv1(ref.conv1_input(f1, f2, m))
    z, _, _, _ = ref.conv2(y)
    p = z.clamp_min(0).flatten(2).max(2).values
    h = (p @ ref.f1.T + ref.c1).clamp_min(0)
    h = (h @ ref.f2.T + ref.c2).clamp_min(0)
    r64 = h @ ref.f3.T + ref.c3
    mi = (m.double() if not m.is_floating_point() else m.float().double()).cuda()
    v64 = mi + 16 * torch.tanh(r64[:, :4].clamp_min(0)) - 8
    v1 = mi + 16 * torch.tanh(o[:, :4].clamp_min(0)) - 8      # the un-clamped coordinate flag_risky reads
    lim = torch.tensor([W[0], H[0], W[1], H[1]], dtype=torch.float64, device=o.device)
    band = _band(o[:, :4], tau)
    eps_o = 0.02
    inside = (v1 > -tau) & (v1 < lim + tau)
    skip = (o[:, :4] > -eps_o) & inside & ((v1 - torch.round(v1)).abs() >= band)
    ratio = ((v1 - v64).abs() / band)[skip]
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print('band', case, 'skipped coords', int(skip.sum()), 'largest |v1 - v64| / band', worst)
    assert ((v1 - v64).abs() < band + 2e-4)[skip].all(), worst
    neg = o[:, :4] <= -eps_o
    assert (r64[:, :4][neg] <= 0).all()
    if REPORT:
        with open(REPORT, 'a') as f:
            f.write(json.dumps({'band_case': case, 'skipped': int(skip.sum()), 'ratio': worst}) + '\n')
