"""float64 restatement of SuperGlue (patch2pix_b200/superglue.py, csrc/superglue.cu), for the tests.

The conventions are those patch2pix_b200/superglue.py states, recalled from SuperGlue's published code and not checked
against that code or its released weights: keypoints normalised by (kpts - [W/2, H/2]) / (0.7 max(W, H)); a keypoint
encoder of Conv1d(k=1) + BatchNorm1d (eval) + ReLU layers on cat(kpts^T, scores), added to the descriptors; 4-head
attention whose channel c belongs to head c % 4, logits scaled by 1/sqrt(dim / 4); merge, then an MLP on cat(x, message),
added as a residual; cross layers take their source from the other image; final_proj, then scores / sqrt(dim);
log_optimal_transport with a dustbin row and column of bin_score, and the mutual-argmax extraction.  Weights are a
state_dict converted to numpy (to_numpy).  Everything is one pair at a time, in numpy float64.
"""
import math

import numpy as np

BN_EPS = 1e-5
HEADS = 4
U32 = 2.0 ** -24      # fp32 unit roundoff


def to_numpy(state_dict):
    return {k: v.detach().cpu().double().numpy() for k, v in state_dict.items()}


def seeded_state_dict(seed, dim=256, enc=(32, 64, 128, 256), n_layers=18, bin_score=1.0, proj_gain=1.0):
    """Random SuperGlue weights (torch tensors, fp32) with SuperGlue's key names and random BN statistics.  Each layer's
    residual branch (mlp.3) and the keypoint encoder's last layer are scaled by 0.1, so that 18 layers keep the
    descriptors' scale, and final_proj by proj_gain (16 makes equal unit descriptors score far above unrelated ones)."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    sd = {}

    def conv(name, cin, cout, gain=1.0):
        sd[f'{name}.weight'] = torch.randn(cout, cin, 1, generator=g) * (gain * gain / cin) ** 0.5
        sd[f'{name}.bias'] = torch.randn(cout, generator=g) * 0.01

    def bn(name, c):
        sd[f'{name}.weight'] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[f'{name}.bias'] = 0.1 * torch.randn(c, generator=g)
        sd[f'{name}.running_mean'] = 0.1 * torch.randn(c, generator=g)
        sd[f'{name}.running_var'] = 0.5 + torch.rand(c, generator=g)
        sd[f'{name}.num_batches_tracked'] = torch.tensor(0)

    chans = [3] + list(enc) + [dim]
    for i in range(1, len(chans)):
        conv(f'kenc.encoder.{3 * (i - 1)}', chans[i - 1], chans[i], 1.0 if i < len(chans) - 1 else 0.1)
        if i < len(chans) - 1:
            bn(f'kenc.encoder.{3 * (i - 1) + 1}', chans[i])
    for k in range(n_layers):
        for p in range(3):
            conv(f'gnn.layers.{k}.attn.proj.{p}', dim, dim)
        conv(f'gnn.layers.{k}.attn.merge', dim, dim)
        conv(f'gnn.layers.{k}.mlp.0', 2 * dim, 2 * dim)
        bn(f'gnn.layers.{k}.mlp.1', 2 * dim)
        conv(f'gnn.layers.{k}.mlp.3', 2 * dim, dim, 0.1)
    conv('final_proj', dim, dim, proj_gain)
    sd['bin_score'] = torch.tensor(float(bin_score))
    return sd


def normalize_keypoints(kpts, h, w):
    """kpts [N, 2] (x, y) -> (kpts - [w/2, h/2]) / (0.7 max(w, h))."""
    return (np.asarray(kpts, np.float64) - np.array([w / 2.0, h / 2.0])) / (0.7 * max(w, h))


def _conv(sd, name, x):
    return sd[f'{name}.weight'][:, :, 0] @ x + sd[f'{name}.bias'][:, None]


def _bn(sd, name, x):
    scale = sd[f'{name}.weight'] / np.sqrt(sd[f'{name}.running_var'] + BN_EPS)
    return (x - sd[f'{name}.running_mean'][:, None]) * scale[:, None] + sd[f'{name}.bias'][:, None]


def _mlp(sd, prefix, n_convs, x):
    for k in range(n_convs):
        x = _conv(sd, f'{prefix}.{3 * k}', x)
        if k < n_convs - 1:
            x = np.maximum(_bn(sd, f'{prefix}.{3 * k + 1}', x), 0.0)
    return x


def _attention(sd, prefix, x, src):
    dim = x.shape[0]
    hd = dim // HEADS
    q, k, v = (_conv(sd, f'{prefix}.proj.{p}', t).reshape(hd, HEADS, -1) for p, t in enumerate((x, src, src)))
    msg = np.empty((hd, HEADS, x.shape[1]))
    for h in range(HEADS):                       # channel c = d * HEADS + h belongs to head h
        logits = q[:, h, :].T @ k[:, h, :] / np.sqrt(hd)
        logits -= logits.max(1, keepdims=True)
        p = np.exp(logits)
        p /= p.sum(1, keepdims=True)
        msg[:, h, :] = v[:, h, :] @ p.T
    return _conv(sd, f'{prefix}.merge', msg.reshape(dim, -1))


def scores(sd, kpts0, kpts1, sc0, sc1, desc0, desc1, shape0, shape1, layer_names, n_enc):
    """One pair: kpts [N, 2], sc [N], desc [D, N], shape (H, W) -> scores [N0, N1] = mdesc0^T mdesc1 / sqrt(D).
    n_enc is the keypoint encoder's conv count (5 for the default config)."""
    dim = desc0.shape[0]
    d = []
    for k, s, e, (h, w) in ((kpts0, sc0, desc0, shape0), (kpts1, sc1, desc1, shape1)):
        inp = np.concatenate([normalize_keypoints(k, h, w).T, np.asarray(s, np.float64)[None]], 0)
        d.append(np.asarray(e, np.float64) + _mlp(sd, 'kenc.encoder', n_enc, inp))
    d0, d1 = d
    for li, name in enumerate(layer_names):
        s0, s1 = (d1, d0) if name == 'cross' else (d0, d1)
        p = f'gnn.layers.{li}'
        m0 = _mlp(sd, f'{p}.mlp', 2, np.concatenate([d0, _attention(sd, f'{p}.attn', d0, s0)], 0))
        m1 = _mlp(sd, f'{p}.mlp', 2, np.concatenate([d1, _attention(sd, f'{p}.attn', d1, s1)], 0))
        d0, d1 = d0 + m0, d1 + m1
    f0, f1 = _conv(sd, 'final_proj', d0), _conv(sd, 'final_proj', d1)
    return f0.T @ f1 / np.sqrt(dim)


def _lse(x, axis):
    mx = x.max(axis, keepdims=True)
    return (mx + np.log(np.exp(x - mx).sum(axis, keepdims=True))).squeeze(axis)


def log_optimal_transport(s, alpha, iters):
    """One pair: scores [n, m] -> (log_assign [n+1, m+1] float64, the largest |u|, |v| over all iterations)."""
    s = np.asarray(s, np.float64)
    n, m = s.shape
    C = np.full((n + 1, m + 1), float(alpha))
    C[:n, :m] = s
    norm = -np.log(n + m)
    log_mu = np.concatenate([np.full(n, norm), [np.log(m) + norm]])
    log_nu = np.concatenate([np.full(m, norm), [np.log(n) + norm]])
    u, v = np.zeros(n + 1), np.zeros(m + 1)
    vmax = 0.0
    for _ in range(iters):
        u = log_mu - _lse(C + v[None, :], 1)
        v = log_nu - _lse(C + u[:, None], 0)
        vmax = max(vmax, np.abs(u).max(), np.abs(v).max())
    return C + u[:, None] + v[None, :] - norm, vmax


def extract(la, threshold):
    """Mutual-argmax extraction on the top-left n x m block of log_assign -> dict of matches0 / matches1 (int, -1 for
    none), mscores0 / mscores1, mutual0 / mutual1, and the row / column argmaxes i0 / i1.  Ties: lowest index."""
    z = np.asarray(la, np.float64)[:-1, :-1]
    n, m = z.shape
    i0, i1 = z.argmax(1), z.argmax(0)
    mutual0 = i1[i0] == np.arange(n)
    mutual1 = i0[i1] == np.arange(m)
    ms0 = np.where(mutual0, np.exp(z.max(1)), 0.0)
    ms1 = np.where(mutual1, ms0[i1], 0.0)
    valid0 = mutual0 & (ms0 > threshold)
    valid1 = mutual1 & valid0[i1]
    return {'matches0': np.where(valid0, i0, -1), 'matches1': np.where(valid1, i1, -1), 'mscores0': ms0,
            'mscores1': ms1, 'mutual0': mutual0, 'mutual1': mutual1, 'i0': i0, 'i1': i1}


def decidable(la, threshold, tol):
    """Rows and columns whose decisions no perturbation of log_assign's n x m block by less than tol / 2 per entry can
    change: their own top-1 / top-2 gap, the gap of the line their argmax points to, and |max - log(threshold)| of the
    row that sets their threshold test all exceed tol.  -> (rows [n] bool, columns [m] bool)."""
    z = np.asarray(la, np.float64)[:-1, :-1]
    n, m = z.shape

    def gap(a, axis):
        if a.shape[axis] < 2:
            return np.full(a.shape[1 - axis], np.inf)
        p = -np.partition(-a, 1, axis=axis)
        return (p[0] - p[1]) if axis == 0 else (p[:, 0] - p[:, 1])

    g0, g1 = gap(z, 1), gap(z, 0)
    i0, i1 = z.argmax(1), z.argmax(0)
    thr_ok = np.abs(z.max(1) - np.log(threshold)) > tol if threshold > 0 else np.ones(n, bool)
    rows = (g0 > tol) & (g1[i0] > tol) & thr_ok
    cols = (g1 > tol) & (g0[i1] > tol) & thr_ok[i1]
    return rows, cols


def decidable_ties(la, threshold, tol):
    """decidable() for matrices with exact ties: duplicated keypoints make bit-identical lines, whose entries are equal
    in float64 and in fp32 alike, and a masked (all -inf) line ties everywhere.  Such a tie resolves to the lowest index
    on both sides, so a line's gap is taken from its maximum to the largest value strictly below it (infinite when
    there is none).  Lines with a NaN are never decided here; compare those
    with extract() exactly.  -> (rows [n] bool, columns [m] bool)."""
    z = np.asarray(la, np.float64)[:-1, :-1]
    n, m = z.shape

    def gap(axis):
        with np.errstate(invalid='ignore'):
            top = z.max(axis)
            below = np.where(z < np.expand_dims(top, axis), z, -np.inf).max(axis)
            g = np.where(np.isneginf(top), np.inf, top - below)
        return np.where(np.isnan(top), -np.inf, g)

    g0, g1 = gap(1), gap(0)
    i0, i1 = z.argmax(1), z.argmax(0)
    with np.errstate(invalid='ignore'):
        thr_ok = np.abs(z.max(1) - np.log(threshold)) > tol if threshold > 0 else np.ones(n, bool)
    # a masked line's whole decision is exact: it points at 0, and that line's argmax is either a finite entry (not
    # mutual) or, masked too, 0 (mutual iff this is line 0), with score exp(-inf) = 0
    rows = (g0 > tol) & (g1[i0] > tol) & thr_ok | np.isneginf(z).all(1)
    cols = (g1 > tol) & (g0[i1] > tol) & thr_ok[i1] | np.isneginf(z).all(0)
    return rows, cols


def sinkhorn_bound(n, m, amax, vmax, iters):
    """Bound on |log_assign - log_assign_fp64| of p2p_sg_sinkhorn (DESIGN.md, "SuperGlue's optimal transport"): each
    half-iteration adds at most delta = u (10 (A + V) + 16 K + 4 lambda + 40) to the error of u or v, with A = max |C|
    (scores and alpha), V = max |u|, |v| over the iterations, K = ceil((max(n, m) + 1) / 256) chunk steps per lane and
    lambda = log(n + m + 1); log_assign adds the errors of u_i and v_j and rounds three more times."""
    W = amax + vmax
    K = math.ceil((max(n, m) + 1) / 256)
    lam = math.log(n + m + 1)
    delta = U32 * (10 * W + 16 * K + 4 * lam + 40)
    return 4 * iters * delta + 4 * U32 * (amax + 2 * vmax + lam)
