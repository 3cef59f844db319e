"""CPU restatement of SuperPoint + nearest-neighbour matching (patch2pix_b200/superpoint.py, csrc/keypoints.cu), for
the tests: the network in torch-CPU fp32, the NMS / border / threshold / top-k rules in numpy, descriptor sampling in
float64 and the matcher's float64 similarities summed over k = 0 .. D-1 in that order.
"""
import numpy as np
import torch
import torch.nn.functional as F

CONVS = [('conv1a', 1, 64, 3), ('conv1b', 64, 64, 3), ('conv2a', 64, 64, 3), ('conv2b', 64, 64, 3),
         ('conv3a', 64, 128, 3), ('conv3b', 128, 128, 3), ('conv4a', 128, 128, 3), ('conv4b', 128, 128, 3),
         ('convPa', 128, 256, 3), ('convPb', 256, 65, 1), ('convDa', 128, 256, 3), ('convDb', 256, 256, 1)]


def seeded_state_dict(seed):
    """Random SuperPoint weights with SuperGlue's key names (He-scaled, small biases)."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for name, cin, cout, k in CONVS:
        sd[f'{name}.weight'] = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
        sd[f'{name}.bias'] = torch.randn(cout, generator=g) * 0.01
    return sd


def heads(sd, image):
    """torch-CPU fp32 network: grey [B, 1, H, W] -> (logits [B, 65, H/8, W/8], raw descriptors [B, 256, H/8, W/8])."""
    def conv(x, n, k):
        return F.conv2d(x, sd[f'{n}.weight'].float(), sd[f'{n}.bias'].float(), padding=k // 2)
    x = image.float()
    for i, s in enumerate('1234'):
        x = F.relu(conv(x, f'conv{s}a', 3))
        x = F.relu(conv(x, f'conv{s}b', 3))
        if i < 3:
            x = F.max_pool2d(x, 2, 2)
    return conv(F.relu(conv(x, 'convPa', 3)), 'convPb', 1), conv(F.relu(conv(x, 'convDa', 3)), 'convDb', 1)


def score_map(logits):
    """[65, Hc, Wc] logits -> [8Hc, 8Wc] fp32 scores (torch-CPU softmax, dustbin dropped, depth-to-space)."""
    s = torch.softmax(torch.as_tensor(logits).float(), 0)[:-1]
    hc, wc = s.shape[1:]
    return s.permute(1, 2, 0).reshape(hc, wc, 8, 8).permute(0, 2, 1, 3).reshape(hc * 8, wc * 8).numpy()


def maxpool(a, r):
    """(2r+1)^2 max, stride 1; out-of-image taps never win."""
    a = np.asarray(a)
    H, W = a.shape
    p = np.full((H + 2 * r, W + 2 * r), -np.inf, dtype=np.float64)
    p[r:r + H, r:r + W] = a
    rows = np.max(np.stack([p[:, d:d + W] for d in range(2 * r + 1)]), 0)
    return np.max(np.stack([rows[d:d + H] for d in range(2 * r + 1)]), 0)


def nms(s, r):
    """SuperGlue's max-pool NMS: the map with every non-kept pixel set to 0."""
    s = np.asarray(s, dtype=np.float32)
    M = s == maxpool(s, r)
    for _ in range(2):
        S = maxpool(M.astype(np.float32), r) > 0
        s2 = np.where(S, np.float32(0), s)
        M = M | ((s2 == maxpool(s2, r)) & ~S)
    return np.where(M, s, np.float32(0))


def keypoints(s, r=4, threshold=0.005, border=4, max_keypoints=-1):
    """[H, W] score map -> (keypoints [N, 2] float32 (x, y), scores [N] float32) by the rules of p2p_sp_keypoints."""
    kept = nms(s, r)
    H, W = kept.shape
    ys, xs = np.mgrid[:H, :W]
    cand = (kept > np.float32(threshold)) & (ys >= border) & (ys < H - border) & (xs >= border) & (xs < W - border)
    idx = np.flatnonzero(cand)                     # row-major
    sc = kept.reshape(-1)[idx]
    if max_keypoints >= 0:
        order = np.lexsort((idx, -sc.astype(np.float64)))[:max_keypoints]
        idx, sc = idx[order], sc[order]
    return np.stack([idx % W, idx // W], 1).astype(np.float32), sc.astype(np.float32)


def sample_descriptors(desc, kps):
    """desc [D, Hc, Wc] raw, kps [N, 2] (x, y) -> [N, D] float64: cells normalised, bilinear at SuperGlue's
    coordinates (grid_sample, align_corners=True, zero padding), renormalised."""
    d = np.asarray(desc, dtype=np.float64)
    D, hc, wc = d.shape
    d = d / np.maximum(np.sqrt((d * d).sum(0)), 1e-12)
    kps = np.asarray(kps, dtype=np.float64).reshape(-1, 2)
    gx = (kps[:, 0] - 3.5) / (8.0 * wc - 4.5) * 2.0 - 1.0
    gy = (kps[:, 1] - 3.5) / (8.0 * hc - 4.5) * 2.0 - 1.0
    ix, iy = (gx + 1.0) * 0.5 * (wc - 1), (gy + 1.0) * 0.5 * (hc - 1)
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    ax, ay = ix - x0, iy - y0
    out = np.zeros((len(kps), D))
    for dx, dy, w in ((0, 0, (1 - ax) * (1 - ay)), (1, 0, ax * (1 - ay)), (0, 1, (1 - ax) * ay), (1, 1, ax * ay)):
        x, y = x0 + dx, y0 + dy
        ok = (x >= 0) & (x < wc) & (y >= 0) & (y < hc)
        out[ok] += w[ok, None] * d[:, y[ok], x[ok]].T
    return out / np.maximum(np.sqrt((out * out).sum(1)), 1e-12)[:, None]


def similarity(d0, d1):
    """float64 [N, M]: sum over k = 0 .. D-1, in that order, of the exact products d0[i, k] * d1[j, k]."""
    a = np.asarray(d0, dtype=np.float32).astype(np.float64)
    b = np.asarray(d1, dtype=np.float32).astype(np.float64)
    S = np.zeros((a.shape[0], b.shape[0]))
    for k in range(a.shape[1]):
        S += a[:, k, None] * b[None, :, k]
    return S


def match(d0, d1, mutual=True, min_sim=None, ratio=None, S=None):
    """-> (matches0 [N] int64 (-1: none), sim0 [N] float64 (0 for none)) by the rules of p2p_match_descriptors_batch."""
    S = similarity(d0, d1) if S is None else S
    N, M = S.shape
    m = np.full(N, -1, dtype=np.int64)
    sim = np.zeros(N)
    if N == 0 or M == 0:
        return m, sim
    j1 = np.argmax(S, 1)                          # first maximum: the lowest index of a tie
    s1 = S[np.arange(N), j1]
    rest = S.copy()
    rest[np.arange(N), j1] = -np.inf
    s2 = rest.max(1) if M > 1 else np.full(N, -np.inf)
    ok = np.ones(N, dtype=bool)
    if mutual:
        ok &= np.argmax(S, 0)[j1] == np.arange(N)
    if min_sim is not None:
        ok &= s1 > float(min_sim)
    if ratio is not None and M > 1:
        r = float(ratio)
        ok &= (1.0 - s1) < r * r * (1.0 - s2)
    m[ok] = j1[ok]
    sim[ok] = s1[ok]
    return m, sim
