"""float64 restatement of NCNet's matcher (the reference's networks/ncn/model.py) for checking the CUDA path.

Written from the operations' definitions, not from the reference's code:
  l2norm        f / sqrt(sum_c f^2 + 1e-6)
  correlation   corr[iA, jA, iB, jB] = <fA[:, iA, jA], fB[:, iB, jB]>
  maxpool4d     max over each k^4 box, with the box offsets (di, dj, dk, dl) of the first maximum in row-major order
  mutual        x * (x / (max over A + 1e-5)) * (x / (max over B + 1e-5))
  conv4d        out[o, a, b, c, d] = bias[o] + sum_{i, taps} w[o, i, taps] * x[i, a + ta - p, ..., d + td - p], zero
                outside the volume ("same" cross-correlation); weights in the reference's pre-permuted layout
                [k, Cout, Cin, k, k, k], i.e. w[o, i, ta, tb, tc, td] = W[ta, o, i, tb, tc, td]
  stack         conv4d + ReLU per layer; symmetric: stack(x) + stack(x^T)^T with x^T swapping the (A) and (B) axes
"""
import torch


def l2norm(f):
    f = f.double()
    return f / torch.sqrt((f * f).sum(1, keepdim=True) + 1e-6)


def correlation(fa, fb):
    """fa [C, hA, wA], fb [C, hB, wB] -> [hA, wA, hB, wB]."""
    c, hA, wA = fa.shape
    _, hB, wB = fb.shape
    return (fa.reshape(c, -1).t() @ fb.reshape(c, -1)).reshape(hA, wA, hB, wB)


def maxpool4d(x, k):
    """x [H1, W1, H2, W2] -> (pooled [H1/k, ..], di, dj, dk, dl int64)."""
    H1, W1, H2, W2 = x.shape
    v = x.reshape(H1 // k, k, W1 // k, k, H2 // k, k, W2 // k, k).permute(0, 2, 4, 6, 1, 3, 5, 7)
    v = v.reshape(H1 // k, W1 // k, H2 // k, W2 // k, k ** 4)
    m = v.max(-1).values
    idx = (v == m.unsqueeze(-1)).double().argmax(-1)          # first maximum
    return m, idx // k ** 3, (idx // k ** 2) % k, (idx // k) % k, idx % k


def mutual(x):
    hA, wA, hB, wB = x.shape
    v = x.reshape(hA * wA, hB * wB)
    ma = v.max(1, keepdim=True).values
    mb = v.max(0, keepdim=True).values
    return (v * ((v / (ma + 1e-5)) * (v / (mb + 1e-5)))).reshape(x.shape)


def conv4d(x, weight, bias):
    """x [Cin, hA, wA, hB, wB] float64; weight [k, Cout, Cin, k, k, k]; bias [Cout] -> [Cout, hA, wA, hB, wB]."""
    w = weight.double().permute(1, 2, 0, 3, 4, 5)              # [Cout, Cin, k, k, k, k]
    k = w.shape[-1]
    p = k // 2
    cin, hA, wA, hB, wB = x.shape
    xp = torch.nn.functional.pad(x.double(), (p, p, p, p, p, p, p, p))
    out = bias.double().reshape(-1, 1, 1, 1, 1).repeat(1, hA, wA, hB, wB)
    for a in range(k):
        for b in range(k):
            for c in range(k):
                for d in range(k):
                    sl = xp[:, a:a + hA, b:b + wA, c:c + hB, d:d + wB].reshape(cin, -1)
                    out += (w[:, :, a, b, c, d] @ sl).reshape(out.shape)
    return out


def nc_stack(x, weights, biases, symmetric=True):
    """x [hA, wA, hB, wB]; weights / biases: per layer, reference layout -> [hA, wA, hB, wB] float64."""
    def run(v):
        v = v.double().unsqueeze(0)
        for w, b in zip(weights, biases):
            v = torch.relu(conv4d(v, w, b))
        return v[0]
    out = run(x)
    if symmetric:
        out = out + run(x.permute(2, 3, 0, 1)).permute(2, 3, 0, 1)
    return out


def forward_feat(fa, fb, weights, biases, ksize, symmetric=True):
    """ImMatchNet.forward_feat(normalize=True) for one pair of layer3 maps [C, h, w] -> (corr4d, deltas | None)."""
    x = correlation(l2norm(fa.unsqueeze(0))[0], l2norm(fb.unsqueeze(0))[0])
    deltas = None
    if ksize > 1:
        x, *deltas = maxpool4d(x, ksize)
    x = mutual(x)
    x = nc_stack(x, weights, biases, symmetric)
    return mutual(x), deltas


def corr_to_matches(corr, deltas=None, ksize=1, do_softmax=True, scale='positive', invert=False, return_indices=True):
    """corr [hA, wA, hB, wB] -> (jA, iA, jB, iB, score) for every B cell (every A cell with invert): the arg-max over
    the other image's cells of the (softmax-normalised over those cells) correlation, indices refined by the maxpool
    offsets (index * ksize + delta).  return_indices=False maps indices to linspace(lo, 1) coordinates of the grid at
    ksize x resolution, lo = 0 ('positive') or -1 ('centered')."""
    hA, wA, hB, wB = corr.shape
    v = corr.double().reshape(hA * wA, hB * wB)
    if invert:
        v = v.t()
    if do_softmax:
        v = torch.softmax(v, 0)
    score, idx = v.max(0)
    mine = torch.arange(v.shape[1])
    a, bcell = (mine, idx) if invert else (idx, mine)
    iA, jA, iB, jB = a // wA, a % wA, bcell // wB, bcell % wB
    if deltas is not None:
        d = [t.reshape(hA, wA, hB, wB)[iA, jA, iB, jB].long() for t in deltas]
        iA, jA, iB, jB = iA * ksize + d[0], jA * ksize + d[1], iB * ksize + d[2], jB * ksize + d[3]
    if return_indices:
        return jA, iA, jB, iB, score
    lo = -1.0 if scale == 'centered' else 0.0
    lin = lambda n: torch.linspace(lo, 1.0, n, dtype=torch.float64)
    return lin(wA * ksize)[jA], lin(hA * ksize)[iA], lin(wB * ksize)[jB], lin(hB * ksize)[iB], score
