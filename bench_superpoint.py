"""Throughput of SuperPoint's post-network steps and of exact descriptor matching (patch2pix_b200.superpoint) against
the same steps in PyTorch.

    python bench_superpoint.py [--pairs 512] [--kp 4096] [--dim 256] [--reps 5]

  (a) detection + descriptors of one 1024 x 768 image from seeded head outputs (logits [1, 65, 96, 128], descriptors
      [1, 256, 96, 128]): p2p_sp_keypoints + p2p_sp_descriptors against PyTorch's softmax, depth-to-space, max-pool
      NMS, nonzero, border mask, topk and grid_sample (SuperGlue's published steps), with max_keypoints -1 and 2048.
  (b) mutual nearest-neighbour matching of --pairs pairs of --kp x --dim unit descriptors in one
      match_descriptors_batch call (tensor-core pass + float64 fix-up, exact), against the same call with option
      match_impl 0 (float64 on the CUDA cores only, same result), a per-pair loop of fp32 torch.matmul + row / column
      argmax, and chunks of batched float64 torch.bmm + argmax.
Every arm's output is checked against the project's before timing: keypoints equal, descriptors within 1e-5, and the
share of rows whose fp32 / fp64 torch match agrees with the exact one.  Each arm is warmed up, then timed --reps times
with CUDA events, the fastest reported.  Prints one JSON line with the card's name, power limit and SM clock.
"""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

from patch2pix_b200 import superpoint as SP


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else None


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def torch_detect(logits, desc, r=4, thr=0.005, border=4, k=-1):
    s = torch.softmax(logits, 1)[:, :-1]
    b, _, h, w = s.shape
    s = s.permute(0, 2, 3, 1).reshape(b, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, h * 8, w * 8)

    def mp(x):
        return F.max_pool2d(x, 2 * r + 1, 1, r)
    s4 = s[:, None]
    M = s4 == mp(s4)
    for _ in range(2):
        S = mp(M.float()) > 0
        s2 = torch.where(S, torch.zeros_like(s4), s4)
        M = M | ((s2 == mp(s2)) & ~S)
    s = torch.where(M, s4, torch.zeros_like(s4))[:, 0]
    kp = torch.nonzero(s[0] > thr)
    H, W = s.shape[1:]
    keep = (kp[:, 0] >= border) & (kp[:, 0] < H - border) & (kp[:, 1] >= border) & (kp[:, 1] < W - border)
    kp = kp[keep]
    sc = s[0][tuple(kp.t())]
    if k >= 0:
        sc, i = torch.topk(sc, min(k, len(sc)))
        kp = kp[i]
    kp = kp.flip(1).float()
    d = F.normalize(desc, p=2, dim=1)
    g = (kp - 3.5) / torch.tensor([8 * w - 4.5, 8 * h - 4.5], device=kp.device)
    g = g * 2 - 1
    d = F.grid_sample(d, g.view(1, 1, -1, 2), mode='bilinear', align_corners=True)
    return kp, sc, F.normalize(d.reshape(1, desc.shape[1], -1), p=2, dim=1)[0].t()


def ours_detect(logits, desc, k=-1):
    kps, scs = SP.detect_keypoints(logits, 4, 0.005, k, 4)
    return kps[0], scs[0], SP.sample_descriptors(desc, kps)[0]


def torch_match(d0, d1, dtype):
    out = []
    for a, b in zip(d0, d1):
        S = a.to(dtype) @ b.to(dtype).t()
        j = S.argmax(1)
        i = S.argmax(0)
        out.append(torch.where(i[j] == torch.arange(len(a), device=a.device), j, -1))
    return out


def torch_match_bmm(A, B, chunk=32):
    out = []
    ar = torch.arange(A.shape[1], device=A.device)
    for c in range(0, A.shape[0], chunk):       # 32 pairs of 4096 x 4096 float64 similarities: 4.3 GB at a time
        S = torch.bmm(A[c:c + chunk].double(), B[c:c + chunk].double().transpose(1, 2))
        j = S.argmax(2)
        i = S.argmax(1)
        out.append(torch.where(torch.gather(i, 1, j) == ar, j, -1))
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=512)
    ap.add_argument('--kp', type=int, default=4096)
    ap.add_argument('--dim', type=int, default=256)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda:0')
    g = torch.Generator(device=dev).manual_seed(0)
    res = {'card': card()}

    logits = torch.randn(1, 65, 96, 128, device=dev, generator=g) * 3
    desc = torch.randn(1, 256, 96, 128, device=dev, generator=g)
    for k in (-1, 2048):
        kp, sc, dd = ours_detect(logits, desc, k)
        tkp, tsc, tdd = torch_detect(logits, desc, k=k)
        if k < 0:
            assert torch.equal(kp, tkp) and torch.equal(sc, tsc), 'keypoints differ from the PyTorch arm'
        else:   # topk's order among exactly equal scores is unspecified: compare as sets, descriptors by keypoint
            assert torch.equal(sc, tsc) and len(kp) == len(tkp)
            key, tkey = kp[:, 1] * 65536 + kp[:, 0], tkp[:, 1] * 65536 + tkp[:, 0]
            o, to = torch.argsort(key), torch.argsort(tkey)
            assert torch.equal(key[o], tkey[to]), 'top-k keypoints differ from the PyTorch arm'
            dd, tdd = dd[o], tdd[to]
        assert (dd - tdd).abs().max().item() < 1e-5
        res[f'detect_k{k}'] = {'keypoints': len(kp), 'ours_ms': timed(lambda: ours_detect(logits, desc, k), a.reps),
                               'torch_ms': timed(lambda: torch_detect(logits, desc, k=k), a.reps)}

    A = F.normalize(torch.randn(a.pairs, a.kp, a.dim, device=dev, generator=g), dim=2)
    B = F.normalize(A + 0.3 * torch.randn(a.pairs, a.kp, a.dim, device=dev, generator=g), dim=2)
    l0, l1 = list(A.unbind(0)), list(B.unbind(0))
    ours = SP.match_descriptors_batch(l0, l1)
    t32 = torch_match(l0[:8], l1[:8], torch.float32)
    t64 = torch_match_bmm(A[:8], B[:8])
    agree32 = sum(int((o[0] == t).sum()) for o, t in zip(ours[:8], t32)) / (8 * a.kp)
    agree64 = sum(int((o[0] == t).sum()) for o, t in zip(ours[:8], t64)) / (8 * a.kp)
    assert agree32 > 0.99 and agree64 > 0.99, (agree32, agree64)
    flops = 2.0 * a.pairs * a.kp * a.kp * a.dim
    h = SP._handle(dev)
    h.set_option('match_impl', 0)
    ours64 = SP.match_descriptors_batch(l0[:8], l1[:8])
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(ours[:8], ours64))
    t_fp64 = timed(lambda: SP.match_descriptors_batch(l0, l1), a.reps)
    h.set_option('match_impl', 1)
    probe = {}
    SP._match_batch(l0, l1, True, None, None, probe)
    fixed = probe['n_fixed'].tolist()
    t_ours = timed(lambda: SP.match_descriptors_batch(l0, l1), a.reps)
    t_t32 = timed(lambda: torch_match(l0, l1, torch.float32), a.reps)
    t_t64 = timed(lambda: torch_match_bmm(A, B), max(1, a.reps // 2))
    res['match'] = {'pairs': a.pairs, 'kp': a.kp, 'dim': a.dim, 'ours_tc_fixup_ms': t_ours,
                    'ours_fp64_only_ms': t_fp64, 'torch_fp32_loop_ms': t_t32, 'torch_fp64_bmm_ms': t_t64,
                    'ours_tc_tflops_3pass_both_sides': 6 * flops / t_ours / 1e9,
                    'fixed_up_rows_cols': fixed, 'eps_max': float(probe['eps'].max()),
                    'agree_fp32': agree32, 'agree_fp64_bmm': agree64}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
