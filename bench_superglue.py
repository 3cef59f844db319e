"""SuperGlue's optimal transport on the GPU: p2p_sg_sinkhorn (one cooperative launch, Sinkhorn + extraction) against an
fp32 PyTorch restatement of log_optimal_transport plus the max / gather extraction, on the same inputs; and the share of
SuperGlue.forward that the optimal transport takes.

    python bench_superglue.py [--sizes 512,1024,2048,4096,8192] [--iters 100] [--reps 10]

Prints the card (name, power limit, max SM clock), then one line per size: time and peak memory per arm, bytes per run
(from the shapes) and the achieved rate, the arms' agreement, and the kernel's error against float64 at the smaller
sizes.  Writes nothing."""
import argparse
import json
import subprocess

import numpy as np
import torch

from oracle import superglue_oracle as O
from patch2pix_b200 import superglue as SG

L2_BYTES = 50 * 2 ** 20
HBM_BPS = 3.35e12          # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                     # report, do not guess
        q = f'nvidia-smi unavailable ({e})'
    return q


def torch_ot(scores, alpha, iters, thr):
    """fp32 PyTorch restatement: log_optimal_transport, then SuperGlue's max / gather extraction."""
    b, n, m = scores.shape
    one = scores.new_tensor(1)
    ms, ns = m * one, n * one
    C = torch.cat([torch.cat([scores, alpha.expand(b, n, 1)], -1), alpha.expand(b, 1, m + 1)], 1)
    norm = -(ms + ns).log()
    log_mu = torch.cat([norm.expand(n), ms.log()[None] + norm]).expand(b, -1)
    log_nu = torch.cat([norm.expand(m), ns.log()[None] + norm]).expand(b, -1)
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(C + v.unsqueeze(1), dim=2)
        v = log_nu - torch.logsumexp(C + u.unsqueeze(2), dim=1)
    la = C + u.unsqueeze(2) + v.unsqueeze(1) - norm
    z = la[:, :-1, :-1]
    max0, max1 = z.max(2), z.max(1)
    i0, i1 = max0.indices, max1.indices
    ar0 = torch.arange(n, device=z.device)[None]
    ar1 = torch.arange(m, device=z.device)[None]
    mutual0 = ar0 == i1.gather(1, i0)
    mutual1 = ar1 == i0.gather(1, i1)
    s0 = torch.where(mutual0, max0.values.exp(), z.new_tensor(0))
    s1 = torch.where(mutual1, s0.gather(1, i1), z.new_tensor(0))
    valid0 = mutual0 & (s0 > thr)
    valid1 = mutual1 & valid0.gather(1, i1)
    return la, torch.where(valid0, i0, -1), torch.where(valid1, i1, -1), s0, s1


def planted(n, m, seed=0, d=64, scale=20.0, dev='cuda'):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.nn.functional.normalize(torch.randn(n, d, generator=g, device=dev), dim=1)
    b = torch.nn.functional.normalize(torch.randn(m, d, generator=g, device=dev), dim=1)
    k = int(0.7 * min(n, m))
    b[:k] = torch.nn.functional.normalize(a[:k] + 0.3 * torch.nn.functional.normalize(
        torch.randn(k, d, generator=g, device=dev), dim=1), dim=1)
    return (a @ b.T * scale)[None].contiguous()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='512,1024,2048,4096,8192')
    ap.add_argument('--iters', type=int, default=100)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-max', type=int, default=1024, help='largest N checked against float64 (CPU time)')
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device('cuda:0')
    print(json.dumps({'card': card(), 'device': torch.cuda.get_device_name(dev)}))
    alpha = torch.tensor(1.0, device=dev)
    thr = 0.2
    for N in (int(s) for s in args.sizes.split(',')):
        scores = planted(N, N)
        reps = max(1, args.reps if N <= 4096 else args.reps // 2)
        t_k, mem_k, ko = timed(lambda: SG._sinkhorn(scores, alpha, args.iters, thr, log_assign=False), reps)
        t_t, mem_t, to = timed(lambda: torch_ot(scores, alpha, args.iters, thr), reps)
        nm = 4 * N * N
        # bytes: the transpose reads and writes 4 N M once; each half-iteration reads 4 N M; the last pass reads both
        bytes_run = 2 * nm + 2 * args.iters * nm + 2 * nm
        bound = 'L2' if 2 * nm <= L2_BYTES else 'HBM'
        kla = SG._sinkhorn(scores, alpha, args.iters, thr, log_assign=True)
        rec = {'N': N, 'iters': args.iters, 'kernel_ms': round(t_k, 3), 'torch_ms': round(t_t, 3),
               'speedup': round(t_t / t_k, 2),
               # the kernel's scratch (the transposed copy, u, v, argmaxes) lives in the handle, outside torch's allocator
               'kernel_peak_MiB': round(mem_k + (nm + 16 * (N + 1)) / 2 ** 20, 1), 'torch_peak_MiB': round(mem_t, 1),
               'kernel_bytes_per_run': bytes_run, 'kernel_GBps': round(bytes_run / t_k / 1e6, 1),
               'working_set': bound,
               'hbm_share': round(bytes_run / t_k / 1e-3 / HBM_BPS, 3) if bound == 'HBM' else 'n/a (L2-resident)',
               'max_abs_dlog_assign_vs_torch': float((kla['log_assign'] - to[0]).abs().max()),
               'matches0_equal': bool(torch.equal(kla['matches0'].long(), to[1])),
               'matches1_equal': bool(torch.equal(kla['matches1'].long(), to[2])),
               'matches0_valid': int((kla['matches0'] >= 0).sum())}
        if N <= args.oracle_max:
            ref, vmax = O.log_optimal_transport(scores[0].double().cpu().numpy(), 1.0, args.iters)
            b = O.sinkhorn_bound(N, N, max(1.0, float(scores.abs().max())), vmax, args.iters)
            rec['max_abs_err_vs_fp64'] = float(np.abs(kla['log_assign'][0].double().cpu().numpy() - ref).max())
            rec['derived_bound'] = b
        del kla, to, ko
        print(json.dumps(rec))
        torch.cuda.empty_cache()

    # share of SuperGlue.forward at N = M = 2048 (random weights, TF32 off)
    N = 2048
    sg = SG.SuperGlue()
    sg.load_state_dict(O.seeded_state_dict(0, proj_gain=16.0))
    sg = sg.to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    data = {'image0': torch.zeros(1, 1, 768, 1024, device=dev), 'image1': torch.zeros(1, 1, 768, 1024, device=dev)}
    for i in (0, 1):
        data[f'keypoints{i}'] = torch.rand(1, N, 2, generator=g, device=dev) * torch.tensor([1023., 767.], device=dev)
        data[f'scores{i}'] = torch.rand(1, N, generator=g, device=dev)
        data[f'descriptors{i}'] = torch.nn.functional.normalize(torch.randn(1, 256, N, generator=g, device=dev), dim=1)
    with torch.no_grad():
        t_f, _, _ = timed(lambda: sg(data), 5)
        t_s, _, sc = timed(lambda: sg.score_matrix(data), 5)
        t_o, _, _ = timed(lambda: SG._sinkhorn(sc, sg.bin_score, 100, 0.2), 5)
    print(json.dumps({'forward_N': N, 'forward_ms': round(t_f, 3), 'gnn_and_scores_ms': round(t_s, 3),
                      'ot_ms': round(t_o, 3), 'ot_share': round(t_o / t_f, 3)}))


if __name__ == '__main__':
    main()
