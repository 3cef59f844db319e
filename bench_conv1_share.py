"""A/B of the mid stage's shared anchor windows (share_windows 0 / 1) on bench.py's workload.

    python bench_conv1_share.py [--runs 3] [--steps 30] [--warmup 3] [--coords 100000]

640x480 synthetic_pair_shifted pairs, consensus NC weights, ptmax 400, panc 8, features resident in HBM, bench.py's
depth-3 pipelined submit / finish loop.  The two arms alternate, `--runs` timed runs of `--steps` pairs each (CUDA events
around the loop): hot-path pairs/s and launches per pair.  After every timed run, a profiled pass of `--prof-steps` pairs
(CUDA events around every launch group) gives the `conv1_mid` scope (sharing on: the prefix, continuation and
unshared-row launches; off: the single conv1 launch) and the sum of all scopes, per pair.  `mid_conv1_kernels_us`:
torch.profiler over mid-stage calls alone, each conv1 launch and the classification / rgb helpers separately.
`mid_1p_3p_max_px`: per arm, the largest |1-pass mid - 3-pass mid| over at least `--coords`
coordinates of the workload's anchors (the risk band, mid_band = 26 thousandths, must cover it).  Also reads
the card's name, power limit and NVML clocks.  Prints one JSON line and writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
from collections import deque

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H, W, PTMAX, PANC = 480, 640, 400, 8
N_DISTINCT = 8


def card(index):
    try:
        import pynvml as N
        N.nvmlInit()
        h = N.nvmlDeviceGetHandleByIndex(index)
        name = N.nvmlDeviceGetName(h)
        return {'name': name.decode() if isinstance(name, bytes) else name,
                'power_limit_w': N.nvmlDeviceGetPowerManagementLimit(h) / 1e3,
                'sm_clock_mhz': N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_SM),
                'sm_clock_max_mhz': N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM),
                'mem_clock_mhz': N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_MEM)}
    except Exception as e:            # no NVML bindings: report what is missing rather than guess
        return {'name': torch.cuda.get_device_name(index), 'nvml': f'unavailable ({type(e).__name__})'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--prof-steps', type=int, default=10)
    ap.add_argument('--coords', type=int, default=100000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError('bench_conv1_share.py needs a CUDA device: there is no CPU fallback')
    from bench import model_config
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_pair_shifted
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda', torch.cuda.current_device())
    cfg = model_config(dev, PANC)
    cfg.weights_dict = make_seeded_state_dict(0, nc_init='consensus')
    net = Patch2PixB200(cfg)
    h = net._handle
    with torch.no_grad():
        feats = []
        for k in range(N_DISTINCT):
            a, b = synthetic_pair_shifted(k, H, W)
            feats.append((net.extract.forward_all(a.to(dev), [], True), net.extract.forward_all(b.to(dev), [], True)))

    def loop(first, steps):
        q = deque()
        for j in range(steps):
            i = first + j
            f1, f2 = feats[i % N_DISTINCT]
            q.append((i, net.submit_coarse(f1, f2, 2, True)))
            if len(q) >= 3:
                i0, t = q.popleft()
                np.random.seed(i0)
                net.finish_match(t, 0.0, PTMAX)
        while q:
            i0, t = q.popleft()
            np.random.seed(i0)
            net.finish_match(t, 0.0, PTMAX)

    def timed(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        l0 = h.launch_count()
        e0.record()
        loop(args.warmup, steps)
        e1.record()
        torch.cuda.synchronize()
        return steps * 1e3 / e0.elapsed_time(e1), (h.launch_count() - l0) / steps

    res = {'card': card(dev.index), 'workload': f'{W}x{H}, ptmax {PTMAX}, panc {PANC}, synthetic_pair_shifted, consensus NC',
           'runs': {0: [], 1: []}, 'launches_per_pair': {}, 'conv1_mid_ms_per_pair': {0: [], 1: []},
           'profile_ms_per_pair': {0: [], 1: []}, 'shared_rows': {}}

    def profiled(share):
        # per-scope CUDA events around every launch group, a separate pass (the events cost host time)
        h.set_option('share_windows', share)
        h.set_option('profile', 1)
        h.profile_read()
        loop(args.warmup, args.prof_steps)
        torch.cuda.synchronize()
        prof = h.profile_read()
        h.set_option('profile', 0)
        res['conv1_mid_ms_per_pair'][share].append(prof['conv1_mid'][0] / args.prof_steps)
        res['profile_ms_per_pair'][share].append(sum(v[0] for v in prof.values()) / args.prof_steps)

    def mid_kernels(share, anch, f1, f2, calls=5):
        # torch.profiler over mid-stage calls alone: every kernel of the window-map conv1 instantiation, in launch order
        # (share 1: prefix, continuation, unshared rows; share 0: the one conv1), plus the helpers, in us per call
        from torch.profiler import ProfilerActivity, profile
        h.set_option('share_windows', share)
        net.forward_fine_match(f1, f2, [anch], 16, 'center', net.regress_mid)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as pr:
            for _ in range(calls):
                net.forward_fine_match(f1, f2, [anch], 16, 'center', net.regress_mid)
            torch.cuda.synchronize()
        evs = sorted((e for e in pr.events() if e.device_type.name == 'CUDA'), key=lambda e: e.time_range.start)
        out = {}
        conv1 = [e.time_range.elapsed_us() for e in evs if 'umma_gemm_kernel<1, false, 1, 2>' in e.name]
        per = len(conv1) // calls
        names = ['prefix', 'continuation', 'unshared'] if share else ['conv1']
        for i in range(per):
            key = names[i] if i < len(names) else f'conv1_{i}'   # the risk band's 3-pass launches are another instantiation
            out[key] = statistics.median(conv1[i::per])
        for tag in ('window_share_classify_kernel', 'window_rgb_kernel'):
            t = [e.time_range.elapsed_us() for e in evs if tag in e.name]
            if t:
                out[tag] = sum(t) / calls
        return out
    with torch.no_grad():
        for share in (0, 1):
            h.set_option('share_windows', share)
            loop(0, args.warmup)
        for r in range(args.runs):
            for share in (0, 1):
                h.set_option('share_windows', share)
                loop(0, args.warmup)
                pps, lpp = timed(args.steps)
                res['runs'][share].append(pps)
                res['launches_per_pair'][share] = lpp
                res['shared_rows'][share] = h.get_option('shared_rows')
                profiled(share)
        f1, f2 = feats[0]
        np.random.seed(0)
        anch = net.match_from_feats(f1, f2, 2, 0.0, True, PTMAX, return_all=True)[4][0].reshape(-1, 4)
        res['mid_conv1_kernels_us'] = {share: mid_kernels(share, anch, f1, f2) for share in (0, 1)}
        # 1-pass vs 3-pass mid, both arms, over the anchors of the workload's pairs
        worst, coords, k = {0: 0.0, 1: 0.0}, 0, 0
        while coords < args.coords:
            f1, f2 = feats[k % N_DISTINCT]
            np.random.seed(1000 + k)
            h.set_option('share_windows', 1)
            g = net.match_from_feats(f1, f2, 2, 0.0, True, PTMAX, return_all=True)
            anch = g[4][0].reshape(-1, 4)
            h.set_option('mid_band', 0)
            h.set_option('mid_passes', 3)
            mid3 = net.forward_fine_match(f1, f2, [anch], 16, 'center', net.regress_mid)[0][0]
            h.set_option('mid_passes', 1)
            for share in (0, 1):
                h.set_option('share_windows', share)
                mid1 = net.forward_fine_match(f1, f2, [anch], 16, 'center', net.regress_mid)[0][0]
                worst[share] = max(worst[share], (mid1 - mid3).abs().max().item())
            coords += anch.numel()
            k += 1
        h.set_option('share_windows', 1)
        h.set_option('mid_passes', 3)
        h.set_option('mid_band', 26)
    r0, r1 = res['runs'][0], res['runs'][1]
    res['median_pairs_s'] = {0: statistics.median(r0), 1: statistics.median(r1)}
    res['median_gain'] = statistics.median(r1) / statistics.median(r0) - 1.0
    res['every_share_run_faster'] = min(r1) > max(r0)
    c0, c1 = statistics.median(res['conv1_mid_ms_per_pair'][0]), statistics.median(res['conv1_mid_ms_per_pair'][1])
    res['conv1_mid_reduction'] = 1.0 - c1 / c0 if c0 > 0 else None
    # issued MACs per anchor group of 8 rows: 8 x 73 k-steps unshared, 8 x 37 + 2 x 36 shared (x 64 x 64 x 512 each)
    res['conv1_mid_issued_mac_ratio'] = (8 * 37 + 2 * 36) / (8 * 73)
    res['mid_1p_3p_max_px'] = worst            # per share_windows arm
    res['mid_1p_3p_coords'] = coords
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
