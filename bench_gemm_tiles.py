"""Where the time of a 128 x 256 conv GEMM tile goes: prints one JSON line.

    python bench_gemm_tiles.py [--reps 3] [--pairs 3]

1. K sweep of the 256-wide 1-pass instantiation through p2p_test_gemm: M = 204,800 rows, N = 512 (3200 tiles, 25
   rounds on 132 SMs), K = 64 x {9, 18, 36, 72, 96} (96 k-steps is the kernel's step-table limit).  Each launch is
   timed by its per-tile trace (first producer stamp to last epilogue stamp); a least-squares line through the time per
   round against the k-steps gives the per-k-step slope and the per-tile intercept.
2. The per-tile phase trace (option tile_trace) of the conv launches on bench.py's workload (640x480, ptmax 400,
   panc 8), with epi_async 0 (staged epilogue) and 1 (fragment epilogues) alternated in this process.  Per launch kind,
   the medians over tiles of: first-stage wait (tile start to first stage ready), main loop (first stage ready to last
   k-step issued), drain (to the accumulators retired), epilogue (to the epilogue done), and the whole tile.
Stamps are %globaltimer ns taken by the first consumer warpgroup's leader thread (and the producer thread).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

STAGES = ('mid', 'fine', 'band')
KINDS = ('conv1', 'conv1_prefix', 'conv1_cont', 'conv1_unshared', 'conv2')


def tag_name(tag):
    return 'test_gemm' if tag == 24 else f'{KINDS[tag & 7]}_{STAGES[tag >> 3]}'


def device_info():
    info = {'card': torch.cuda.get_device_name(0)}
    try:
        import pynvml as N
        N.nvmlInit()
        h = N.nvmlDeviceGetHandleByIndex(0)
        info['power_limit_w'] = N.nvmlDeviceGetEnforcedPowerLimit(h) / 1e3
        info['sm_max_mhz'] = N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM)
        info['_h'] = h
    except Exception as e:          # NVML missing: report it, the timings stand on their own
        info['nvml_error'] = str(e)
    return info


def sm_clock(info):
    if '_h' not in info:
        return None
    import pynvml as N
    return N.nvmlDeviceGetClockInfo(info['_h'], N.NVML_CLOCK_SM)


def decompose(st):
    """Per-tile phases (us) of one traced launch: stamps [tiles][8]."""
    s = st.astype(np.int64)
    ph = {'first_stage_wait': s[:, 2] - s[:, 1], 'main_loop': s[:, 3] - s[:, 2], 'drain': s[:, 4] - s[:, 3],
          'epilogue': s[:, 5] - s[:, 4], 'tile': s[:, 5] - s[:, 1]}
    rounds = int(np.bincount(s[:, 6]).max())
    return {k: float(np.median(v)) / 1e3 for k, v in ph.items()}, {
        'tiles': int(s.shape[0]), 'rounds': rounds, 'span_us': float(s[:, 5].max() - s[:, 0].min()) / 1e3}


def k_sweep(h, reps, info):
    from patch2pix_b200 import _lib
    M, N = 204800, 512
    out, clocks = [], []
    b = torch.randn(N, 64 * 96, device='cuda')
    c = torch.empty(M, N, device='cuda')
    for ks in (9, 18, 36, 72, 96):
        K = 64 * ks
        a = torch.randn(M, K, device='cuda')
        bk = b[:, :K].contiguous()
        spans, phases = [], []
        for r in range(reps + 1):
            h.set_option('tile_trace', 1)
            _lib.check(h.lib.p2p_test_gemm(h.h, _lib.ptr(a), _lib.ptr(bk), _lib.ptr(c), M, N, K, 1, 0, 1.0,
                                           h.stream()))
            tr = h.tile_traces()
            clocks.append(sm_clock(info))
            if r == 0:
                continue                  # warm-up
            ph, meta = decompose(tr[0][1])
            spans.append(meta['span_us'])
            phases.append(ph)
        meta['span_us'] = float(np.median(spans))
        out.append({'k_steps': ks, **meta, 'us_per_round': meta['span_us'] / meta['rounds'],
                    'phases_us': {k: float(np.median([p[k] for p in phases])) for k in phases[0]}})
        del a
    h.set_option('tile_trace', 0)
    x = np.array([o['k_steps'] for o in out], dtype=np.float64)
    y = np.array([o['us_per_round'] for o in out])
    slope, icpt = np.polyfit(x, y, 1)
    return {'M': M, 'N': N, 'points': out, 'fit_us_per_k_step': float(slope), 'fit_us_per_tile_intercept': float(icpt),
            'sm_mhz_samples': clocks}


def workload(net, pairs, info):
    from patch2pix_b200.synth import synthetic_pair_shifted
    h = net._handle
    feats = []
    for p in range(pairs):
        im1, im2 = synthetic_pair_shifted(p, 480, 640)
        with torch.no_grad():
            feats.append((net.extract.forward_all(im1.cuda(), [], early_feat=True),
                          net.extract.forward_all(im2.cuda(), [], early_feat=True)))
    res, clocks = {}, []
    for rep in range(3):                 # the first round warms up
        for e in (0, 1):
            h.set_option('epi_async', e)
            acc = {}
            for p, (f1, f2) in enumerate(feats):
                h.set_option('tile_trace', 1)
                np.random.seed(p)
                with torch.no_grad():
                    net.match_from_feats(f1, f2, 2, ptmax=400)
                for tag, st in h.tile_traces():
                    if st.shape[0] == 0:      # a launch with no rows (e.g. no unshared rows)
                        continue
                    ph, meta = decompose(st)
                    acc.setdefault(tag_name(tag), []).append((ph, meta))
                clocks.append(sm_clock(info))
            if rep == 0:
                continue
            for name, lst in acc.items():
                r = res.setdefault(f'epi_async={e}', {}).setdefault(name, [])
                r.extend(lst)
    h.set_option('tile_trace', 0)
    h.set_option('epi_async', 1)
    summary = {}
    for arm, d in res.items():
        summary[arm] = {}
        for name, lst in sorted(d.items()):
            summary[arm][name] = {'launches': len(lst),
                                  'phases_us': {k: float(np.median([p[k] for p, _ in lst])) for k in lst[0][0]},
                                  'tiles': lst[0][1]['tiles'], 'rounds': lst[0][1]['rounds'],
                                  'span_us': float(np.median([m['span_us'] for _, m in lst]))}
    return {'pairs': pairs, 'arms': summary, 'sm_mhz_samples': clocks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--pairs', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_gemm_tiles.py measures on the GPU'
    from argparse import Namespace
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.synth import make_seeded_state_dict
    info = device_info()
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=8, shared=False)
    cfg = Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34', feat_idx=[0, 1, 2, 3],
                    weights_dict=make_seeded_state_dict(0, nc_init='consensus'), change_stride=True,
                    regressor_config=rc)
    net = Patch2PixB200(cfg)
    line = {'metric': 'gemm tile decomposition'}
    line['k_sweep'] = k_sweep(net._handle, args.reps, info)
    line['workload'] = workload(net, args.pairs, info)
    line.update({k: v for k, v in info.items() if not k.startswith('_')})
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
