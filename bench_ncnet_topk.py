"""Times corr_to_matches_topk on the GPU (topk.cu, one launch per call) against a PyTorch arm on the same GPU written
the way the reference computes it (softmax of the whole volume, torch.topk, index gathers, a per-batch loop for the
relocalisation offsets), on the volumes a user gets from ImMatchNet.forward_feat: 1024x768 images -> 64x48 ResNet101
layer3 features -> a 32x24x32x24 volume at relocalisation 2 (with deltas) or 64x48x64x48 at relocalisation 0.
Batches of 1 and 4 pairs, topk 1, 8 and 64, both directions.

    python bench_ncnet_topk.py [--reps N] [--skip-reloc0]

Prints one JSON line per workload: ms per call of each arm (CUDA events, after warm-up; the kernel arm includes the
packing of the delta tuple, as every call does), the bytes of the volume read per call over the kernel arm's time and
as a share of the H100 SXM's 3.35 TB/s, the share of ranks outside ties (value equal to a neighbouring rank's in the
PyTorch arm) where both arms pick the same cell, the largest score difference, and the card's name and power limit."""
import argparse
import json
import subprocess

import torch

from patch2pix_b200 import synth
from patch2pix_b200.ncnet import ImMatchNet, corr_to_matches_topk

HBM_BYTES_PER_S = 3.35e12


def torch_topk(corr, delta4d, topk, ksize, do_softmax, invert):
    """The reference's algorithm in PyTorch, with topk + 1 ranks kept to mark ties."""
    b, _, hA, wA, hB, wB = corr.shape
    nA, nB = hA * wA, hB * wB
    dim = 2 if invert else 1
    v = corr.view(b, nA, nB)
    if do_softmax:
        v = torch.softmax(v, dim)
    n_slice = nB if invert else nA
    vals, idx = torch.topk(v, min(topk + 1, n_slice), dim=dim, largest=True, sorted=True)
    if invert:
        a, bc = torch.arange(nA, device=corr.device).view(1, nA, 1).expand_as(idx), idx
    else:
        a, bc = idx, torch.arange(nB, device=corr.device).view(1, 1, nB).expand_as(idx)
    # tie mark per rank: equal to the value of the rank above or below
    eq = vals[..., :-1] == vals[..., 1:] if invert else vals[:, :-1] == vals[:, 1:]
    tie = torch.zeros_like(vals, dtype=torch.bool)
    if invert:
        tie[..., :-1] |= eq
        tie[..., 1:] |= eq
        sel = (slice(None), slice(None), slice(0, topk))
    else:
        tie[:, :-1] |= eq
        tie[:, 1:] |= eq
        sel = (slice(None), slice(0, topk))
    a, bc, score, tie = [t[sel].reshape(b, -1) for t in (a, bc, vals, tie)]
    iA, jA, iB, jB = a // wA, a % wA, bc // wB, bc % wB
    if delta4d is not None:
        for i in range(b):
            flat = a[i] * nB + bc[i]
            d = [t[i, 0].reshape(-1)[flat].long() for t in delta4d]
            iA[i], jA[i], iB[i], jB[i] = iA[i] * ksize + d[0], jA[i] * ksize + d[1], iB[i] * ksize + d[2], \
                jB[i] * ksize + d[3]
    return (jA, iA, jB, iB, score), tie


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def volumes(reloc, b, dev):
    ks, ch = [3, 3, 3], [10, 10, 1]
    net = ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=reloc)
    sd = net.state_dict()
    ws, bs = synth.ncnet_stack_weights(7, ks, ch)
    for i, (w, bb) in enumerate(zip(ws, bs)):
        sd[f'NeighConsensus.conv.{2 * i}.weight'], sd[f'NeighConsensus.conv.{2 * i}.bias'] = w, bb
    net.load_state_dict(sd)
    pairs = [synth.ncnet_features(100 + i, 1024, (64, 48), (64, 48)) for i in range(b)]
    fa = torch.cat([p[0] for p in pairs]).to(dev)
    fb = torch.cat([p[1] for p in pairs]).to(dev)
    r = net.forward_feat(fa, fb)
    del net
    return r if reloc > 1 else (r, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--skip-reloc0', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ncnet_topk.py needs a CUDA device')
    dev = torch.device('cuda:0')
    gpu = card()
    for reloc in (2, 0):
        if reloc == 0 and args.skip_reloc0:
            continue
        ks = max(reloc, 1)
        for b in (1, 4):
            corr, delta = volumes(reloc, b, dev)
            nbytes = corr.numel() * 4
            for inv in (False, True):
                for k in (1, 8, 64):
                    ours = lambda: corr_to_matches_topk(corr, delta, topk=k, ksize=ks, invert_matching_direction=inv)
                    ref = lambda: torch_topk(corr, delta, k, ks, True, inv)
                    t_ours, t_ref = timed(ours, args.reps), timed(ref, args.reps)
                    got, (want, tie) = ours(), ref()
                    same = torch.stack([g == w for g, w in zip(got[:4], want[:4])]).all(0)
                    clear = ~tie
                    print(json.dumps({
                        'volume': list(corr.shape[2:]), 'relocalization': reloc, 'batch': b, 'topk': k,
                        'direction': 'inverted' if inv else 'forward',
                        'kernel_ms': round(t_ours, 4), 'torch_ms': round(t_ref, 4),
                        'speedup': round(t_ref / t_ours, 2),
                        'volume_bytes': nbytes, 'kernel_GBps': round(nbytes / t_ours / 1e6, 1),
                        'kernel_share_of_3.35TBps': round(nbytes / (t_ours * 1e-3) / HBM_BYTES_PER_S, 3),
                        'index_agreement_outside_ties': round(same[clear].double().mean().item(), 6),
                        'ranks_outside_ties': round(clear.double().mean().item(), 4),
                        'max_score_diff': (got[4] - want[4]).abs().max().item(), 'gpu': gpu}), flush=True)
            del corr, delta
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
