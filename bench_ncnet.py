"""Times NCNet's NeighConsensus stack on the tensor cores (nc_stack.cu) against a PyTorch Conv4d (fp32 cuDNN conv3d loop)
on the same GPU, and the whole ImMatchNet.forward_feat, at the volumes a user runs:
1024x768 images -> 64x48 ResNet101 layer3 features -> relocalisation 2 -> a 32x24x32x24 volume, and the same features
at relocalisation 0 (a 64x48x64x48 volume).

    python bench_ncnet.py [--reps N] [--skip-reloc0]

Prints one JSON line per case: ms per call (CUDA events, after warm-up), algorithmic TFLOP/s (2 * MACs of the true
Conv4d layers, both nets in symmetric mode, over the measured time), the largest output difference between the two
arms relative to max |output|, and the card's name and power limit."""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

from patch2pix_b200.ncnet import ImMatchNet, NeighConsensus


def conv4d_cudnn(x, w, b):
    """x [Cin, hA, wA, hB, wB]; w [k, Cout, Cin, k, k, k] -> [Cout, ...]: one conv3d per (output A row, first-axis tap)."""
    k = w.shape[0]
    p = k // 2
    hA = x.shape[1]
    xp = F.pad(x, (0, 0, 0, 0, 0, 0, p, p))                # zero rows along the first A axis
    out = []
    for i in range(hA):
        acc = None
        for t in range(k):
            y = F.conv3d(xp[:, i + t].unsqueeze(0), w[t], bias=b if t == 0 else None, padding=p)
            acc = y if acc is None else acc + y
        out.append(acc[0])
    return torch.stack(out, 1)


def stack_cudnn(x, ws, bs):
    def run(v):
        v = v.unsqueeze(0)
        for w, b in zip(ws, bs):
            v = torch.relu(conv4d_cudnn(v, w, b))
        return v[0]
    return run(x) + run(x.permute(2, 3, 0, 1)).permute(2, 3, 0, 1)


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


def weights(ks, ch, seed):
    g = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for i, (k, c) in enumerate(zip(ks, ch)):
        cin = 1 if i == 0 else ch[i - 1]
        ws.append((torch.rand(k, c, cin, k, k, k, generator=g) - 0.35) / (cin * k ** 4) ** 0.5)
        bs.append(0.05 * torch.randn(c, generator=g))
    return ws, bs


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception:
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--skip-reloc0', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ncnet.py needs a CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda:0')
    gpu = card()
    g = torch.Generator().manual_seed(0)
    fa = torch.rand(1, 1024, 64, 48, generator=g).to(dev)
    fb = torch.rand(1, 1024, 64, 48, generator=g).to(dev)
    for ks, ch in (([3, 3, 3], [16, 16, 1]), ([5, 5, 5], [16, 16, 1])):
        ws, bs = weights(ks, ch, sum(ks))
        for reloc in (2, 0):
            if reloc == 0 and args.skip_reloc0:
                continue
            net = ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=reloc)
            sd = net.state_dict()
            for i, (w, b) in enumerate(zip(ws, bs)):
                sd[f'NeighConsensus.conv.{2 * i}.weight'], sd[f'NeighConsensus.conv.{2 * i}.bias'] = w, b
            net.load_state_dict(sd)
            s = max(reloc, 1)
            hA, wA = 64 // s, 48 // s
            x = (torch.rand(1, 1, hA, wA, hA, wA, generator=g) ** 4).to(dev)
            nc = net.NeighConsensus
            reps = args.reps if reloc == 2 else max(1, args.reps // 2)
            t_nc = timed(lambda: nc(x), reps)
            t_ff = timed(lambda: net.forward_feat(fa, fb), reps)
            wd, bd = [w.to(dev) for w in ws], [b.to(dev) for b in bs]
            with torch.no_grad():
                t_ref = timed(lambda: stack_cudnn(x[0, 0], wd, bd), max(1, reps // 2))
                ref = stack_cudnn(x[0, 0], wd, bd)
                out = nc(x)[0, 0]
            V = (hA * wA) ** 2
            macs = sum(V * k ** 4 * c * (1 if i == 0 else ch[i - 1]) for i, (k, c) in enumerate(zip(ks, ch))) * 2
            print(json.dumps({
                'stack': f'{ks}/{ch}', 'volume': [hA, wA, hA, wA], 'relocalization': reloc,
                'nc_stack_ms': round(t_nc, 3), 'cudnn_conv4d_ms': round(t_ref, 3), 'forward_feat_ms': round(t_ff, 3),
                'nc_stack_tflops': round(2 * macs / t_nc / 1e9, 2), 'cudnn_conv4d_tflops': round(2 * macs / t_ref / 1e9, 2),
                'max_rel_diff': (out - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30), 'gpu': gpu}),
                flush=True)
            del net, nc, x, ref, out
            torch.cuda.empty_cache()
    # cost per layer: stacks of 1, 2 and 3 layers at the relocalisation-2 volume.  Layer 1 (1 input channel) and the
    # 1-channel last layer run the same padded 16-channel MMAs as a 16 -> 16 layer.
    for k in (3, 5):
        x = (torch.rand(1, 1, 32, 24, 32, 24, generator=g) ** 4).to(dev)
        t = {}
        for ks, ch in (([k], [1]), ([k, k], [16, 1]), ([k, k, k], [16, 16, 1])):
            ws, bs = weights(ks, ch, k)
            nc = NeighConsensus(kernel_sizes=ks, channels=ch)
            nc.load_state_dict({f'conv.{2 * i}.{n}': v for i, (w, b) in enumerate(zip(ws, bs))
                                for n, v in (('weight', w), ('bias', b))})
            t[len(ks)] = timed(lambda: nc(x), args.reps)
        print(json.dumps({'per_layer': f'k={k}', 'volume': [32, 24, 32, 24], 'stack_1_layer_ms': round(t[1], 3),
                          'stack_2_layers_ms': round(t[2], 3), 'stack_3_layers_ms': round(t[3], 3),
                          'added_16to16_layer_ms': round(t[3] - t[2], 3), 'gpu': gpu}), flush=True)


if __name__ == '__main__':
    main()
