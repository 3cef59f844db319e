"""Benchmark of the refiner workflow (Patch2Pix refining another matcher's coarse matches, utils/eval/model_helper.py
refine_matches): image files in, refined matches out.

  refine_files   eval_helper.refine_matches on two 1536 x 1023 PNGs at imsize 1024, i.e. 1024 x 682 tensors, a size
                 that is not a multiple of 8, with N coarse rows from a stand-in matcher;
  refine_files8  the same on 1536 x 1020 PNGs (1024 x 680 tensors, a multiple of 8), to show what the odd size costs;
  load_gpu       load_im_tensor of one file (decode on the host, resize / normalise / grey on the GPU);
  load_host      the reference's loader on the host: Pillow resize and convert('L'), to_tensor / normalize arithmetic
                 in torch on the CPU, then the upload.

    python bench_refiner.py [--steps K] [--warmup W] [--rows 1000 3200]
Prints one JSON line per measurement, with the GPU's name and power limit.  Everything written goes to a temporary
directory.
"""
import argparse
import json
import subprocess
import tempfile
import time
from argparse import Namespace

import numpy as np
import torch


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(','))
    except Exception:                 # nvidia-smi missing: the name from torch, the limit unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return {'gpu': name, 'power_limit': power}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return {'ms_median': float(np.median(t)), 'ms_min': float(np.min(t)), 'ms_max': float(np.max(t)), 'steps': steps}


def host_loader(path, device, imsize):
    """utils/datasets/preprocess.py:7-30 on the host, then the upload."""
    from PIL import Image
    from patch2pix_b200.preprocess import tensor_size
    im = Image.open(path)
    wo, ho = im.width, im.height
    wt, ht = tensor_size(wo, ho, imsize)
    if (wt, ht) != (wo, ho):
        im = im.resize((wt, ht), Image.BICUBIC)
    gray = torch.from_numpy(np.array(im.convert('L'))).float().div(255)[None, None].to(device)
    x = torch.from_numpy(np.array(im)).permute(2, 0, 1).float().div(255)
    x = (x - torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)) / torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)
    return x[None].to(device), gray, (wo / wt, ho / ht)


def random_matcher(n, seed=0):
    """Stand-in coarse matcher: n float32 rows spread over both grey images, on their device."""
    def matcher(g1, g2):
        gen = torch.Generator().manual_seed(seed)
        dims = torch.tensor([g1.shape[-1], g1.shape[-2], g2.shape[-1], g2.shape[-2]], dtype=torch.float32)
        return (torch.rand(n, 4, generator=gen) * dims).to(g1.device)
    return matcher


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rows', type=int, nargs='+', default=[1000, 3200])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_refiner.py measures on a CUDA device; none is present')
    from PIL import Image
    from patch2pix_b200.eval_helper import refine_matches
    from patch2pix_b200.model import Patch2PixB200
    from patch2pix_b200.preprocess import load_im_tensor
    from patch2pix_b200.synth import make_seeded_state_dict, synthetic_photo_pair
    rc = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256], feat_comb='pre',
                   psize=[16, 16], pshift=8, panc=1, shared=False)
    net = Patch2PixB200(Namespace(training=False, device='cuda:0', regr_batch=1200, backbone='ResNet34',
                                  feat_idx=[0, 1, 2, 3], weights_dict=make_seeded_state_dict(0), change_stride=True,
                                  regressor_config=rc))
    info = gpu_info()
    dev = torch.device('cuda:0')
    with tempfile.TemporaryDirectory() as tmp:
        files = {}
        for tag, h in (('refine_files', 1023), ('refine_files8', 1020)):
            a, b = synthetic_photo_pair(0, (h, 1536), (h, 1536))
            files[tag] = (f'{tmp}/{tag}_a.png', f'{tmp}/{tag}_b.png')
            Image.fromarray(a).save(files[tag][0])
            Image.fromarray(b).save(files[tag][1])
        for n in args.rows:
            for tag in ('refine_files', 'refine_files8'):
                p1, p2 = files[tag]
                m = random_matcher(n)
                r = timed(lambda: refine_matches(p1, p2, net, m, io_thres=0.0, imsize=1024), args.steps, args.warmup)
                size = tuple(load_im_tensor(p1, dev, 1024)[0].shape[-2:])
                print(json.dumps({'bench': tag, 'rows': n, 'tensor_hw': size, **r, **info}), flush=True)
        p1 = files['refine_files'][0]
        r = timed(lambda: load_im_tensor(p1, dev, 1024, handle=net._handle), args.steps, args.warmup)
        print(json.dumps({'bench': 'load_gpu', 'file_hw': (1023, 1536), 'imsize': 1024, **r, **info}), flush=True)
        r = timed(lambda: host_loader(p1, dev, 1024), args.steps, args.warmup)
        print(json.dumps({'bench': 'load_host', 'file_hw': (1023, 1536), 'imsize': 1024, **r, **info}), flush=True)


if __name__ == '__main__':
    main()
