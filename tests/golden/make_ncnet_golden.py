"""Generate tests/golden/ncnet_golden.npz by running the LIVE reference's ImMatchNet, NeighConsensus and
corr_to_matches (networks/ncn/) on the CPU.

Run where the reference is checked out (it does not travel with the repository):
    python tests/golden/make_ncnet_golden.py [/path/to/reference]
The reference is imported unmodified; the only shim makes torchvision's resnet101(pretrained=True) build without
downloading weights (every weight is then overwritten from the seeded checkpoint).  use_cuda=False everywhere.
"""
import importlib.util
import os
import sys
import tempfile
import warnings
from argparse import Namespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
warnings.filterwarnings('ignore')

import torchvision.models as tvm                                            # noqa: E402
_rn101 = tvm.resnet101
tvm.resnet101 = lambda pretrained=False, **kw: _rn101(weights=None)         # shim: no download
import networks.ncn.model as ncm                                            # noqa: E402
from networks.ncn.extract_ncmatches import corr_to_matches                  # noqa: E402

from patch2pix_b200 import synth                                            # noqa: E402

_spec = importlib.util.spec_from_file_location('ncnet_cases', os.path.join(HERE, 'ncnet_cases.py'))
K = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(K)


def np_(t):
    return t.detach().cpu().numpy()


def nc_module(ks, ch, seed, sym):
    nc = ncm.NeighConsensus(use_cuda=False, kernel_sizes=ks, channels=ch, symmetric_mode=sym)
    ws, bs = synth.ncnet_stack_weights(seed, ks, ch)
    for i, (w, b) in enumerate(zip(ws, bs)):
        nc.conv[2 * i].weight.data.copy_(w)
        nc.conv[2 * i].bias.data.copy_(b)
    return nc


def main():
    out = {}
    torch.set_grad_enabled(False)
    # (a)
    for ks, ch, wseed in K.NC_STACKS:
        for sym in (True, False):
            nc = nc_module(ks, ch, wseed, sym)
            for shape, xseed in K.NC_VOLUMES:
                g = torch.Generator().manual_seed(xseed)
                x = torch.rand(1, 1, *shape, generator=g) - 0.1
                out[f'nc_{"_".join(map(str, ks))}_{"_".join(map(str, ch))}_{int(sym)}_{xseed}'] = np_(nc(x))[0, 0]
    # (b) + (d)
    ks, ch, wseed = K.FEAT_STACK
    fa, fb = synth.ncnet_features(K.FEAT_SEED, K.FEAT_C, *K.FEAT_SIZES)
    for reloc in K.RELOCS:
        net = ncm.ImMatchNet(use_cuda=False, ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=reloc)
        ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
        for i, (w, b) in enumerate(zip(ws, bs)):
            net.NeighConsensus.conv[2 * i].weight.data.copy_(w)
            net.NeighConsensus.conv[2 * i].bias.data.copy_(b)
        r = net.forward_feat(fa, fb)
        corr, delta = (r if reloc > 1 else (r, None))
        out[f'ff_r{reloc}_corr'] = np_(corr)
        if delta is not None:
            for n, d in zip('ijkl', delta):
                out[f'ff_r{reloc}_d{n}'] = np_(d)
                out[f'ff_r{reloc}_d{n}_dtype'] = np.array(str(d.dtype))
        for inv, scale, ri in K.C2M_ARGS:
            res = corr_to_matches(corr, delta4d=delta, ksize=max(reloc, 1), do_softmax=True, scale=scale,
                                  invert_matching_direction=inv, return_indices=ri)
            key = K.c2m_key(reloc, inv, scale, ri)
            for n, t in zip(('a0', 'a1', 'a2', 'a3', 'score'), res):
                out[f'{key}_{n}'] = np_(t)
            out[f'{key}_dtypes'] = np.array([str(t.dtype) for t in res])
    # (c)
    ks, ch = K.CKPT_STACK
    net = ncm.ImMatchNet(use_cuda=False, ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=2)
    names = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    sd = synth.ncnet_state_dict(K.CKPT_SEED, names, ks, ch)
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, 'ncnet.pth.tar')
        torch.save({'state_dict': sd, 'args': Namespace(ncons_kernel_sizes=ks, ncons_channels=ch)}, path)
        ncm_torch_load = torch.load
        torch.load = lambda *a, **kw: ncm_torch_load(*a, **{**kw, 'weights_only': False})
        try:
            net = ncm.ImMatchNet(use_cuda=False, checkpoint=path, relocalization_k_size=2)
        finally:
            torch.load = ncm_torch_load
    ia, ib = synth.ncnet_images(K.IMG_SEED, *K.IMG_SIZES)
    fa_ = net.FeatureExtraction(ia)
    fb_ = net.FeatureExtraction(ib)
    corr, delta = net({'source_image': ia, 'target_image': ib})
    out['fwd_corr'] = np_(corr)
    for n, d in zip('ijkl', delta):
        out[f'fwd_d{n}'] = np_(d)
    # maxpool boxes whose best correlation beats the runner-up clearly: there the deltas must agree exactly
    c4 = torch.einsum('chw,cij->hwij', fa_[0], fb_[0])
    h1, w1, h2, w2 = c4.shape
    v = c4.reshape(h1 // 2, 2, w1 // 2, 2, h2 // 2, 2, w2 // 2, 2).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(
        h1 // 2, w1 // 2, h2 // 2, w2 // 2, 16)
    top = v.topk(2, -1).values
    out['fwd_delta_clear'] = np_((top[..., 0] - top[..., 1]) > 1e-4 * top[..., 0].abs().clamp_min(1e-30))
    np.savez_compressed(os.path.join(HERE, 'ncnet_golden.npz'), **out)
    print('wrote', os.path.join(HERE, 'ncnet_golden.npz'), len(out), 'arrays')


if __name__ == '__main__':
    main()
