"""Generate tests/golden/ncnet_topk_golden.npz by running the LIVE reference's ImMatchNet.forward_feat and
corr_to_matches_topk (networks/ncn/) on the CPU.

Run where the reference is checked out (it does not travel with the repository):
    python tests/golden/make_ncnet_topk_golden.py [/path/to/reference]
The reference is imported unmodified; the only shim makes torchvision's resnet101(pretrained=True) build without
downloading weights (forward_feat never runs the backbone).  use_cuda=False everywhere.
"""
import importlib.util
import os
import sys
import warnings

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
from networks.ncn.extract_ncmatches import corr_to_matches_topk             # noqa: E402

from patch2pix_b200 import synth                                            # noqa: E402

_spec = importlib.util.spec_from_file_location('ncnet_topk_cases', os.path.join(HERE, 'ncnet_topk_cases.py'))
K = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(K)


def np_(t):
    return t.detach().cpu().numpy()


def main():
    out = {}
    torch.set_grad_enabled(False)
    pairs = [synth.ncnet_features(s, K.FEAT_C, *K.FEAT_SIZES) for s in K.FEAT_SEEDS]
    ks, ch, wseed = K.STACK
    ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
    for reloc in K.RELOCS:
        net = ncm.ImMatchNet(use_cuda=False, ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=reloc)
        for i, (w, b) in enumerate(zip(ws, bs)):
            net.NeighConsensus.conv[2 * i].weight.data.copy_(w)
            net.NeighConsensus.conv[2 * i].bias.data.copy_(b)
        # one forward_feat per pair, stacked: the reference's NCNet maxpool4d mixes the items of a batch
        rs = [net.forward_feat(fa, fb) for fa, fb in pairs]
        if reloc > 1:
            corr = torch.cat([r[0] for r in rs])
            delta = tuple(torch.cat([r[1][c] for r in rs]) for c in range(4))
        else:
            corr, delta = torch.cat(rs), None
        out[f'r{reloc}_corr'] = np_(corr)
        if delta is not None:
            for n, d in zip('ijkl', delta):
                out[f'r{reloc}_d{n}'] = np_(d)
        _, _, hA, wA, hB, wB = corr.shape
        for key, inv, sm, k, fmt in K.cases(reloc):
            kk = (hB * wB if inv else hA * wA) if k == 'all' else k
            d = None
            if fmt is not None:
                d = tuple(t.clone() for t in delta) if fmt == 'mixed' else tuple(t.long() for t in delta)
            res = corr_to_matches_topk(corr, delta4d=d, topk=kk, ksize=max(reloc, 1), do_softmax=sm,
                                       invert_matching_direction=inv)
            for n, t in zip(('jA', 'iA', 'jB', 'iB', 'score'), res):
                out[f'{key}_{n}'] = np_(t)
            out[f'{key}_dtypes'] = np.array([str(t.dtype) for t in res])
    path = os.path.join(HERE, 'ncnet_topk_golden.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, len(out), 'arrays')


if __name__ == '__main__':
    main()
