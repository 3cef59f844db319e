"""Golden vectors for image pairs of DIFFERENT sizes, written by the LIVE reference on CPU.

Run in the authoring container only (the reference does not travel to the GPU box):
    python tests/golden/make_unequal_golden.py
Writes tests/golden/unequal_*.npz.  The reference, its import-time shims and the helpers come from make_golden.py.
Every image pair is synthetic_pair_sized (two overlapping views of one texture at their own sizes) with the
'consensus' NC weights; pair indices are picked so that the reference's own candidate list has as few fp32-tie rows
(and pooling windows as few fp32 ties) as possible; the fixtures record where they are.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import (L2Normalize, MutualMatching, build_ref, filter_coarse, maxpool4d, np_,  # noqa: E402
                         reference_tie_rows)

from patch2pix_b200.synth import make_seeded_state_dict, synthetic_pair_sized  # noqa: E402


def delta_tie_cells(net, feat1, feat2, k=2, tie_eps=1e-6):
    """Pooled cells whose k^4 window holds a top-2 gap <= tie_eps in the reference's own correlation: their
    relocalisation delta is an fp32 coin flip in any implementation."""
    corr = net.combine(L2Normalize(feat1, dim=1), L2Normalize(feat2, dim=1))
    sl = torch.cat([corr[:, :, i::k, j::k, a::k, b::k] for i in range(k) for j in range(k) for a in range(k) for b in range(k)], 1)
    top2 = sl.topk(2, dim=1)[0]
    return (top2[:, 0] - top2[:, 1]) <= tie_eps


def _tie_rows(net, im1, im2):
    with torch.no_grad():
        corr4d, delta4d, f1, f2 = net.forward(im1, im2, ksize=2, return_feats=True)
        return int(reference_tie_rows(net, corr4d, f1[-1], f2[-1], 2).sum()) + int(delta_tie_cells(net, f1[-1], f2[-1]).sum())


def _pick_pair(net, size1, size2, first, tries=20):
    """Pair index in [first, first + tries) whose candidate list holds the fewest fp32-tie rows of the reference
    (the first one with none).  Larger pairs hold a few such rows whatever the index; the fixtures record them."""
    best = None
    for idx in range(first, first + tries):
        n = _tie_rows(net, *synthetic_pair_sized(idx, size1, size2))
        if n == 0:
            return idx
        if best is None or n < best[0]:
            best = (n, idx)
    return best[1]


def case_stages(net, name, size1, size2, first):
    """predict_fine with the coarse-stage intermediates (as make_golden.case_stages, on an unequal pair)."""
    pair_idx = _pick_pair(net, size1, size2, first)
    im1, im2 = synthetic_pair_sized(pair_idx, size1, size2)
    out = {'pair_idx': pair_idx, 'size1': np.array(size1), 'size2': np.array(size2), 'ksize': 2}
    with torch.no_grad():
        f1s, f2s = [], []
        net.extract.forward_all(im1, f1s, early_feat=True)
        net.extract.forward_all(im2, f2s, early_feat=True)
        corr = net.combine(L2Normalize(f1s[-1], dim=1), L2Normalize(f2s[-1], dim=1))
        pooled, mi, mj, mk, ml = maxpool4d(corr, k_size=2)
        out['pooled'] = np_(pooled)
        out['delta'] = np.stack([np_(mi), np_(mj), np_(mk), np_(ml)]).astype(np.int8)
        out['delta_fp32_tie'] = np_(delta_tie_cells(net, f1s[-1], f2s[-1]))
        out['ncn'] = np_(net.ncn(MutualMatching(pooled)))
        corr4d, delta4d = net.forward_coarse_match(f1s[-1], f2s[-1], ksize=2)
        out['corr4d'] = np_(corr4d)
        cm, sc = net.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net.upsample, center=True)
        out['cand_matches'] = np_(cm)
        out['cand_scores'] = np_(sc)
        fine, fine_p, mid, mid_p, coarse = net.predict_fine(im1, im2, ksize=2, return_all=True)
        out['fine'] = np_(fine[0]).reshape(-1, 4)
        out['fine_p'] = np_(fine_p[0]).reshape(-1)
        out['mid'] = np_(mid[0]).reshape(-1, 4)
        out['mid_p'] = np_(mid_p[0]).reshape(-1)
        out['coarse'] = np_(coarse[0])
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, 'pair', pair_idx, 'coarse', out['coarse'].shape)


def case_train_sequence(net8, name, size1, size2, ptmax, np_seed, first):
    """train_patch2pix.py:97-118 forward sequence under eval()/no_grad (ptmax, panc=8) on an unequal pair."""
    pair_idx = _pick_pair(net8, size1, size2, first, tries=8)
    im1, im2 = synthetic_pair_sized(pair_idx, size1, size2)
    out = {'pair_idx': pair_idx, 'size1': np.array(size1), 'size2': np.array(size2), 'ptmax': ptmax, 'np_seed': np_seed}
    with torch.no_grad():
        corr4d, delta4d, feats1, feats2 = net8.forward(im1, im2, ksize=2, return_feats=True)
        cm, sc = net8.cal_coarse_matches(corr4d, delta4d, ksize=2, upsample=net8.upsample, center=True)
        out['cand_matches'] = np_(cm)
        out['cand_scores'] = np_(sc)
        out['cand_fp32_tie'] = np_(reference_tie_rows(net8, corr4d, feats1[-1], feats2[-1], 2))
        np.random.seed(np_seed)
        cm, sc = filter_coarse(cm, sc, 0.0, True, ptmax=ptmax)
        cm = net8.shift_to_anchors(cm)
        out['anchors'] = np_(cm[0])
        mid, mid_p = net8.forward_fine_match(feats1, feats2, cm, psize=16, ptype='center', regressor=net8.regress_mid)
        fine, fine_p = net8.forward_fine_match(feats1, feats2, mid, psize=16, ptype='center', regressor=net8.regress_fine)
        out['mid'] = np_(mid[0])
        out['mid_p'] = np_(mid_p[0])
        out['fine'] = np_(fine[0])
        out['fine_p'] = np_(fine_p[0])
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, 'pair', pair_idx, 'anchors', out['anchors'].shape)


if __name__ == '__main__':
    torch.manual_seed(0)
    sdc = make_seeded_state_dict(0, nc_init='consensus')
    netc1 = build_ref(dict(sdc), panc=1)
    netc8 = build_ref(dict(sdc), panc=8)
    case_stages(netc1, 'unequal_96x128_128x96', (96, 128), (128, 96), 1)             # transposed aspect
    case_stages(netc1, 'unequal_128x160_96x224', (128, 160), (96, 224), 21)          # H1 > H2 while W1 < W2
    case_train_sequence(netc8, 'unequal_trainseq_160x240_192x128', (160, 240), (192, 128), 40, 777, 41)
