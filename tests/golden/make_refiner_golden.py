"""Golden vectors of the refiner workflow at image sizes that are not multiples of 8, from the LIVE reference on CPU.

Run in the authoring container only (the reference does not travel to the GPU box):
    python tests/golden/make_refiner_golden.py
Writes tests/golden/refiner_*.npz with the import-time shims of make_golden.py:
  refiner_refine_<H1>x<W1>_<H2>x<W2>  Patch2Pix.refine_matches on synthetic_pair_sized images, float32 coarse rows
                                      (borders, out of range, inside one image only) at io_thres 0 / 0.5, their int64
                                      truncation at io_thres 0, and the reference's mid rows of both with its fp32 tie rows
                                      (a mid coordinate within 2e-4 px of an integer: its trunc() is a coin flip);
  refiner_load_im_tensor              load_im_tensor of synthetic_photo_pair PNGs, with and without a downscale;
  refiner_files                       utils/eval/model_helper.refine_matches from PNG files with grid_coarse_matcher.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import build_ref, np_  # noqa: E402  (sets up the reference's import path and shims)

# shim 3: utils/datasets/__init__.py imports the training datasets (and transforms3d through them); the loaders in
# utils/datasets/preprocess.py need none of that, so the package is registered without running its __init__
import types  # noqa: E402
import utils  # noqa: E402
_ds = types.ModuleType('utils.datasets')
_ds.__path__ = [os.path.join(list(utils.__path__)[0], 'datasets')]
sys.modules['utils.datasets'] = _ds

from utils.datasets.preprocess import load_im_tensor          # noqa: E402
from utils.eval.model_helper import refine_matches as ref_refine_matches   # noqa: E402
from patch2pix_b200.synth import grid_coarse_matcher, make_seeded_state_dict, synthetic_pair_sized, synthetic_photo_pair  # noqa: E402,E501

# every residue of H and W mod 8 appears at least once, plus one photo-sized pair
REFINE_CASES = [((97, 133), (120, 161), 60), ((9, 203), (64, 15), 40), ((682, 1024), (768, 1023), 80)]
LOAD_CASES = [((45, 61), None), ((130, 97), 64), ((61, 90), 50), ((37, 203), 100)]
FILE_CASES = [((150, 203), (161, 190), None), ((150, 203), (161, 190), 128)]
TIE = 2e-4


def refine_rows(size1, size2, n, seed=77):
    """float32 coarse rows: random over [-5 %, 105 %] of each image plus border / out-of-range / one-image rows."""
    (h1, w1), (h2, w2) = size1, size2
    g = torch.Generator().manual_seed(seed)
    dims = torch.tensor([w1, h1, w2, h2], dtype=torch.float32)
    cm = torch.rand(n, 4, generator=g) * dims * 1.1 - 0.05 * dims
    cm[0] = torch.tensor([0.0, 0.0, w2 - 1.0, h2 - 1.0])
    cm[1] = torch.tensor([w1 - 1.0, h1 - 1.0, 0.0, 0.0])
    cm[2] = torch.tensor([float(w1), float(h1), float(w2), float(h2)])
    cm[3] = torch.tensor([w1 + 3.0, -2.5, 7.999, 8.0])
    cm[4] = torch.tensor([w1 / 2, h1 / 2, w2 + 20.0, h2 + 5.0])
    cm[5] = torch.tensor([-30.0, h1 + 9.0, w2 / 2, h2 / 2])
    cm[6] = torch.tensor([w1 - 0.5, h1 - 8.5, w2 - 7.5, h2 - 0.25])
    return cm


def case_refine(net, pair_idx, size1, size2, n):
    im1, im2 = synthetic_pair_sized(pair_idx, size1, size2)
    cm = refine_rows(size1, size2, n)
    out = {'pair_idx': pair_idx, 'size1': np.array(size1), 'size2': np.array(size2), 'coarse_in': np_(cm)}
    with torch.no_grad():
        f1s, f2s = [], []
        net.extract.forward_all(im1, f1s, early_feat=True)
        net.extract.forward_all(im2, f2s, early_feat=True)
        for tag, rows in (('', cm), ('_i', cm.long())):
            mid, _ = net.forward_fine_match(f1s, f2s, rows.unsqueeze(0), psize=16, ptype='center',
                                            regressor=net.regress_mid)
            out['mid' + tag] = np_(mid[0]).reshape(-1, 4)
            out['mid_tie' + tag] = (np.abs(out['mid' + tag] - np.round(out['mid' + tag])) < TIE).any(1)
        for tag, rows, thr in (('', cm, 0.0), ('_t', cm, 0.5), ('_i', cm.long(), 0.0)):
            r, s, c = net.refine_matches(im1, im2, rows.clone(), io_thres=thr)
            out['refined' + tag], out['scores' + tag], out['coarse' + tag] = r, s, c
    name = f'refiner_refine_{size1[0]}x{size1[1]}_{size2[0]}x{size2[1]}'
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, out['refined'].shape, out['refined_t'].shape, 'mid ties', int(out['mid_tie'].sum()))


def case_load_im_tensor(tmp):
    from PIL import Image
    out = {}
    for k, (size, imsize) in enumerate(LOAD_CASES):
        img, _ = synthetic_photo_pair(10 + k, size, size)
        path = os.path.join(tmp, f'load{k}.png')
        Image.fromarray(img).save(path)
        im, gray, scale = load_im_tensor(path, 'cpu', imsize, with_gray=True)
        out[f'im{k}'], out[f'gray{k}'], out[f'scale{k}'] = np_(im), np_(gray), np.array(scale)
        print('load', k, size, imsize, tuple(im.shape), scale)
    np.savez_compressed(os.path.join(HERE, 'refiner_load_im_tensor.npz'), **out)


def case_files(net, tmp):
    from PIL import Image
    out = {}
    for k, (size1, size2, imsize) in enumerate(FILE_CASES):
        a, b = synthetic_photo_pair(20 + k, size1, size2)
        p1, p2 = os.path.join(tmp, f'f{k}a.png'), os.path.join(tmp, f'f{k}b.png')
        Image.fromarray(a).save(p1)
        Image.fromarray(b).save(p2)
        matcher = grid_coarse_matcher()
        with torch.no_grad():
            for tag, thr in (('', 0.0), ('_t', 0.5)):
                r, s, c = ref_refine_matches(p1, p2, net, matcher, io_thres=thr, imsize=imsize)
                out[f'refined{k}{tag}'], out[f'scores{k}{tag}'], out[f'coarse{k}{tag}'] = r, s, c
            out[f'coarse_only{k}'] = ref_refine_matches(p1, p2, net, matcher, imsize=imsize, coarse_only=True)[0]
            im1, g1, _ = load_im_tensor(p1, 'cpu', imsize)
            im2, g2, _ = load_im_tensor(p2, 'cpu', imsize)
            f1s, f2s = [], []
            net.extract.forward_all(im1, f1s, early_feat=True)
            net.extract.forward_all(im2, f2s, early_feat=True)
            mid, _ = net.forward_fine_match(f1s, f2s, matcher(g1, g2).unsqueeze(0), psize=16, ptype='center',
                                            regressor=net.regress_mid)
        m = np_(mid[0]).reshape(-1, 4)
        out[f'mid_tie{k}'] = (np.abs(m - np.round(m)) < TIE).any(1)
        print('files', k, size1, size2, imsize, out[f'refined{k}'].shape, out[f'refined{k}_t'].shape,
              'mid ties', int(out[f'mid_tie{k}'].sum()))
    np.savez_compressed(os.path.join(HERE, 'refiner_files.npz'), **out)


if __name__ == '__main__':
    torch.manual_seed(0)
    sd = make_seeded_state_dict(0)
    net = build_ref(dict(sd), panc=1)
    with tempfile.TemporaryDirectory() as tmp:
        case_load_im_tensor(tmp)
        case_files(net, tmp)
    for i, (s1, s2, n) in enumerate(REFINE_CASES):
        case_refine(net, 30 + i, s1, s2, n)
