"""The refiner workflow at any image size, without a GPU: the CPU oracle against fixtures of the live reference
(tests/golden/make_refiner_golden.py), the loader's size and grey arithmetic against Pillow itself, and the inputs the
refiner refuses (files that are not RGB, images below 8 x 8)."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from patch2pix_b200.model import refine_level_shapes
from patch2pix_b200.preprocess import load_im_tensor, tensor_size
from patch2pix_b200.synth import synthetic_pair_sized, synthetic_photo_pair

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
REFINE = ['refiner_refine_97x133_120x161', 'refiner_refine_9x203_64x15', 'refiner_refine_682x1024_768x1023']
LOAD_CASES = [((45, 61), None), ((130, 97), 64), ((61, 90), 50), ((37, 203), 100)]    # as make_refiner_golden.py


@pytest.mark.parametrize('name', REFINE)
def test_oracle_refine_matches_odd_sizes(name, seeded_sd):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    im1, im2 = synthetic_pair_sized(int(g['pair_idx']), tuple(g['size1']), tuple(g['size2']))
    cm = torch.from_numpy(g['coarse_in'])
    with torch.no_grad():
        r, s, c = O.refine_matches(im1, im2, cm.clone(), seeded_sd, 0.0)
        ri, si, ci = O.refine_matches(im1, im2, cm.long(), seeded_sd, 0.0)
    # the oracle reproduces the reference on every row whose trunc(mid) is not an fp32 coin flip
    keep = ~g['mid_tie']
    np.testing.assert_allclose(r[keep], g['refined'][keep], atol=1e-3, rtol=0)
    np.testing.assert_allclose(s, g['scores'], atol=1e-4, rtol=0)
    assert np.array_equal(c, g['coarse'])
    np.testing.assert_allclose(ri, g['refined_i'], atol=1e-3, rtol=0)
    np.testing.assert_allclose(si, g['scores_i'], atol=1e-4, rtol=0)
    assert np.array_equal(ci, g['coarse_i'])
    # io_thres 0.5: the reference's filter over its own scores
    pos = np.where(g['scores'] > 0.5)[0]
    sel = pos if len(pos) else np.arange(len(g['scores']))
    assert np.array_equal(g['coarse_t'], g['coarse'][sel]) and np.array_equal(g['scores_t'], g['scores'][sel])


def test_refine_level_shapes():
    sd = None
    for H, W in ((97, 133), (9, 203), (64, 15), (682, 1024), (768, 1023), (8, 8), (96, 128)):
        im = torch.zeros(1, 3, H, W)
        if sd is None:
            from patch2pix_b200.synth import make_seeded_state_dict
            sd = make_seeded_state_dict(0, regressors=False)
        with torch.no_grad():
            feats = O.backbone_forward_all(im, sd)
        assert [tuple(f.shape[1:]) for f in feats[:4]] == refine_level_shapes(H, W), (H, W)
    assert refine_level_shapes(96, 128) == [(3, 96, 128), (64, 48, 64), (64, 24, 32), (128, 12, 16)]
    for H, W in ((7, 100), (100, 7), (0, 0)):
        with pytest.raises(RuntimeError):
            refine_level_shapes(H, W)


def test_grey_arithmetic_is_pillows():
    """The loader's grey image is (19595 R + 38470 G + 7471 B + 0x8000) >> 16, as Pillow's convert('L'), on all 2^24
    colours."""
    from PIL import Image
    a = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    pil = np.asarray(Image.fromarray(rgb).convert('L')).reshape(-1)
    r, g, b = (rgb.reshape(-1, 3)[:, i].astype(np.int64) for i in range(3))
    assert np.array_equal(pil, (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16)


def test_tensor_size_is_the_references_rule():
    """Downscale only above imsize, int(round()) with Python's round (half to even), else the image's own size."""
    assert tensor_size(1536, 1023, 1024) == (1024, 682)
    assert tensor_size(1023, 1536, 1024) == (682, 1024)
    assert tensor_size(8, 5, 4) == (4, 2)            # 5 * 0.5 = 2.5 rounds to 2
    assert tensor_size(8, 7, 4) == (4, 4)            # 3.5 rounds to 4
    assert tensor_size(100, 50, None) == (100, 50) and tensor_size(100, 50, 0) == (100, 50)
    assert tensor_size(100, 50, 100) == (100, 50) and tensor_size(100, 50, 400) == (100, 50)
    g = np.load(os.path.join(GOLD, 'refiner_load_im_tensor.npz'))
    for k, ((h, w), imsize) in enumerate(LOAD_CASES):
        wt, ht = tensor_size(w, h, imsize)
        assert g[f'im{k}'].shape == (1, 3, ht, wt) and g[f'gray{k}'].shape == (1, 1, ht, wt), k
        assert tuple(g[f'scale{k}']) == (w / wt, h / ht), k


def test_load_im_tensor_fixture_is_pillow_arithmetic(tmp_path):
    """The fixtures' grey image is Pillow's resize + convert('L') / 255, the RGB tensor Pillow's resize through
    to_tensor / normalize: the arithmetic the GPU loader restates."""
    from PIL import Image
    g = np.load(os.path.join(GOLD, 'refiner_load_im_tensor.npz'))
    mean = np.array([0.485, 0.456, 0.406], np.float32).reshape(3, 1, 1)
    std = np.array([0.229, 0.224, 0.225], np.float32).reshape(3, 1, 1)
    for k, (size, imsize) in enumerate(LOAD_CASES):
        img, _ = synthetic_photo_pair(10 + k, size, size)
        im = Image.fromarray(img)
        wt, ht = tensor_size(im.width, im.height, imsize)
        if (wt, ht) != (im.width, im.height):
            im = im.resize((wt, ht), Image.BICUBIC)
        grey = np.asarray(im.convert('L')).astype(np.float32) / np.float32(255)
        assert np.array_equal(g[f'gray{k}'][0, 0], grey), k
        x = np.asarray(im).astype(np.float32).transpose(2, 0, 1) / np.float32(255)
        assert np.array_equal(g[f'im{k}'][0], (x - mean) / std), k


@pytest.mark.parametrize('mode', ['L', 'RGBA', 'P', 'CMYK'])
def test_load_im_tensor_refuses_non_rgb(tmp_path, mode):
    from PIL import Image
    img, _ = synthetic_photo_pair(1, (20, 24), (20, 24))
    path = str(tmp_path / ('im.png' if mode != 'CMYK' else 'im.jpg'))
    Image.fromarray(img).convert(mode).save(path)
    with pytest.raises(RuntimeError, match='RGB'):
        load_im_tensor(path, 'cuda:0')
