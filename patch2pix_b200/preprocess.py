"""GPU image preprocessing behind the reference's loader names (utils/datasets/preprocess.py:32-91).

`load_im_flexible` in the reference = PIL decode -> cal_rescale_size -> bicubic resize -> ToTensor -> Normalize, all on
the host.  Here only the (file-format) decode stays on the host; resize + tensor conversion + normalisation run in
libp2p_b200 (`p2p_preprocess_image`, bit-exact restatement of Pillow's 8-bit resampling) and the result is born on the
device, so `estimate_matches` never ships a float image over PCIe (3 bytes per pixel instead of 12).
"""
import numpy as np
import torch

from . import _lib


def cal_rescale_size(image_size, w, h, k_size=2, scale_factor=1 / 16, no_print=True):
    """utils/datasets/preprocess.py:83-91 (verbatim arithmetic)."""
    wt = int(np.floor(w / (max(w, h) / image_size) * scale_factor / k_size) / scale_factor * k_size)
    ht = int(np.floor(h / (max(w, h) / image_size) * scale_factor / k_size) / scale_factor * k_size)
    if not no_print:
        n = wt * ht * scale_factor * scale_factor / (k_size ** 2)
        print(f'Target size {image_size} Original: (w={w},h={h}), Rescaled: (w={wt},h={ht}) , matches resolution: {n}')
    return wt, ht


def preprocess_image(rgb, k_size=2, upsample=16, imsize=None, device='cuda:0', handle=None, return_resized=False):
    """The tensor half of load_im_flexible (preprocess.py:41-60) for a decoded RGB uint8 image [H,W,3]
    (numpy array, CPU or CUDA tensor) -> (img [3,ht,wt] float32 on `device`, scale (wo/wt, ho/ht))."""
    if isinstance(rgb, np.ndarray):
        rgb = torch.from_numpy(np.array(rgb, copy=True, order='C'))     # own, writable copy (PIL arrays are read-only)
    if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3:
        raise RuntimeError('preprocess_image expects an RGB uint8 image [H,W,3]')
    device = torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError('preprocess_image runs on a CUDA device (no CPU fallback)')
    ho, wo = int(rgb.shape[0]), int(rgb.shape[1])
    if not (imsize and imsize > 0):
        imsize = max(wo, ho)
    elif imsize > max(wo, ho):          # disable up-sampling (preprocess.py:43-44)
        imsize = max(wo, ho)
    wt, ht = cal_rescale_size(imsize, wo, ho, k_size, 1.0 / upsample)
    if wt <= 0 or ht <= 0:
        raise RuntimeError(f'image {wo}x{ho} is too small for k_size {k_size}, upsample {upsample}')
    h = handle or _lib.default_handle(device)
    with torch.cuda.device(device):
        src = rgb if rgb.is_cuda else (rgb if rgb.is_pinned() else rgb.pin_memory()).to(device, non_blocking=True)
        src = src.contiguous()
        out = torch.empty(3, ht, wt, dtype=torch.float32, device=device)
        res = torch.empty(ht, wt, 3, dtype=torch.uint8, device=device) if return_resized else None
        _lib.check(h.lib.p2p_preprocess_image(h.h, _lib.ptr(src), ho, wo, ht, wt, _lib.ptr(out), _lib.ptr(res), h.stream()))
    scale = (wo / wt, ho / ht)
    return (out, scale, res) if return_resized else (out, scale)


def load_im_flexible(im_path, k_size=2, upsample=16, imsize=None, crop_square=False, device='cuda:0', handle=None):
    """utils/datasets/preprocess.py:32-60 with everything after the file decode on the GPU."""
    from PIL import Image                        # host I/O only: file-format decoding
    img = np.asarray(Image.open(im_path).convert('RGB'))
    out, scale = preprocess_image(img, k_size, upsample, imsize, device, handle)
    if crop_square:                              # "mainly for beauty plotting" (preprocess.py:55-57)
        _, hh, ww = out.shape
        out = out[:, :ww, :]
    return out, scale


def tensor_size(wo, ho, imsize=None):
    """load_im_tensor's target size (utils/datasets/preprocess.py:11-16): downscale only when max(wo, ho) > imsize > 0,
    to int(round(ho * s)) x int(round(wo * s)) with s = imsize / max(wo, ho) (Python's round); otherwise the image keeps
    its own size.  -> (wt, ht)"""
    if imsize and imsize > 0 and max(wo, ho) > imsize:
        s = imsize / max(wo, ho)
        return int(round(wo * s)), int(round(ho * s))
    return wo, ho


def load_im_tensor(im_path, device, imsize=None, with_gray=True, handle=None):
    """utils/datasets/preprocess.py:7-30, the refiner's loader, with everything after the file decode on the GPU:
    the Pillow-exact bicubic downscale, ToTensor + Normalize and the grey image (Pillow's convert('L') / 255) come out
    of one launch chain.  -> (im [1,3,ht,wt], grey [1,1,ht,wt], (wo / wt, ho / ht)) on `device`, or (im, scale)
    without `with_gray`.  Only RGB files are read (the reference's Normalize fails on any other mode)."""
    from PIL import Image                        # host I/O only: file-format decoding
    with Image.open(im_path) as im:
        if im.mode != 'RGB':
            raise RuntimeError(f'load_im_tensor reads RGB images only; {im_path} is {im.mode}')
        rgb = np.asarray(im)
    device = torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError('load_im_tensor runs on a CUDA device (no CPU fallback)')
    ho, wo = int(rgb.shape[0]), int(rgb.shape[1])
    wt, ht = tensor_size(wo, ho, imsize)
    if wt <= 0 or ht <= 0:
        raise RuntimeError(f'imsize {imsize} shrinks the {wo}x{ho} image {im_path} to nothing')
    h = handle or _lib.default_handle(device)
    with torch.cuda.device(device):
        src = torch.from_numpy(np.array(rgb, copy=True, order='C')).pin_memory().to(device, non_blocking=True)
        out = torch.empty(1, 3, ht, wt, dtype=torch.float32, device=device)
        gray = torch.empty(1, 1, ht, wt, dtype=torch.float32, device=device) if with_gray else None
        _lib.check(h.lib.p2p_preprocess_image_gray(h.h, _lib.ptr(src), ho, wo, ht, wt, _lib.ptr(out), _lib.ptr(gray),
                                                   h.stream()))
    scale = (wo / wt, ho / ht)
    return (out, gray, scale) if with_gray else (out, scale)
