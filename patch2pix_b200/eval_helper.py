"""Mirror of the reference's matcher glue (utils/eval/model_helper.py:28-109), device-resident.

`estimate_matches` starts from normalised image tensors [1,3,H,W] plus the (sx, sy) scale factors of the loader and
reproduces the reference exactly -- `predict_coarse` / `predict_fine`, the `io_thres` inlier filter with its "keep
everything if nothing passes" rule, the rescaling to original-image pixels in float64 -- but filter and rescaling run
in one kernel and the result crosses PCIe in ONE copy.  `estimate_matches_from_files` adds the loader: only the
file-format decode stays on the host, resize / ToTensor / Normalize run on the GPU (patch2pix_b200.preprocess).
"""
from argparse import Namespace
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .model import Patch2PixB200

MAX_THRESHOLDS = 16       # kMaxHomThresholds / kMaxRelposeThresholds of the statistics kernels


def load_model(state_dict, regressor_config=None, device='cuda:0', method='patch2pix'):
    """utils/eval/model_helper.py:28-62 without the checkpoint file I/O: `state_dict` is the loaded
    `ckpt['state_dict']`; `regressor_config` the checkpoint's Namespace (panc is forced to 1 as in :46)."""
    config = Namespace(training=False, device=torch.device(device), regr_batch=1200, backbone='ResNet34',
                       feat_idx=None, weights_dict=state_dict, regressor_config=None, change_stride=True)
    if 'patch2pix' in method:
        if regressor_config is None:
            regressor_config = Namespace(conv_dims=[512, 512], conv_kers=[3, 3], conv_strs=[2, 1], fc_dims=[512, 256],
                                         feat_comb='pre', psize=[16, 16], pshift=8, panc=1, shared=False)
        config.feat_idx = [0, 1, 2, 3]
        config.regressor_config = regressor_config
        config.regressor_config.panc = 1
    return Patch2PixB200(config)


def load_checkpoint(ckpt_path, device='cuda:0', method='patch2pix', lprint=print):
    """utils/eval/model_helper.py:28-62 + utils/common/setup_helper.py:25-30 including the file I/O.

    Released checkpoints are pickled dicts {'backbone', 'feat_idx', 'state_dict', 'regressor_config': Namespace,
    ['last_epoch']}; torch >= 2.6 refuses the Namespace under `weights_only=True`, so the file is read with
    `weights_only=False` (SURVEY.md s8c shim 3) onto the CPU -- `pack_weights` does the one upload. An 'nc'
    checkpoint may be a bare state_dict (:54-57). Only the released architecture is accepted."""
    ckpt = torch.load(ckpt_path, map_location='cpu', weights_only=False)
    lprint('\nLoad model method:{} '.format(method))
    if 'patch2pix' in method:
        if ckpt.get('backbone', 'ResNet34') != 'ResNet34' or list(ckpt.get('feat_idx', [0, 1, 2, 3])) != [0, 1, 2, 3]:
            raise RuntimeError('only the released ResNet34 / feat_idx [0,1,2,3] configuration is supported, got '
                               f"{ckpt.get('backbone')} / {ckpt.get('feat_idx')}")
        if 'last_epoch' in ckpt:
            lprint(f"Ckpt:{ckpt_path} epochs:{ckpt['last_epoch'] + 1}")
        else:
            lprint(f'Ckpt:{ckpt_path}')
        return load_model(ckpt['state_dict'], ckpt.get('regressor_config'), device=device, method=method)
    if 'nc' in method:
        sd = ckpt['state_dict'] if isinstance(ckpt, dict) and 'state_dict' in ckpt else ckpt
        lprint('Load pretrained weights: {}'.format(ckpt_path))
        return load_model(sd, None, device=device, method=method)
    raise ValueError('Wrong method name.')


def _finalize_device(net, fine, scores, coarse, io_thres, upscale, verify=None):
    """The device half of _finalize, enqueued without a host sync -> (packed, n, kind): packed holds the n rows of
    p2p_finalize_matches (9 float64 each), the kept-row count at [n * 9] and, with `verify`, the RANSAC or pose buffer
    from [n * 9 + 1] on; kind is verify[0] or None."""
    import ctypes as C
    from . import _lib
    h = net._handle
    n = int(scores.shape[0])
    dev = scores.device
    extra = 0
    if verify is not None:
        from . import pose as P
        from . import verify as V
        kind = verify[0] if isinstance(verify, (tuple, list)) and len(verify) > 0 else None
        if not (kind in ('F', 'H', 'DEGENSAC') and len(verify) == 2 or kind == 'E' and len(verify) == 4):
            raise ValueError("verify must be None, ('F', px_th), ('H', px_th), ('DEGENSAC', px_th) or "
                             "('E', px_th, K1, K2)")
        px_th = verify[1]
        extra = P.out_size(n) if kind == 'E' else V.out_size(n)
    packed = torch.empty(n * 9 + 1 + extra, dtype=torch.float64, device=dev)
    up = (C.c_double * 4)(*[float(v) for v in upscale])
    fine_c = fine.reshape(-1, 4).contiguous() if fine is not None else None
    scores_c = scores.reshape(-1).contiguous()
    coarse_c = coarse.contiguous()
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_finalize_matches(h.h, _lib.ptr(fine_c), _lib.ptr(scores_c), _lib.ptr(coarse_c), n, float(io_thres),
                                              up, _lib.ptr(packed), h.stream()))
    n_dev = C.c_void_p(packed.data_ptr() + n * 9 * 8)
    if verify is not None and kind == 'E':   # E RANSAC + pose on the kept, rescaled rows, in place (cv2's defaults)
        out = packed[n * 9 + 1:]
        intr = P.reference_intrinsics(verify[2], verify[3])
        P.find_essential_into(h, packed, 9, n, n_dev, intr, px_th, 0.999, 1000, 0, out)
        P.recover_pose_into(h, packed, 9, n, n_dev, intr, out.data_ptr(), out.data_ptr() + 184, out)
    elif verify is not None:      # RANSAC on the kept, rescaled rows (refined columns 0..3), in place, count read on the device
        model = {'F': V.MODEL_F, 'H': V.MODEL_H, 'DEGENSAC': V.MODEL_F_DEGENSAC}[kind]
        V.find_model_into(h, model, packed, 9, n, n_dev, px_th, 0.999, 10000, 0, packed[n * 9 + 1:])
    return packed, n, (kind if verify is not None else None)


def _finalize(net, fine, scores, coarse, io_thres, upscale, verify=None):
    """One launch (+ the RANSAC launches with `verify`) and ONE device->host copy for the tail of estimate_matches
    (model_helper.py:97-109)."""
    return _finalize_host(*_finalize_device(net, fine, scores, coarse, io_thres, upscale, verify))


def _finalize_host(packed, n, kind):
    host = packed.cpu().numpy()                      # the single synchronising copy
    m = int(host[n * 9])
    rows = host[:n * 9].reshape(n, 9)[:m]
    out = (rows[:, 0:4].copy(), rows[:, 4].astype(np.float32), rows[:, 5:9].copy())
    if kind is None:
        return out
    from . import pose as P
    from . import verify as V
    if kind == 'E':
        E, mask, _, R, t, _ = P.parse_host(host[n * 9 + 1:], n)
        return out + (mask[:m], E, R, t)
    model, mask = V.parse_host(host[n * 9 + 1:], n)
    return out + (mask[:m], model)


def estimate_matches(net, im1, im2, scale1=(1.0, 1.0), scale2=(1.0, 1.0), ksize=2, ncn_thres=0.0, mutual=True,
                     io_thres=0.25, eval_type='fine', verify=None):
    """utils/eval/model_helper.py:64-109 on image tensors -> (matches, scores, coarse_matches) numpy arrays
    (float64 matches in original-image pixels, float32 scores), with the inlier filter and the rescaling on the device
    and a single device->host copy (the reference does three `.cpu()` round trips).

    verify=('F', px_th) or ('H', px_th) also runs RANSAC (patch2pix_b200.verify, conf 0.999, 10000 iterations, seed 0)
    on the device on those matches, px_th in original-image pixels, still before the single copy, and returns
    (matches, scores, coarse_matches, inliers, model): a bool mask over the matches and the 3x3 float64 F or H
    (None when no model was found).  verify=('DEGENSAC', px_th) runs F RANSAC with the DEGENSAC plane-degeneracy
    check instead (the notebook's pydegensac.findFundamentalMatrix) and returns what ('F', px_th) returns.

    verify=('E', px_th, K1, K2), with K1, K2 the 3x3 intrinsics in original-image pixels, runs the reference's
    matches2relapose_cv instead (patch2pix_b200.pose: E RANSAC at conf 0.999 and 1000 iterations, then pose recovery on
    its inliers) and returns (matches, scores, coarse_matches, inliers, E, R, t): the E-RANSAC mask, E (None when no
    model was found), R and t [3, 1] (x2 = R x1 + t)."""
    res = _finalize_host(*match_device(net, im1, im2, scale1, scale2, ksize, ncn_thres, mutual, io_thres, eval_type,
                                       verify))
    if eval_type == 'coarse':
        return (res[0], res[1], res[0]) + res[3:]
    return res


def match_device(net, im1, im2, scale1=(1.0, 1.0), scale2=(1.0, 1.0), ksize=2, ncn_thres=0.0, mutual=True,
                 io_thres=0.25, eval_type='fine', verify=None):
    """estimate_matches up to, not including, its device->host copy -> (packed, n, kind) as _finalize_device.  The
    coarse matcher's rows repeat the coarse columns in the refined slots."""
    upscale = tuple(scale1) + tuple(scale2)
    im1 = im1.to(net.device)
    im2 = im2.to(net.device)
    with torch.no_grad():
        if eval_type == 'coarse':
            coarse_matches, scores = net.predict_coarse(im1, im2, ksize=ksize, ncn_thres=ncn_thres, mutual=mutual)
            return _finalize_device(net, None, scores[0], coarse_matches[0], float('-inf'), upscale, verify)
        if eval_type != 'fine':
            raise ValueError("eval_type must be 'coarse' or 'fine'")
        fine_matches, fine_scores, coarse_matches = net.predict_fine(im1, im2, ksize=ksize, ncn_thres=ncn_thres,
                                                                    mutual=mutual)
    return _finalize_device(net, fine_matches[0], fine_scores[0], coarse_matches[0], io_thres, upscale, verify)


def estimate_matches_from_files(net, im1_path, im2_path, ksize=2, ncn_thres=0.0, mutual=True, io_thres=0.25,
                                eval_type='fine', imsize=None, verify=None):
    """utils/eval/model_helper.py:64-72 + the above: image files in, numpy matches out.  Only the file decode runs on
    the host; resize / ToTensor / Normalize are GPU kernels (patch2pix_b200.preprocess)."""
    from .preprocess import load_im_flexible
    im1, sc1 = load_im_flexible(im1_path, ksize, net.upsample, imsize=imsize, device=net.device, handle=net._handle)
    im2, sc2 = load_im_flexible(im2_path, ksize, net.upsample, imsize=imsize, device=net.device, handle=net._handle)
    return estimate_matches(net, im1.unsqueeze(0), im2.unsqueeze(0), sc1, sc2, ksize, ncn_thres, mutual, io_thres, eval_type,
                            verify)


# ---- the evaluation protocols' pair runner -------------------------------------------------------------------------
def check_thresholds(values, what='thresholds'):
    """A threshold list as float64: 1..MAX_THRESHOLDS finite, positive, strictly increasing values, else ValueError."""
    t = np.asarray([float(v) for v in values], dtype=np.float64)
    if not (1 <= t.size <= MAX_THRESHOLDS and np.all(np.isfinite(t)) and np.all(t > 0) and np.all(np.diff(t) > 0)):
        raise ValueError(f'{what} must be 1..{MAX_THRESHOLDS} finite, positive, strictly increasing values, got '
                         f'{list(values)}')
    return t


def as_rows(out, dev):
    """Matches as a matcher returns them (numpy or a tensor, or a tuple whose first element is those) -> contiguous
    [N, 4] float64 rows on `dev`; ValueError on any other shape."""
    if isinstance(out, tuple):
        out = out[0]
    if isinstance(out, torch.Tensor):
        rows = out.detach().to(device=dev, dtype=torch.float64)
    else:
        rows = torch.from_numpy(np.ascontiguousarray(out, dtype=np.float64)).to(dev)
    if rows.numel() == 0:
        rows = rows.reshape(0, 4)
    if rows.dim() != 2 or rows.shape[1] != 4:
        raise ValueError(f'matches must be [N, 4] rows (x0, y0, x1, y1), got shape {tuple(rows.shape)}')
    return rows.contiguous()


def prefetch(items, load):
    """Yields (i, load(items[i]), or the exception it raised) for the items in order; `load` runs on one worker thread,
    one item ahead of the item being yielded."""
    items = list(items)
    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(load, items[0]) if items else None
        for i in range(len(items)):
            cur = nxt
            nxt = pool.submit(load, items[i + 1]) if i + 1 < len(items) else None
            try:
                got = cur.result()
            except Exception as e:
                got = e
            yield i, got


class PairRunner:
    """Runs a matcher on image pairs for the evaluation protocols: a Patch2PixB200 (put in eval mode) as
    estimate_matches_from_files(..., ksize, ncn_thres, True, io_thres, eval_type, imsize) runs it, or any callable
    (path0, path1) -> [N, 4] rows.  `dev` and `h` are the device and handle the protocol's own launches use."""

    def __init__(self, matcher, ksize=2, eval_type='fine', io_thres=0.25, ncn_thres=0.0, imsize=1024):
        from . import _lib
        self.matcher = matcher
        self.is_net = isinstance(matcher, Patch2PixB200)
        self.ksize, self.eval_type, self.io_thres, self.ncn_thres, self.imsize = (ksize, eval_type, io_thres,
                                                                                  ncn_thres, imsize)
        if self.is_net:
            matcher.eval()
            self.dev, self.h = matcher.device, matcher._handle
        else:
            self.dev = torch.device('cuda', torch.cuda.current_device())
            self.h = _lib.default_handle(self.dev)

    def decode(self, paths):
        """The image files as pinned RGB uint8 tensors [H, W, 3] for the net; None for a callable, which reads its
        own files."""
        if not self.is_net:
            return None
        from PIL import Image
        return [torch.from_numpy(np.array(Image.open(p).convert('RGB'))).pin_memory() for p in paths]

    def prepare(self, rgb):
        """A decoded image -> (x [1, 3, H, W] on the device, scale), the input of match."""
        from .preprocess import preprocess_image
        x, scale = preprocess_image(rgb, self.ksize, self.matcher.upsample, self.imsize, self.dev, self.h)
        return x.unsqueeze(0), scale

    def match(self, a, b, verify=None):
        """match_device on two prepared images -> (packed, n), without a host sync."""
        packed, n, _ = match_device(self.matcher, a[0], b[0], a[1], b[1], self.ksize, self.ncn_thres, True,
                                    self.io_thres, self.eval_type, verify)
        return packed, n

    def call(self, path0, path1):
        """The callable on two image files -> [N, 4] float64 rows on the device."""
        return as_rows(self.matcher(path0, path1), self.dev)


def refine_matches(im1_path, im2_path, net, coarse_matcher, io_thres=0.0, imsize=None, coarse_only=False):
    """utils/eval/model_helper.py:111-127: Patch2Pix as the refiner of another matcher's coarse matches.  Both images
    are loaded with load_im_tensor (any size; only the file decode runs on the host), `coarse_matcher(grey1, grey2)`
    gets the [1,1,H,W] grey device tensors and returns [N,4] (x1, y1, x2, y2) rows in those images' pixels (numpy or
    torch, int64 / float32 / float64), and net.refine_matches refines them.  -> (refined, scores, coarse): float64
    matches in original-image pixels and float32 scores, filtered by `scores > io_thres` when io_thres > 0 (keeping
    every row if none passes); coarse_only -> (coarse, None, None)."""
    from .preprocess import load_im_tensor
    im1, grey1, sc1 = load_im_tensor(im1_path, net.device, imsize, with_gray=True, handle=net._handle)
    im2, grey2, sc2 = load_im_tensor(im2_path, net.device, imsize, with_gray=True, handle=net._handle)
    upscale = np.array([sc1 + sc2])
    coarse_matches = coarse_matcher(grey1, grey2)
    if coarse_only:
        cm = coarse_matches.cpu().numpy() if isinstance(coarse_matches, torch.Tensor) else np.asarray(coarse_matches)
        return upscale * cm, None, None
    with torch.no_grad():
        refined, scores, coarse = net.refine_matches(im1, im2, coarse_matches, io_thres)
    return upscale * refined, scores, upscale * coarse
