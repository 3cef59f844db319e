"""Seeded weights and synthetic image pairs (no network, no checkpoints).

The reference's pretrained checkpoint cannot be downloaded offline
(pretrained/download.sh), so parity and throughput are measured on seeded
random weights that carry the reference's ``state_dict`` key names and shapes
(SURVEY.md s8c; names probed from networks/patch2pix.py:13-61,
networks/modules.py:56-99, networks/ncn/conv4d.py:118-120,
networks/resnet.py:96-123).  BatchNorm running statistics / affines and all
biases are randomised (a default-initialised BN is the identity and would hide
folding bugs) and the running variances are calibrated so that activations
stay O(1) through the regressor, like a trained network's.
"""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

_LAYERS = (('layer1', 3, 64), ('layer2', 4, 128), ('layer3', 6, 256))


def _xavier(gen, *shape, fan_in=None, fan_out=None):
    rf = 1
    for s in shape[2:]:
        rf *= s
    fan_in = fan_in if fan_in is not None else shape[1] * rf
    fan_out = fan_out if fan_out is not None else shape[0] * rf
    bound = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(*shape, generator=gen) * 2 - 1) * bound


def _bn(sd, gen, name, c, var):
    sd[name + '.weight'] = 0.8 + 0.4 * torch.rand(c, generator=gen)
    sd[name + '.bias'] = 0.1 * torch.randn(c, generator=gen)
    sd[name + '.running_mean'] = 0.1 * math.sqrt(var) * torch.randn(c, generator=gen)
    sd[name + '.running_var'] = var * (0.7 + 0.6 * torch.rand(c, generator=gen))


def make_seeded_state_dict(seed=0, backbone=True, regressors=True, nc_init='uniform'):
    """Flat fp32 dict with the reference's state_dict names (layer4 / num_batches_tracked omitted).

    nc_init: 'uniform' -- NeighConsensus weights uniform in +-0.1 (an untrained net: its output is
    unrelated to the correlation, a pair yields 10-20 mutual matches and exact zeros / ties abound);
    'consensus' -- trained-like filters (positive on the 4D-diagonal taps, slightly negative elsewhere):
    coherent match neighbourhoods are reinforced, the rest is zeroed by the ReLUs, so a pair of overlapping
    views yields ~1000 distinct mutual matches at 640x480 with top-1/top-2 margins >~ 1e-5 (the benchmark workload).
    Every other tensor is identical between the two modes."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    if backbone:
        sd['extract.conv1.weight'] = _xavier(g, 64, 3, 7, 7)
        _bn(sd, g, 'extract.bn1', 64, 1.0)
        cin = 64
        for lname, nblk, c in _LAYERS:
            for i in range(nblk):
                p = f'extract.{lname}.{i}'
                sd[p + '.conv1.weight'] = _xavier(g, c, cin if i == 0 else c, 3, 3)
                _bn(sd, g, p + '.bn1', c, 1.0)
                sd[p + '.conv2.weight'] = _xavier(g, c, c, 3, 3)
                _bn(sd, g, p + '.bn2', c, 1.0)
                if i == 0 and cin != c:
                    sd[p + '.downsample.0.weight'] = _xavier(g, c, cin, 1, 1)
                    _bn(sd, g, p + '.downsample.1', c, 1.0)
            cin = c
    # NCNet: Conv4d weights are stored pre-permuted [k1, Cout, Cin, k2, k3, k4]
    sd['ncn.conv.0.weight'] = (torch.rand(3, 16, 1, 3, 3, 3, generator=g) * 2 - 1) * 0.1
    sd['ncn.conv.0.bias'] = 0.01 * torch.randn(16, generator=g)
    sd['ncn.conv.2.weight'] = (torch.rand(3, 1, 16, 3, 3, 3, generator=g) * 2 - 1) * 0.1
    sd['ncn.conv.2.bias'] = 0.01 * torch.randn(1, generator=g)
    if nc_init == 'consensus':
        # what a trained neighbourhood-consensus filter looks like: positive weights on the 9 "diagonal" taps, where the
        # A-offset equals the B-offset ((a+d, b+d) neighbours of a true match are matches too), slightly negative
        # elsewhere, so that incoherent / constant regions cancel and ReLU zeroes them (~97 % exact zeros at 640x480)
        gn = torch.Generator().manual_seed(12345 + seed)      # own stream: the tensors below stay as in 'uniform'

        def layer(cout, cin):                                   # layout [k1, Cout, Cin, k2, k3, k4] = taps (a, b, d, e)
            w = (torch.rand(3, cout, cin, 3, 3, 3, generator=gn) * 2 - 1) * 0.02 - 0.045
            for a in range(3):
                for b in range(3):
                    w[a, :, :, b, a, b] += 0.4 * (0.5 + torch.rand(cout, cin, generator=gn))
            return w
        sd['ncn.conv.0.weight'], sd['ncn.conv.2.weight'] = layer(16, 1), layer(1, 16)
    elif nc_init != 'uniform':
        raise ValueError("nc_init must be 'uniform' or 'consensus'")
    if regressors:
        for r in ('regress_mid', 'regress_fine'):
            sd[f'{r}.conv.0.weight'] = _xavier(g, 512, 518, 3, 3)
            _bn(sd, g, f'{r}.conv.1', 512, 0.0039)
            sd[f'{r}.conv.2.weight'] = _xavier(g, 512, 512, 3, 3)
            _bn(sd, g, f'{r}.conv.3', 512, 1.0)
            sd[f'{r}.fc.0.weight'] = _xavier(g, 512, 512)
            sd[f'{r}.fc.0.bias'] = 0.05 * torch.randn(512, generator=g)
            _bn(sd, g, f'{r}.fc.1', 512, 4.0)
            sd[f'{r}.fc.3.weight'] = _xavier(g, 256, 512)
            sd[f'{r}.fc.3.bias'] = 0.05 * torch.randn(256, generator=g)
            _bn(sd, g, f'{r}.fc.4', 256, 0.7)
            sd[f'{r}.fc.6.weight'] = _xavier(g, 5, 256)
            sd[f'{r}.fc.6.bias'] = 0.05 * torch.randn(5, generator=g)
    return sd


def synthetic_pair(pair_idx, height, width):
    """Deterministic 'two views of one texture' pair (SURVEY.md s8d): a low-frequency
    random texture plus noise, cropped twice with an (8,-8) px shift so that some true
    mutual matches exist.  Returns im1, im2 as [1,3,H,W] fp32 on CPU."""
    g = torch.Generator().manual_seed(1000 + int(pair_idx))
    low = torch.randn(1, 3, height // 8 + 4, width // 8 + 4, generator=g)
    base = F.interpolate(low, size=(height + 32, width + 32), mode='bicubic', align_corners=False)
    base = base + 0.3 * torch.randn(1, 3, height + 32, width + 32, generator=g)
    im1 = base[:, :, 16:16 + height, 16:16 + width].contiguous()
    im2 = base[:, :, 8:8 + height, 24:24 + width].contiguous()
    return im1, im2


def shifted_pair_offset(pair_idx):
    """(dx, dy) of synthetic_pair_shifted: multiples of 16 px, never (0, 0)."""
    g = torch.Generator().manual_seed(2000 + int(pair_idx))
    dx = 16 * int(torch.randint(-3, 4, (1,), generator=g))
    dy = 16 * int(torch.randint(-2, 3, (1,), generator=g))
    if dx == 0 and dy == 0:
        dx = 16
    return dx, dy


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _rotation(axis_angle):
    th = float(np.linalg.norm(axis_angle))
    if th == 0:
        return np.eye(3)
    K = _skew(axis_angle / th)
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


def synthetic_two_view(seed, n, outlier_ratio, noise_px, planar=False, width=640, height=480, focal2=None):
    """Seeded two-view scene for match verification: a random camera pair (focal 500 px, principal point at the
    image centre, camera 2 rotated up to ~0.15 rad and translated by ~1 unit at 4-8 units of depth), round(n * (1 -
    outlier_ratio)) true correspondences visible in both images with N(0, noise_px^2) noise on every coordinate, and
    uniformly random outlier pairs, shuffled.  With `planar` the 3-D points lie on one plane.
    `focal2` (default: 500) is the focal length of camera 2, in px.
    Returns dict(pts1 [n, 2], pts2 [n, 2] float64, F (x2^T F x1 = 0, unit norm), H (x2 ~ H x1 with H[2][2] = 1, or
    None unless planar), inlier [n] bool, K1, K2 (3x3 intrinsics), R, t (camera 2 from camera 1: X2 = R X1 + t))."""
    rng = np.random.default_rng(int(seed))
    Kc = np.array([[500.0, 0, width / 2], [0, 500.0, height / 2], [0, 0, 1]])
    K2 = Kc if focal2 is None else np.array([[float(focal2), 0, width / 2], [0, float(focal2), height / 2], [0, 0, 1]])
    R = _rotation(rng.uniform(-0.09, 0.09, 3))
    t = np.array([rng.uniform(0.6, 1.0) * rng.choice([-1, 1]), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    normal = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0])
    normal /= np.linalg.norm(normal)
    d = rng.uniform(5.0, 7.0)                                   # plane normal^T X = d (camera-1 frame)
    n_in = int(round(n * (1.0 - outlier_ratio)))
    p1, p2 = np.zeros((0, 2)), np.zeros((0, 2))
    while p1.shape[0] < n_in:
        m = 4 * n_in + 16
        uv = rng.uniform([0, 0], [width, height], (m, 2))
        ray = np.linalg.solve(Kc, np.concatenate([uv, np.ones((m, 1))], 1).T).T
        depth = d / (ray @ normal) if planar else rng.uniform(4.0, 8.0, m)
        X = ray * depth[:, None]
        X2 = X @ R.T + t
        q = X2 @ K2.T
        ok = (X[:, 2] > 0) & (X2[:, 2] > 0.5)
        q = q[ok, :2] / q[ok, 2:3]
        inside = (q[:, 0] >= 0) & (q[:, 0] < width) & (q[:, 1] >= 0) & (q[:, 1] < height)
        p1 = np.concatenate([p1, uv[ok][inside]])
        p2 = np.concatenate([p2, q[inside]])
    p1 = p1[:n_in] + rng.normal(0, noise_px, (n_in, 2))
    p2 = p2[:n_in] + rng.normal(0, noise_px, (n_in, 2))
    n_out = n - n_in
    o1 = rng.uniform([0, 0], [width, height], (n_out, 2))
    o2 = rng.uniform([0, 0], [width, height], (n_out, 2))
    perm = rng.permutation(n)
    pts1 = np.concatenate([p1, o1])[perm]
    pts2 = np.concatenate([p2, o2])[perm]
    inlier = np.concatenate([np.ones(n_in, bool), np.zeros(n_out, bool)])[perm]
    Ki = np.linalg.inv(Kc)
    K2i = Ki if focal2 is None else np.linalg.inv(K2)
    F = K2i.T @ _skew(t) @ R @ Ki
    F /= np.linalg.norm(F)
    H = None
    if planar:
        H = K2 @ (R + np.outer(t, normal) / d) @ Ki
        H /= H[2, 2]
    return dict(pts1=pts1, pts2=pts2, F=F, H=H, inlier=inlier, K1=Kc.copy(), K2=K2.copy(), R=R, t=t)


PLANE, OFF_PLANE, OUTLIER = 0, 1, 2


def synthetic_dominant_plane(seed, n, outlier_ratio, off_plane_ratio, noise_px, focal2=None, width=640, height=480):
    """Seeded two-view scene where most true correspondences lie on one plane, as on building facades and ground planes:
    round(n * (1 - outlier_ratio)) inliers, a fraction `off_plane_ratio` of them at general depth and the rest on the
    plane, plus uniformly random outlier pairs, shuffled.  Both inlier sets come from `synthetic_two_view(seed, ...)`
    (planar and not), which share one camera pair per seed, so F, R and t hold for every inlier and H for the plane.
    Returns the dict of synthetic_two_view (H of the plane) plus `label` [n] int8: PLANE, OFF_PLANE or OUTLIER."""
    n_in = int(round(n * (1.0 - outlier_ratio)))
    n_off = int(round(n_in * off_plane_ratio))
    pl = synthetic_two_view(seed, n_in - n_off, 0.0, noise_px, planar=True, width=width, height=height, focal2=focal2)
    gen = synthetic_two_view(seed, n_off, 0.0, noise_px, width=width, height=height, focal2=focal2)
    rng = np.random.default_rng([int(seed), 1])           # own stream for the outliers and the order
    n_out = n - n_in
    o1 = rng.uniform([0, 0], [width, height], (n_out, 2))
    o2 = rng.uniform([0, 0], [width, height], (n_out, 2))
    label = np.concatenate([np.full(n_in - n_off, PLANE), np.full(n_off, OFF_PLANE), np.full(n_out, OUTLIER)])
    perm = rng.permutation(n)
    label = label.astype(np.int8)[perm]
    return dict(pl, pts1=np.concatenate([pl['pts1'], gen['pts1'], o1])[perm],
                pts2=np.concatenate([pl['pts2'], gen['pts2'], o2])[perm], inlier=label != OUTLIER, label=label)


def synthetic_pair_shifted(pair_idx, height, width, noise=0.6):
    """Benchmark workload (round 2): two overlapping views of one texture whose offset is a multiple
    of 16 px (= one pooled correlation cell at ksize 2), so that coarse cells correspond one to one in
    the overlap, plus strong independent noise on the second view (std 0.6 against a unit-variance texture:
    with less noise the four true fine-level matches inside a 2^4 pooling window all have cosine
    1 - O(1e-6) and ~10 % of the reference's own relocalisation deltas are fp32 coin flips).  With the
    'consensus' NC weights this gives ~1000 distinct mutual matches at 640x480 (vs 13-17 for
    `synthetic_pair`), i.e. filter_coarse(ptmax=400) samples 400 DISTINCT proposals.
    Returns im1, im2 as [1,3,H,W] fp32 on CPU."""
    g = torch.Generator().manual_seed(2000 + int(pair_idx))
    dx = 16 * int(torch.randint(-3, 4, (1,), generator=g))
    dy = 16 * int(torch.randint(-2, 3, (1,), generator=g))
    if dx == 0 and dy == 0:
        dx = 16
    low = torch.randn(1, 3, height // 8 + 12, width // 8 + 12, generator=g)
    base = F.interpolate(low, size=(height + 96, width + 96), mode='bicubic', align_corners=False)
    base = base + 0.3 * torch.randn(1, 3, height + 96, width + 96, generator=g)
    im1 = base[:, :, 48:48 + height, 48:48 + width].contiguous()
    im2 = base[:, :, 48 + dy:48 + dy + height, 48 + dx:48 + dx + width].contiguous()
    im2 = im2 + noise * torch.randn(im2.shape, generator=g)
    return im1, im2


def synthetic_pair_sized(pair_idx, size1, size2, noise=0.6):
    """Two overlapping views of one texture at their own sizes size1 = (H1, W1) and size2 = (H2, W2), built like
    `synthetic_pair_shifted`: view 2's crop is offset from view 1's by a multiple of 16 px (shifted_pair_offset-style
    draw) and carries independent noise.  This is what a portrait photo matched against a landscape one looks like
    after load_im_flexible.  Returns im1 [1,3,H1,W1], im2 [1,3,H2,W2] fp32 on CPU."""
    (h1, w1), (h2, w2) = (int(s) for s in size1), (int(s) for s in size2)
    g = torch.Generator().manual_seed(3000 + int(pair_idx))
    dx = 16 * int(torch.randint(-3, 4, (1,), generator=g))
    dy = 16 * int(torch.randint(-2, 3, (1,), generator=g))
    if dx == 0 and dy == 0:
        dx = 16
    height, width = max(h1, h2), max(w1, w2)
    low = torch.randn(1, 3, height // 8 + 12, width // 8 + 12, generator=g)
    base = F.interpolate(low, size=(height + 96, width + 96), mode='bicubic', align_corners=False)
    base = base + 0.3 * torch.randn(1, 3, height + 96, width + 96, generator=g)
    im1 = base[:, :, 48:48 + h1, 48:48 + w1].contiguous()
    im2 = base[:, :, 48 + dy:48 + dy + h2, 48 + dx:48 + dx + w2].contiguous()
    im2 = im2 + noise * torch.randn(im2.shape, generator=g)
    return im1, im2


def write_colmap_model(model_dir, cameras, images):
    """COLMAP binary model (little-endian) with the given cameras [(id, model_id, width, height, params)] and images
    [(id, qvec (w, x, y, z), tvec, camera_id, name)] or [(..., name, point3D_ids)]: cameras.bin and images.bin in
    model_dir.  An image without point3D_ids has no 2D points; with them, 2D point k is (k, 0) with point3D_ids[k]."""
    import struct
    os.makedirs(model_dir, exist_ok=True)
    with open(os.path.join(model_dir, 'cameras.bin'), 'wb') as f:
        f.write(struct.pack('<Q', len(cameras)))
        for cid, model_id, w, h, params in cameras:
            f.write(struct.pack('<iiQQ', cid, model_id, w, h) + struct.pack(f'<{len(params)}d', *params))
    with open(os.path.join(model_dir, 'images.bin'), 'wb') as f:
        f.write(struct.pack('<Q', len(images)))
        for iid, q, t, cid, name, *ids in images:
            ids = np.asarray(ids[0] if ids else [], dtype='<i8').reshape(-1)
            pts = np.zeros(len(ids), dtype=[('xy', '<f8', (2,)), ('id', '<i8')])
            pts['xy'][:, 0] = np.arange(len(ids))
            pts['id'] = ids
            f.write(struct.pack('<i7di', iid, *q, *t, cid) + name.encode('utf-8') + b'\x00' +
                    struct.pack('<Q', len(ids)) + pts.tobytes())


def synthetic_overlap_images(seed, n_images, n2d=8000, frac=(0.2, 0.6), vary_n2d=False, identical=()):
    """Images [(id, qvec, tvec, camera_id, name, point3D_ids)] for write_colmap_model, for the overlap precompute:
    image i has n2d keypoints (uniform in 1 .. n2d with vary_n2d), each triangulated (a 3D point id > 0) with a
    probability drawn per image from U(frac), else -1 or 0.  Each pair (a, b) in `identical` gives image b image a's
    ids.  Names are a seeded permutation, so file order and name order differ."""
    rng = np.random.default_rng([int(seed), 11])
    perm = rng.permutation(n_images)
    ids = []
    for i in range(n_images):
        n = int(rng.integers(1, n2d + 1)) if vary_n2d else n2d
        p = rng.uniform(*frac)
        ids.append(np.where(rng.uniform(size=n) < p, rng.integers(1, 2 ** 40, n), rng.choice([-1, 0], n)))
    for a, b in identical:
        ids[b] = ids[a].copy()
    q = [1.0, 0.0, 0.0, 0.0]
    return [(i + 1, q, [0.0, 0.0, float(i)], 1, f'im_{perm[i]:05d}.jpg', ids[i]) for i in range(n_images)]


def synthetic_val_scene(root, scene, seed, sizes, ext='.png', missing=(), min_overlap=0.3):
    """One scene of a validation tree in the layout of the reference's PhotoTourism validation sets:
    root/scene/dense/images/<names>, dense/sparse/{cameras,images}.bin and dense/sparse/ov_pairs.npy
    ({min_overlap: pair names}).  Pair k is two views of one texture (synthetic_pair_shifted(seed * 1000 + k)) at
    sizes[k] = (width, height) as 8-bit images, or, with sizes[k] = ((w1, h1), (w2, h2)), two views of different sizes
    (synthetic_pair_sized(seed * 1000 + k)).  Each image has a seeded SIMPLE_PINHOLE camera of its own size and a
    seeded pose (the poses do not describe the textures: the matches are real, the pose errors are not meaningful).
    Pair indices in `missing` name a second image that is not written.  Returns the pair names."""
    from PIL import Image
    rng = np.random.default_rng([int(seed), 7])
    im_dir = os.path.join(root, scene, 'dense', 'images')
    os.makedirs(im_dir, exist_ok=True)
    cameras, images, pairs = [], [], []
    for k, size in enumerate(sizes):
        if isinstance(size[0], (tuple, list)):
            (w1, h1), (w2, h2) = size
            views = synthetic_pair_sized(int(seed) * 1000 + k, (h1, w1), (h2, w2))
        else:
            w, h = size
            views = synthetic_pair_shifted(int(seed) * 1000 + k, h, w)
        names = []
        for v, im in enumerate(views):
            h, w = im.shape[2], im.shape[3]
            name = f'{scene}_{k:03d}_{v}{ext}'
            if not (v == 1 and k in missing):
                rgb = (im[0].permute(1, 2, 0).numpy() * 48.0 + 128.0).clip(0, 255).astype(np.uint8)
                Image.fromarray(rgb).save(os.path.join(im_dir, name), **({'quality': 90} if ext == '.jpg' else {}))
            iid = len(images) + 1
            q = np.concatenate([[1.0], rng.uniform(-0.1, 0.1, 3)])
            cameras.append((iid, 0, w, h, [0.9 * max(w, h), w / 2.0, h / 2.0]))
            images.append((iid, q / np.linalg.norm(q), rng.normal(0.0, 1.0, 3), iid, name))
            names.append(name)
        pairs.append(tuple(names))
    model_dir = os.path.join(root, scene, 'dense', 'sparse')
    write_colmap_model(model_dir, cameras, images)
    np.save(os.path.join(model_dir, 'ov_pairs.npy'), {min_overlap: pairs})
    return pairs


def synthetic_photo_pair(seed, size1, size2, shift=(8, 16)):
    """Two 8-bit RGB views ([H,W,3] uint8 numpy) of one blocky texture at their own sizes size1 = (H1, W1) and
    size2 = (H2, W2), view 2 cropped shift = (dy, dx) px further into it.  Integer arithmetic only, so every machine
    writes the same pixels: the files the refiner's loader reads in tests and benchmarks."""
    rng = np.random.default_rng(4000 + int(seed))
    (h1, w1), (h2, w2) = (tuple(int(v) for v in s) for s in (size1, size2))
    dy, dx = shift
    H, W = max(h1, h2 + dy), max(w1, w2 + dx)
    low = rng.integers(0, 256, size=(H // 8 + 2, W // 8 + 2, 3), dtype=np.int32)
    base = np.repeat(np.repeat(low, 8, 0), 8, 1)[:H + 4, :W + 4]
    base = (base[:H, :W] + base[4:H + 4, :W] + base[:H, 4:W + 4] + base[4:H + 4, 4:W + 4]) // 4
    img = np.clip(base + rng.integers(-12, 13, size=base.shape), 0, 255).astype(np.uint8)
    return img[:h1, :w1].copy(), img[dy:dy + h2, dx:dx + w2].copy()


def grid_coarse_matcher(shift=(8, 16), step=12, dtype=torch.float32):
    """Deterministic stand-in for a third-party coarse matcher (SuperPoint, SuperGlue, ...) in the refiner workflow:
    called with the two grey images [1,1,H,W], it returns [N,4] (x1, y1, x2, y2) rows of `dtype` on their device, a
    grid in image 1 shifted by shift = (dy, dx) into image 2, plus rows on and past the borders of each image."""
    def matcher(grey1, grey2):
        h1, w1 = grey1.shape[-2:]
        h2, w2 = grey2.shape[-2:]
        ys, xs = torch.meshgrid(torch.arange(2, h1 + 8, step, dtype=torch.float64),
                                torch.arange(3, w1 + 8, step, dtype=torch.float64), indexing='ij')
        x1, y1 = xs.flatten() + 0.375, ys.flatten() + 0.625
        rows = torch.stack([x1, y1, x1 - shift[1], y1 - shift[0]], 1)
        edge = torch.tensor([[0.0, 0.0, w2 - 1.0, h2 - 1.0], [w1 - 1.0, h1 - 1.0, 0.0, 0.0], [w1, h1, w2, h2],
                             [w1 + 3.0, -2.5, 7.999, 8.0], [w1 / 2, h1 / 2, w2 + 20.0, h2 + 5.0],
                             [-30.0, h1 + 9.0, w2 / 2, h2 / 2]], dtype=torch.float64)
        return torch.cat([edge, rows]).to(dtype=dtype, device=grey1.device)
    return matcher


# ---- HPatches-layout sequences -----------------------------------------------------------------------------------------
def _hpatches_h(rng, split, w1, h1, w2, h2):
    """A mild random homography from a (w1, h1) image to a (w2, h2) one, about the image centres: near identity for
    'i' (illumination) sequences, rotation, scale, shear and perspective for 'v' (viewpoint) ones.  H[2][2] = 1."""
    if split == 'i':
        th, s, sh, persp, t = rng.uniform(-0.01, 0.01), rng.uniform(0.99, 1.01), 0.0, (0.0, 0.0), rng.uniform(-3, 3, 2)
    else:
        th, s, sh = rng.uniform(-0.25, 0.25), rng.uniform(0.8, 1.2), rng.uniform(-0.05, 0.05)
        persp = rng.uniform(-0.25, 0.25, 2) / max(w1, h1)
        t = rng.uniform(-0.05, 0.05, 2) * (w2, h2)
    A = s * np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]]) @ np.array([[1.0, sh], [0.0, 1.0]])
    M = np.eye(3)
    M[:2, :2] = A
    M[2, :2] = persp
    T1 = np.array([[1.0, 0, -(w1 - 1) / 2], [0, 1.0, -(h1 - 1) / 2], [0, 0, 1.0]])
    T2 = np.array([[1.0, 0, (w2 - 1) / 2 + t[0]], [0, 1.0, (h2 - 1) / 2 + t[1]], [0, 0, 1.0]])
    H = T2 @ M @ T1
    return H / H[2, 2]


def synthetic_hpatches_tree(root, seed, seqs):
    """HPatches-sequences layout under `root` from a seed, for tests and benchmarks: per sequence, root/name/1.ppm ..
    6.ppm and H_1_2 .. H_1_6.  `seqs` lists names (split from the i_ / v_ prefix, seeded size) or (name, (w, h)).
    1.ppm is a blocky 8-bit texture cropped from a larger canvas; k.ppm is the canvas warped by H_1_k (fp64 numpy inverse
    mapping, nearest pixel, 0 outside the canvas): a near-identity H and a brightness change for i_ sequences, rotation,
    scale, shear and perspective (and a size of its own) for v_ ones.  H_1_k is written with %.17g, so np.loadtxt reads
    back exactly the H used.  -> {name: [H_1_2 .. H_1_6]}"""
    from PIL import Image
    out = {}
    for idx, item in enumerate(seqs):
        name, size = (item, None) if isinstance(item, str) else (item[0], item[1])
        split = name[:1]
        rng = np.random.default_rng([int(seed), 5, idx])
        w1, h1 = (int(v) for v in size) if size is not None else (int(rng.integers(160, 321)), int(rng.integers(128, 257)))
        m = max(w1, h1) // 2
        cw, ch = w1 + 2 * m, h1 + 2 * m
        low = rng.integers(0, 256, size=(ch // 8 + 2, cw // 8 + 2, 3), dtype=np.int32)
        base = np.repeat(np.repeat(low, 8, 0), 8, 1)[:ch + 4, :cw + 4]
        base = (base[:ch, :cw] + base[4:ch + 4, :cw] + base[:ch, 4:cw + 4] + base[4:ch + 4, 4:cw + 4]) // 4
        canvas = np.clip(base + rng.integers(-12, 13, size=base.shape), 0, 255).astype(np.uint8)
        d = os.path.join(root, name)
        os.makedirs(d, exist_ok=True)
        Image.fromarray(canvas[m:m + h1, m:m + w1].copy()).save(os.path.join(d, '1.ppm'))
        Hs = []
        for k in range(2, 7):
            if split == 'v':
                w2, h2 = int(w1 * rng.uniform(0.85, 1.15)), int(h1 * rng.uniform(0.85, 1.15))
            else:
                w2, h2 = w1, h1
            H = _hpatches_h(rng, split, w1, h1, w2, h2)
            Hi = np.linalg.inv(H)
            v, u = np.mgrid[0:h2, 0:w2].astype(np.float64)
            q = Hi[2, 0] * u + Hi[2, 1] * v + Hi[2, 2]
            with np.errstate(all='ignore'):
                x = (Hi[0, 0] * u + Hi[0, 1] * v + Hi[0, 2]) / q
                y = (Hi[1, 0] * u + Hi[1, 1] * v + Hi[1, 2]) / q
            xi, yi = np.floor(x + 0.5) + m, np.floor(y + 0.5) + m
            ok = (q > 0) & (xi >= 0) & (xi < cw) & (yi >= 0) & (yi < ch)
            img = np.zeros((h2, w2, 3), dtype=np.uint8)
            img[ok] = canvas[yi[ok].astype(np.int64), xi[ok].astype(np.int64)]
            if split == 'i':
                gain, bias = rng.uniform(0.6, 1.4), rng.uniform(-20, 20)
                img = np.clip(np.floor(img * gain + bias), 0, 255).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(d, f'{k}.ppm'))
            np.savetxt(os.path.join(d, f'H_1_{k}'), H, fmt='%.17g')
            Hs.append(H)
        out[name] = Hs
    return out


# ---- relative-pose pair lists (SuperGlue's text format, LoFTR's scene-info .npz) ------------------------------------
def synthetic_relpose_pair(seed, size=(320, 240)):
    """A seeded two-view scene of a textured plane for the relative-pose evaluation: cameras as synthetic_two_view's
    (principal points at the image centres, camera 1 rotated up to 0.09 rad per axis and translated by ~1 unit, the
    plane 5-7 units away), each with its own focal length (0.8-1.2 x the width), so f_mean differs from view 1's mean
    focal length.  Image 0 is a blocky 8-bit texture cropped from a larger canvas; image 1 is the canvas seen through the
    plane's homography K1 (R + t n^T / d) K0^-1 (fp64 inverse mapping, nearest pixel, 0 outside), so the ground-truth
    pose is exact for every pixel.  size = (w, h) of both images.
    -> dict(img0, img1 [h, w, 3] uint8, K0, K1 (3x3), T_0to1 (4x4: x1 = R x0 + t))."""
    rng = np.random.default_rng([int(seed), 11])
    w, h = (int(v) for v in size)
    K0, K1 = (np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1.0]]) for f in rng.uniform(0.8, 1.2, 2) * w)
    R = _rotation(rng.uniform(-0.09, 0.09, 3))
    t = np.array([rng.uniform(0.6, 1.0) * rng.choice([-1, 1]), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    normal = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), 1.0])
    normal /= np.linalg.norm(normal)
    d = rng.uniform(5.0, 7.0)
    m = max(w, h) // 2
    cw, ch = w + 2 * m, h + 2 * m
    low = rng.integers(0, 256, size=(ch // 8 + 2, cw // 8 + 2, 3), dtype=np.int32)
    base = np.repeat(np.repeat(low, 8, 0), 8, 1)[:ch + 4, :cw + 4]
    base = (base[:ch, :cw] + base[4:ch + 4, :cw] + base[:ch, 4:cw + 4] + base[4:ch + 4, 4:cw + 4]) // 4
    canvas = np.clip(base + rng.integers(-12, 13, size=base.shape), 0, 255).astype(np.uint8)
    Hi = np.linalg.inv(K1 @ (R + np.outer(t, normal) / d) @ np.linalg.inv(K0))
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    q = Hi[2, 0] * u + Hi[2, 1] * v + Hi[2, 2]
    with np.errstate(all='ignore'):
        x = (Hi[0, 0] * u + Hi[0, 1] * v + Hi[0, 2]) / q
        y = (Hi[1, 0] * u + Hi[1, 1] * v + Hi[1, 2]) / q
    xi, yi = np.floor(x + 0.5) + m, np.floor(y + 0.5) + m
    ok = (q > 0) & (xi >= 0) & (xi < cw) & (yi >= 0) & (yi < ch)
    img1 = np.zeros((h, w, 3), dtype=np.uint8)
    img1[ok] = canvas[yi[ok].astype(np.int64), xi[ok].astype(np.int64)]
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return dict(img0=canvas[m:m + h, m:m + w].copy(), img1=img1, K0=K0, K1=K1, T_0to1=T)


def synthetic_relpose_tree(root, seed, n_pairs, fmt='txt', size=(320, 240)):
    """Seeded pair list and images for the relative-pose evaluation under `root`: pair k's images are
    images/pair{k:03d}_0.png and _1.png (synthetic_relpose_pair(seed * 1000 + k, size)), listed in
      fmt 'txt': root/pairs.txt, SuperGlue's format (name0 name1 0 0 K0 (9) K1 (9) T_0to1 (16), written with %.17g,
        so it reads back exactly);
      fmt 'npz': root/scene_info.npz, the layout patch2pix_b200.relpose.read_pairs_npz reads: image_paths (object array
        of paths relative to root), intrinsics [2n, 3, 3], poses [2n, 4, 4] world -> camera (a seeded pose for image 0
        of each pair, T_0to1 @ it for image 1) and pair_infos (object array of ((2k, 2k + 1), overlap, an empty [0, 2]
        array of central matches)).
    -> (pair-list path, [dict(K0, K1, T_0to1)] per pair)."""
    from PIL import Image
    if fmt not in ('txt', 'npz'):
        raise ValueError("fmt must be 'txt' or 'npz'")
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    gts, names = [], []
    for k in range(n_pairs):
        sc = synthetic_relpose_pair(int(seed) * 1000 + k, size)
        nm = [f'images/pair{k:03d}_{i}.png' for i in range(2)]
        for i in range(2):
            Image.fromarray(sc[f'img{i}']).save(os.path.join(root, nm[i]))
        gts.append(dict(K0=sc['K0'], K1=sc['K1'], T_0to1=sc['T_0to1']))
        names.append(nm)
    if fmt == 'txt':
        path = os.path.join(root, 'pairs.txt')
        with open(path, 'w') as f:
            for nm, g in zip(names, gts):
                vals = np.concatenate([g['K0'].reshape(-1), g['K1'].reshape(-1), g['T_0to1'].reshape(-1)])
                f.write(' '.join([nm[0], nm[1], '0', '0'] + ['%.17g' % v for v in vals]) + '\n')
        return path, gts
    rng = np.random.default_rng([int(seed), 12])
    paths = np.empty(2 * n_pairs, dtype=object)
    Ks, poses = np.zeros((2 * n_pairs, 3, 3)), np.zeros((2 * n_pairs, 4, 4))
    infos = np.empty(n_pairs, dtype=object)
    for k, (nm, g) in enumerate(zip(names, gts)):
        T0 = np.eye(4)
        T0[:3, :3], T0[:3, 3] = _rotation(rng.uniform(-1.0, 1.0, 3)), rng.uniform(-5.0, 5.0, 3)
        paths[2 * k], paths[2 * k + 1] = nm
        Ks[2 * k], Ks[2 * k + 1] = g['K0'], g['K1']
        poses[2 * k], poses[2 * k + 1] = T0, g['T_0to1'] @ T0
        infos[k] = ((2 * k, 2 * k + 1), float(rng.uniform(0.1, 0.7)), np.zeros((0, 2)))
    path = os.path.join(root, 'scene_info.npz')
    np.savez(path, image_paths=paths, intrinsics=Ks, poses=poses, pair_infos=infos)
    return path, gts


# ---- NCNet (ImMatchNet) test data: regenerated from seeds, so fixtures store outputs only ----------------------------
def ncnet_stack_weights(seed, kernel_sizes, channels):
    """Conv4d weights in the reference's pre-permuted layout [k, Cout, Cin, k, k, k] and biases [Cout], fp32, scaled so
    that activations stay O(1) and mostly positive through the ReLUs."""
    g = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for i, (k, c) in enumerate(zip(kernel_sizes, channels)):
        cin = 1 if i == 0 else channels[i - 1]
        ws.append((torch.rand(k, c, cin, k, k, k, generator=g) - 0.35) / (cin * k ** 4) ** 0.5)
        bs.append(0.05 * torch.randn(c, generator=g))
    return ws, bs


def ncnet_state_dict(seed, names_shapes, kernel_sizes, channels):
    """A seeded ImMatchNet state_dict for the given (name, shape) list: ResNet101 convs He-scaled, BatchNorm near
    identity, NeighConsensus from ncnet_stack_weights.  Names keep their order, so any holder of the same list
    regenerates the same tensors."""
    g = torch.Generator().manual_seed(seed)
    ws, bs = ncnet_stack_weights(seed + 1, kernel_sizes, channels)
    nc = {}
    for i, (w, b) in enumerate(zip(ws, bs)):
        nc[f'NeighConsensus.conv.{2 * i}.weight'], nc[f'NeighConsensus.conv.{2 * i}.bias'] = w, b
    sd = {}
    for name, shape in names_shapes:
        shape = tuple(shape)
        if name in nc:
            sd[name] = nc[name]
        elif name.endswith('num_batches_tracked'):
            sd[name] = torch.zeros((), dtype=torch.int64)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            sd[name] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif name.endswith('running_var'):
            sd[name] = 0.5 + torch.rand(shape, generator=g)
        elif name.endswith('running_mean'):
            sd[name] = 0.1 * torch.randn(shape, generator=g)
        elif name.endswith('weight'):
            sd[name] = 0.25 + 0.5 * torch.rand(shape, generator=g)
        else:
            sd[name] = 0.1 * torch.randn(shape, generator=g)
    return sd


def ncnet_features(seed, c, size1, size2):
    """A pair of layer3-like feature maps [1, c, h, w] with a shared structure (so that matches are distinct)."""
    g = torch.Generator().manual_seed(seed)
    fa = torch.rand(1, c, *size1, generator=g)
    fb = torch.rand(1, c, *size2, generator=g)
    fa[:, :, : size1[0] // 2] += 2 * torch.rand(1, c, size1[0] // 2, size1[1], generator=g)
    fb[:, :, : min(size2[0], size1[0]) // 2, : min(size2[1], size1[1])] += \
        fa[:, :, : min(size2[0], size1[0]) // 2, : min(size2[1], size1[1])]
    return fa, fb


def ncnet_images(seed, size1, size2):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, 3, *size1, generator=g), torch.rand(1, 3, *size2, generator=g)


# ---- absolute pose and InLoc-layout trees ------------------------------------------------------------------------------
def synthetic_abspose(seed, n, outlier_ratio, noise_px, width=1024, height=768, focal=900.0):
    """Seeded 2D-3D correspondences with a known pose, for absolute-pose RANSAC: a pinhole camera (focal `focal`,
    principal point at the image centre) with a random orientation, its centre about 100 units from the world origin (so
    the world coordinates are far from zero, as InLoc's are), round(n * (1 - outlier_ratio)) world points 2-20 units in
    front of it projected into the image with N(0, noise_px^2) pixel noise, and outliers pairing uniform pixels with
    world points drawn like the true ones, shuffled.
    -> dict(pts2d [n, 2], pts3d [n, 3] float64, K (3x3), R, t (x_cam = R X + t), inlier [n] bool)."""
    rng = np.random.default_rng([int(seed), 21])
    K = np.array([[focal, 0, width / 2], [0, focal, height / 2], [0, 0, 1.0]])
    R = _rotation(rng.normal(0.0, 1.0, 3))
    C = rng.uniform(-10.0, 10.0, 3) + np.array([100.0, -60.0, 25.0])
    t = -R @ C

    def points(m):
        uv = rng.uniform([0, 0], [width, height], (m, 2))
        ray = np.linalg.solve(K, np.concatenate([uv, np.ones((m, 1))], 1).T).T
        return uv, (ray * rng.uniform(2.0, 20.0, m)[:, None] - t) @ R
    n_in = int(round(n * (1.0 - outlier_ratio)))
    uv, X = points(n_in)
    uv = uv + rng.normal(0.0, noise_px, uv.shape)
    _, Xo = points(n - n_in)
    uvo = rng.uniform([0, 0], [width, height], (n - n_in, 2))
    perm = rng.permutation(n)
    return dict(pts2d=np.concatenate([uv, uvo])[perm], pts3d=np.concatenate([X, Xo])[perm], K=K, R=R, t=t,
                inlier=np.concatenate([np.ones(n_in, bool), np.zeros(n - n_in, bool)])[perm])


INLOC_FOCAL = 4032.0 * 28.0 / 36.0    # hloc's focal length of InLoc's iPhone 7 queries


def _look_at(C, target, roll):
    z = target - C
    z = z / np.linalg.norm(z)
    x = np.cross(np.array([0.0, 0.0, 1.0]), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])                                  # rows: camera axes in world coordinates
    return _rotation(np.array([0.0, 0.0, roll])) @ R


def _render_plane(scene, K, R, t, w, h):
    """World points [h, w, 3] of the plane seen through each pixel centre (NaN off the textured area or behind the
    camera) and the image [h, w, 3] uint8 (nearest texel, 0 where NaN)."""
    O, e1, e2, nrm, texel, canvas = (scene[k] for k in ('O', 'e1', 'e2', 'n', 'texel', 'canvas'))
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    ray = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1) @ R   # world directions
    C = -R.T @ t
    lam = ((O - C) @ nrm) / (ray @ nrm)
    X = C + lam[..., None] * ray
    a = ((X - O) @ e1) / texel + canvas.shape[1] / 2
    b = ((X - O) @ e2) / texel + canvas.shape[0] / 2
    ai, bi = np.floor(a + 0.5), np.floor(b + 0.5)
    ok = (lam > 0) & (ai >= 0) & (ai < canvas.shape[1]) & (bi >= 0) & (bi < canvas.shape[0])
    img = np.zeros((h, w, 3), dtype=np.uint8)
    img[ok] = canvas[bi[ok].astype(np.int64), ai[ok].astype(np.int64)]
    X[~ok] = np.nan
    return X, img


def _quat(R):
    from .localize import rotmat_to_qvec
    return rotmat_to_qvec(R)


def synthetic_inloc_tree(root, seed, n_queries, n_db, size=(320, 240)):
    """Seeded InLoc-layout tree under `root`, in the layout patch2pix_b200.localize reads: a textured plane about 100
    units from the world origin, seen by
      query/iphone7/IMG_{k:04d}.JPG: query k, focal INLOC_FOCAL, principal point at the image centre;
      database/cutouts/DUC1/{s:03d}/DUC_cutout_{s:03d}_{30 j}_0.jpg (+ .jpg.mat): n_db cutouts per query from nearby
        cameras, each with its scan `XYZcut` [h, w, 3] in the scan's own frame (NaN off the plane and in a few seeded
        rectangular holes);
      database/alignments/DUC1/transformations/DUC_trans_{s:03d}.txt: the scan-to-world transform, 4x4 rows on lines
        7-10 (counted from 0) after a header;
      pairs.txt: hloc's retrieval list ('query db' per line, grouped by query);
      gt_poses.txt: the queries' poses as localize writes them (name qw qx qy qz tx ty tz, world -> camera).
    Images are size = (w, h) PNG data behind .JPG / .jpg names (PIL reads either).
    -> dict(pairs, gt (paths), queries {query name: (K, R, t)}, db {db name: (K, R, t)}, scene)."""
    from PIL import Image
    from scipy.io import savemat
    rng = np.random.default_rng([int(seed), 31])
    w, h = (int(v) for v in size)
    canvas_px = 1024
    low = rng.integers(0, 256, size=(canvas_px // 8 + 2, canvas_px // 8 + 2, 3), dtype=np.int32)
    base = np.repeat(np.repeat(low, 8, 0), 8, 1)[:canvas_px + 4, :canvas_px + 4]
    base = (base[:canvas_px, :canvas_px] + base[4:, :canvas_px] + base[:canvas_px, 4:] + base[4:, 4:]) // 4
    canvas = np.clip(base + rng.integers(-12, 13, size=base.shape), 0, 255).astype(np.uint8)
    nrm = np.array([rng.uniform(-0.2, 0.2), 1.0, rng.uniform(-0.1, 0.1)])
    nrm /= np.linalg.norm(nrm)
    e1 = np.cross(np.array([0.0, 0.0, 1.0]), nrm)
    e1 /= np.linalg.norm(e1)
    scene = dict(O=np.array([120.0, -40.0, 30.0]), n=nrm, e1=e1, e2=np.cross(nrm, e1), texel=0.002, canvas=canvas)
    K = np.array([[INLOC_FOCAL, 0, w / 2], [0, INLOC_FOCAL, h / 2], [0, 0, 1.0]])

    def camera(center_off, target_off, dist):
        C = scene['O'] + scene['n'] * dist + scene['e1'] * center_off[0] + scene['e2'] * center_off[1]
        T = scene['O'] + scene['e1'] * target_off[0] + scene['e2'] * target_off[1]
        R = _look_at(C, T, rng.uniform(-0.1, 0.1))
        return R, -R @ C
    for d in ('query/iphone7', 'database/cutouts/DUC1', 'database/alignments/DUC1/transformations'):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    queries, db, lines, gt_lines = {}, {}, [], []
    for k in range(n_queries):
        qname = f'query/iphone7/IMG_{k:04d}.JPG'
        tgt = rng.uniform(-0.4, 0.4, 2)
        R, t = camera(tgt + rng.uniform(-0.5, 0.5, 2), tgt, rng.uniform(5.0, 7.0))
        _, img = _render_plane(scene, K, R, t, w, h)
        Image.fromarray(img).save(os.path.join(root, qname), format='PNG')
        queries[qname] = (K, R, t)
        q = _quat(R)
        gt_lines.append(' '.join([os.path.basename(qname)] + ['%.17g' % v for v in np.concatenate([q, t])]))
        for j in range(n_db):
            s = k * n_db + j
            dname = f'database/cutouts/DUC1/{s:03d}/DUC_cutout_{s:03d}_{30 * j}_0.jpg'
            os.makedirs(os.path.dirname(os.path.join(root, dname)), exist_ok=True)
            Rd, td = camera(tgt + rng.uniform(-0.5, 0.5, 2), tgt + rng.uniform(-0.03, 0.03, 2), rng.uniform(5.0, 7.0))
            X, img = _render_plane(scene, K, Rd, td, w, h)
            Image.fromarray(img).save(os.path.join(root, dname), format='PNG')
            Ta = np.eye(4)
            Ta[:3, :3], Ta[:3, 3] = _rotation(np.array([0.0, 0.0, rng.uniform(-np.pi, np.pi)])), rng.uniform(-50, 50, 3)
            Xl = (X - Ta[:3, 3]) @ Ta[:3, :3]                  # the scan's own frame: X = Ta[:3, :3] Xl + Ta[:3, 3]
            for _ in range(3):
                y0, x0 = int(rng.integers(0, h - 8)), int(rng.integers(0, w - 8))
                Xl[y0:y0 + int(rng.integers(2, 9)), x0:x0 + int(rng.integers(2, 9))] = np.nan
            savemat(os.path.join(root, dname + '.mat'), {'XYZcut': Xl})
            with open(os.path.join(root, 'database/alignments/DUC1/transformations', f'DUC_trans_{s:03d}.txt'),
                      'w') as f:
                f.write(f'DUC_scan_{s:03d}.ptx\n\nAfter general icp:\n')
                f.write('\n'.join(' '.join('%.17g' % v for v in row) for row in np.eye(4)) + '\n')
                f.write('\n'.join(' '.join('%.17g' % v for v in row) for row in Ta) + '\n')
            db[dname] = (K, Rd, td)
            lines.append(f'{qname} {dname}')
    pairs = os.path.join(root, 'pairs.txt')
    with open(pairs, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    gt = os.path.join(root, 'gt_poses.txt')
    with open(gt, 'w') as f:
        f.write('\n'.join(gt_lines) + '\n')
    return dict(pairs=pairs, gt=gt, queries=queries, db=db, scene=scene)


def inloc_gt_matcher(tree, step=8):
    """Callable (query_path, db_path) -> [N, 4] (xq, yq, xdb, ydb) ground-truth matches of a synthetic_inloc_tree: a
    pixel grid of the query, its plane points projected into the cutout, kept inside the cutout."""
    def matcher(qpath, dpath):
        qn = next(k for k in tree['queries'] if qpath.endswith(k))
        dn = next(k for k in tree['db'] if dpath.endswith(k))
        K, R, t = tree['queries'][qn]
        Kd, Rd, td = tree['db'][dn]
        w, h = int(round(2 * K[0, 2])), int(round(2 * K[1, 2]))
        X, _ = _render_plane(tree['scene'], K, R, t, w, h)
        v, u = np.mgrid[0:h:step, 0:w:step]
        X = X[v, u].reshape(-1, 3)
        P = X @ Rd.T + td
        with np.errstate(invalid='ignore'):
            xd = Kd[0, 0] * P[:, 0] / P[:, 2] + Kd[0, 2]
            yd = Kd[1, 1] * P[:, 1] / P[:, 2] + Kd[1, 2]
            ok = np.isfinite(xd) & (xd >= 0) & (xd <= w - 1) & (yd >= 0) & (yd <= h - 1)
        return np.stack([u.reshape(-1), v.reshape(-1), xd, yd], 1)[ok].astype(np.float64)
    return matcher


def _radial_undistort(f, cx, cy, k, x, y, iters=20):
    """Normalised rays of distorted pixels under SIMPLE_RADIAL (f, cx, cy, k): Newton on u (1 + k r^2) = x."""
    xd, yd = (x - cx) / f, (y - cy) / f
    u, v = xd.copy(), yd.copy()
    for _ in range(iters):
        r2 = u * u + v * v
        a = 1.0 + k * r2
        fu, fv = u * a - xd, v * a - yd
        j00, j11, j01 = a + 2 * k * u * u, a + 2 * k * v * v, 2 * k * u * v
        det = j00 * j11 - j01 * j01
        u, v = u - (j11 * fu - j01 * fv) / det, v - (j00 * fv - j01 * fu) / det
    return u, v


def _radial_project(cam, R, t, X):
    f, cx, cy, k = cam
    P = X @ R.T + t
    with np.errstate(invalid='ignore', divide='ignore'):
        u, v = P[..., 0] / P[..., 2], P[..., 1] / P[..., 2]
    r2 = u * u + v * v
    return f * u * (1 + k * r2) + cx, f * v * (1 + k * r2) + cy, P[..., 2]


def _radial_plane_points(scene, cam, R, t, x, y):
    """World points on the scene plane seen through distorted pixels (x, y) (NaN behind the camera or off the plane)."""
    u, v = _radial_undistort(*cam, x, y)
    ray = np.stack([u, v, np.ones_like(u)], -1) @ R
    C = -R.T @ t
    lam = ((scene['O'] - C) @ scene['n']) / (ray @ scene['n'])
    X = C + lam[..., None] * ray
    X[lam <= 0] = np.nan
    return X


def synthetic_aachen_tree(root, seed, n_db, n_queries, size=(320, 240), focal=180.0, k=-0.05, db_neighbours=3,
                          query_neighbours=3):
    """Seeded Aachen-layout tree under `root`, in metres: a textured plane 10 m wide through the origin, seen from 5-7 m
    by SIMPLE_RADIAL cameras (f = focal, principal point at the centre, k != 0), written as
      images/db/{i:04d}.png, images/query/{k:04d}.png: PNG images rendered with the distortion;
      model/cameras.bin, images.bin: the database cameras and poses (write_colmap_model; no 2D points);
      db_pairs.txt: each database image with its next db_neighbours along the row of cameras;
      query_pairs.txt: each query with its query_neighbours nearest database images (camera centres);
      queries.txt: 'name SIMPLE_RADIAL w h f cx cy k' per query;  gt_poses.txt: the queries' poses (localize's format,
      file names without their directory).
    -> dict(images, model, db_pairs, query_pairs, queries, gt, cams {name: (f, cx, cy, k)}, poses {name: (R, t)},
    scene)."""
    from PIL import Image
    rng = np.random.default_rng([int(seed), 47])
    w, h = (int(v) for v in size)
    canvas_px = 1024
    low = rng.integers(0, 256, size=(canvas_px // 8 + 2, canvas_px // 8 + 2, 3), dtype=np.int32)
    base = np.repeat(np.repeat(low, 8, 0), 8, 1)[:canvas_px + 4, :canvas_px + 4]
    base = (base[:canvas_px, :canvas_px] + base[4:, :canvas_px] + base[:canvas_px, 4:] + base[4:, 4:]) // 4
    canvas = np.clip(base + rng.integers(-12, 13, size=base.shape), 0, 255).astype(np.uint8)
    nrm = np.array([rng.uniform(-0.1, 0.1), 1.0, rng.uniform(-0.1, 0.1)])
    nrm /= np.linalg.norm(nrm)
    e1 = np.cross(np.array([0.0, 0.0, 1.0]), nrm)
    e1 /= np.linalg.norm(e1)
    scene = dict(O=np.zeros(3), n=nrm, e1=e1, e2=np.cross(nrm, e1), texel=10.0 / canvas_px, canvas=canvas)
    cam = (float(focal), w / 2.0, h / 2.0, float(k))
    root = str(root)
    for d in ('images/db', 'images/query', 'model'):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)

    def render(R, t):
        X = _radial_plane_points(scene, cam, R, t, u, v)
        a = ((X - scene['O']) @ scene['e1']) / scene['texel'] + canvas_px / 2
        b = ((X - scene['O']) @ scene['e2']) / scene['texel'] + canvas_px / 2
        with np.errstate(invalid='ignore'):
            ai, bi = np.floor(a + 0.5), np.floor(b + 0.5)
            ok = (ai >= 0) & (ai < canvas_px) & (bi >= 0) & (bi < canvas_px)
        img = np.zeros((h, w, 3), dtype=np.uint8)
        img[ok] = canvas[bi[ok].astype(np.int64), ai[ok].astype(np.int64)]
        return img

    def camera(off):
        C = scene['n'] * rng.uniform(5.0, 7.0) + scene['e1'] * off[0] + scene['e2'] * off[1]
        T = scene['e1'] * (0.6 * off[0]) + scene['e2'] * (0.6 * off[1]) + rng.uniform(-0.2, 0.2, 3)
        R = _look_at(C, T, rng.uniform(-0.1, 0.1))
        return R, -R @ C
    poses, cams, db_imgs, centres = {}, {}, [], []
    for i in range(n_db):
        name = f'db/{i:04d}.png'
        off = np.array([-2.0 + 4.0 * i / max(n_db - 1, 1), rng.uniform(-0.5, 0.5)])
        R, t = camera(off)
        Image.fromarray(render(R, t)).save(os.path.join(root, 'images', name), format='PNG')
        poses[name], cams[name] = (R, t), cam
        db_imgs.append((i + 1, _quat(R), t, 1, name))
        centres.append(-R.T @ t)
    write_colmap_model(os.path.join(root, 'model'), [(1, 2, w, h, list(cam))], db_imgs)
    names = [d[4] for d in db_imgs]
    with open(os.path.join(root, 'db_pairs.txt'), 'w') as f:
        for i in range(n_db):
            for j in range(i + 1, min(n_db, i + 1 + db_neighbours)):
                f.write(f'{names[i]} {names[j]}\n')
    qlines, plines, glines = [], [], []
    centres = np.array(centres)
    for q in range(n_queries):
        name = f'query/{q:04d}.png'
        R, t = camera(np.array([rng.uniform(-1.6, 1.6), rng.uniform(-0.4, 0.4)]))
        Image.fromarray(render(R, t)).save(os.path.join(root, 'images', name), format='PNG')
        poses[name], cams[name] = (R, t), cam
        qlines.append(f'{name} SIMPLE_RADIAL {w} {h} ' + ' '.join('%.17g' % x for x in cam))
        near = np.argsort(np.linalg.norm(centres - (-R.T @ t), axis=1), kind='stable')[:query_neighbours]
        plines += [f'{name} {names[j]}' for j in near]
        glines.append(' '.join([os.path.basename(name)] + ['%.17g' % x for x in np.concatenate([_quat(R), t])]))
    out = dict(images=os.path.join(root, 'images'), model=os.path.join(root, 'model'),
               db_pairs=os.path.join(root, 'db_pairs.txt'), query_pairs=os.path.join(root, 'query_pairs.txt'),
               queries=os.path.join(root, 'queries.txt'), gt=os.path.join(root, 'gt_poses.txt'), cams=cams,
               poses=poses, scene=scene)
    for key, lines in (('query_pairs', plines), ('queries', qlines), ('gt', glines)):
        with open(out[key], 'w') as f:
            f.write('\n'.join(lines) + '\n')
    return out


def aachen_gt_matcher(tree, step=8):
    """Callable (path0, path1) -> [N, 4] exact correspondences of a synthetic_aachen_tree: a pixel grid of image 0,
    its plane points projected, with the distortion, into image 1 and kept inside it."""
    def matcher(p0, p1):
        n0 = next(k for k in tree['poses'] if p0.endswith(k))
        n1 = next(k for k in tree['poses'] if p1.endswith(k))
        c0, c1 = tree['cams'][n0], tree['cams'][n1]
        w, h = int(round(2 * c0[1])), int(round(2 * c0[2]))
        v, u = np.mgrid[0:h:step, 0:w:step].astype(np.float64)
        u, v = u.reshape(-1) + 0.5, v.reshape(-1) + 0.5
        X = _radial_plane_points(tree['scene'], c0, *tree['poses'][n0], u, v)
        x1, y1, z1 = _radial_project(c1, *tree['poses'][n1], X)
        with np.errstate(invalid='ignore'):
            ok = np.isfinite(x1) & (z1 > 0) & (x1 >= 0) & (x1 <= 2 * c1[1] - 1) & (y1 >= 0) & (y1 <= 2 * c1[2] - 1)
        return np.stack([u, v, x1, y1], 1)[ok]
    return matcher
