"""NCNet's matcher on the GPU: the general NeighConsensus stack (nc_stack.cu) and ImMatchNet.forward_feat against
the float64 oracle, the stack against the fixed Patch2Pix NeighConsensus, and its independence of the grid."""
import numpy as np
import pytest
import torch

from oracle import ncnet_oracle as O

pytestmark = pytest.mark.gpu

STACKS = [([3, 3, 3], [10, 10, 1]), ([5, 5, 5], [16, 16, 1]), ([3, 5], [8, 1]), ([5], [1]), ([3, 3, 3], [16, 16, 1])]
# (hA, wA, hB, wB), input scale: dimensions below k, a single-row and a 150-wide B grid, tiny / large / zero inputs
SHAPES = [((3, 4, 5, 6), 1.0), ((2, 3, 1, 150), 1.0), ((6, 5, 9, 11), 1e-3), ((4, 6, 2, 9), 37.0), ((3, 3, 3, 3), 0.0)]


def _weights(ks, ch, seed):
    g = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for i, (k, c) in enumerate(zip(ks, ch)):
        cin = 1 if i == 0 else ch[i - 1]
        ws.append((torch.rand(k, c, cin, k, k, k, generator=g) - 0.35) / (cin * k ** 4) ** 0.5)
        bs.append(0.05 * torch.randn(c, generator=g))
    return ws, bs


def _module(ks, ch, sym, ws, bs):
    from patch2pix_b200.ncnet import NeighConsensus
    nc = NeighConsensus(kernel_sizes=ks, channels=ch, symmetric_mode=sym)
    sd = {}
    for i, (w, b) in enumerate(zip(ws, bs)):
        sd[f'conv.{2 * i}.weight'], sd[f'conv.{2 * i}.bias'] = w, b
    nc.load_state_dict(sd)
    return nc.eval()


def _clear_boxes(fa, fb, k, margin=1e-4):
    """maxpool boxes whose float64 maximum leads the runner-up by more than `margin` (relative): there the offsets of
    any fp32-grade correlation must equal the oracle's."""
    c = O.correlation(O.l2norm(fa.unsqueeze(0))[0], O.l2norm(fb.unsqueeze(0))[0])
    h1, w1, h2, w2 = c.shape
    v = c.reshape(h1 // k, k, w1 // k, k, h2 // k, k, w2 // k, k).permute(0, 2, 4, 6, 1, 3, 5, 7)
    top = v.reshape(h1 // k, w1 // k, h2 // k, w2 // k, k ** 4).topk(2, -1).values
    return (top[..., 0] - top[..., 1]) > margin * top[..., 0].abs().clamp_min(1e-30)


def _check(out, ref):
    scale = max(ref.abs().max().item(), 1e-30)
    assert torch.isfinite(out).all()
    np.testing.assert_allclose(out.double().numpy(), ref.numpy(), rtol=2e-4, atol=5e-6 * scale)


@pytest.mark.parametrize('sym', [True, False])
@pytest.mark.parametrize('ks, ch', STACKS)
def test_nc_stack_vs_oracle(ks, ch, sym):
    ws, bs = _weights(ks, ch, sum(ks) * 10 + len(ch))
    nc = _module(ks, ch, sym, ws, bs)
    for (hA, wA, hB, wB), amp in SHAPES:
        g = torch.Generator().manual_seed(hA * 1000 + wB)
        x = (torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1) * amp
        out = nc(x.cuda()).cpu()
        ref = O.nc_stack(x[0, 0], [w.double() for w in ws], [b.double() for b in bs], sym)
        _check(out[0, 0], ref)


def test_nc_stack_matches_the_fixed_patch2pix_neigh_consensus(consensus_sd):
    """[3, 3] / [16, 1] through the general stack against p2p_neigh_consensus (nc_umma.cu) on the same weights."""
    from patch2pix_b200 import _lib
    ws = [consensus_sd['ncn.conv.0.weight'], consensus_sd['ncn.conv.2.weight']]
    bs = [consensus_sd['ncn.conv.0.bias'], consensus_sd['ncn.conv.2.bias']]
    nc = _module([3, 3], [16, 1], True, ws, bs)
    h = _lib.Handle('cuda:0')
    w = [t.float().contiguous() for t in (ws[0], bs[0], ws[1], bs[1])]
    _lib.check(h.lib.p2p_set_ncn_weights(h.h, *[_lib.ptr(t) for t in w]))
    for (hA, wA, hB, wB), amp in SHAPES[:4] + [((15, 20, 15, 20), 1.0)]:
        g = torch.Generator().manual_seed(hA + 7 * wB)
        x = ((torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1) * amp).cuda()
        fixed = torch.empty_like(x)
        _lib.check(h.lib.p2p_neigh_consensus(h.h, _lib.ptr(x), hA, wA, hB, wB, _lib.ptr(fixed), h.stream()))
        out = nc(x)
        torch.cuda.synchronize()
        ref = O.nc_stack(x[0, 0].cpu(), [t.double() for t in ws], [t.double() for t in bs], True)
        _check(out[0, 0].cpu(), ref)
        scale = max(fixed.abs().max().item(), 1e-30)
        np.testing.assert_allclose(out.cpu().numpy(), fixed.cpu().numpy(), rtol=2e-4, atol=5e-6 * scale)


def test_nc_stack_independent_of_grid_and_repeatable():
    ks, ch = [5, 3, 3], [16, 16, 1]
    ws, bs = _weights(ks, ch, 5)
    nc = _module(ks, ch, True, ws, bs)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(2, 1, 5, 7, 6, 9, generator=g).cuda()
    base = nc(x)
    assert torch.equal(nc(x), base)
    for i in range(2):
        assert torch.equal(nc(x[i:i + 1]), base[i:i + 1])
    h = nc._handle(x.device)
    for n in (1, 3, 131):
        h.set_option('num_sms', n)
        try:
            assert torch.equal(nc(x), base), n
        finally:
            h.set_option('num_sms', 0)


@pytest.mark.parametrize('ksize', [1, 2])
def test_forward_feat_vs_oracle(ksize):
    """ImMatchNet.forward_feat on C = 1024 layer3-like features of different sizes for the two images."""
    from patch2pix_b200.ncnet import ImMatchNet
    ks, ch = [3, 3, 3], [10, 10, 1]
    ws, bs = _weights(ks, ch, 21)
    net = ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=ksize if ksize > 1 else 0)
    sd = net.state_dict()
    for i, (w, b) in enumerate(zip(ws, bs)):
        sd[f'NeighConsensus.conv.{2 * i}.weight'], sd[f'NeighConsensus.conv.{2 * i}.bias'] = w, b
    net.load_state_dict(sd)
    g = torch.Generator().manual_seed(ksize)
    fa = torch.rand(2, 1024, 8, 10, generator=g)
    fb = torch.rand(2, 1024, 12, 6, generator=g)
    fa[:, :, 2:4] += 2 * torch.rand(2, 1024, 2, 10, generator=g)
    r = net.forward_feat(fa.cuda(), fb.cuda())
    corr, deltas = (r if ksize > 1 else (r, None))
    assert corr.shape == (2, 1, 8 // ksize, 10 // ksize, 12 // ksize, 6 // ksize) and corr.dtype == torch.float32
    if ksize > 1:
        assert [d.dtype for d in deltas] == [torch.float32] * 3 + [torch.int64]
    for i in range(2):
        ref, rd = O.forward_feat(fa[i], fb[i], [w.double() for w in ws], [b.double() for b in bs], ksize)
        _check(corr[i, 0].cpu(), ref)
        if ksize > 1:
            for d, e in zip(deltas, rd):
                assert torch.equal(d[i, 0].cpu().long(), e), 'deltas differ'
        one = net.forward_feat(fa[i:i + 1].cuda(), fb[i:i + 1].cuda())
        assert torch.equal((one[0] if ksize > 1 else one)[0], corr[i])


def test_forward_from_images_vs_oracle():
    """ImMatchNet.forward: the torchvision ResNet101 layer3 backbone (TF32 off) then the CUDA matcher."""
    from patch2pix_b200.ncnet import ImMatchNet
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(0)
        net = ImMatchNet(ncons_kernel_sizes=[3, 3], ncons_channels=[16, 1], relocalization_k_size=2)
        ws, bs = _weights([3, 3], [16, 1], 4)
        sd = net.state_dict()
        for i, (w, b) in enumerate(zip(ws, bs)):
            sd[f'NeighConsensus.conv.{2 * i}.weight'], sd[f'NeighConsensus.conv.{2 * i}.bias'] = w, b
        net.load_state_dict(sd)
        assert next(net.FeatureExtraction.parameters()).is_cuda      # placed on the GPU as the reference's use_cuda
        g = torch.Generator().manual_seed(9)
        ia, ib = torch.rand(1, 3, 192, 256, generator=g), torch.rand(1, 3, 160, 224, generator=g)
        corr, deltas = net({'source_image': ia.cuda(), 'target_image': ib.cuda()})
        with torch.no_grad():
            fa, fb = net.FeatureExtraction(ia.cuda()).cpu(), net.FeatureExtraction(ib.cuda()).cpu()
        ref, rd = O.forward_feat(fa[0], fb[0], [w.double() for w in ws], [b.double() for b in bs], 2)
        _check(corr[0, 0].cpu(), ref)
        assert corr.shape == (1, 1, 6, 8, 5, 7)
        assert [d.dtype for d in deltas] == [torch.float32] * 3 + [torch.int64]
        clear = _clear_boxes(fa[0], fb[0], 2)
        assert clear.sum() >= 200
        for d, e in zip(deltas, rd):
            assert torch.equal(d[0, 0].cpu().long()[clear], e[clear]), 'deltas differ'

    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_deep_stack_vs_oracle():
    """Six layers: the compounding weight-norm bound still leaves fp32-grade results."""
    ks, ch = [3, 5, 3, 3, 5, 3], [8, 16, 8, 12, 4, 1]
    ws, bs = _weights(ks, ch, 77)
    for sym in (True, False):
        nc = _module(ks, ch, sym, ws, bs)
        for (hA, wA, hB, wB), amp in SHAPES[:4]:
            g = torch.Generator().manual_seed(hA * 1000 + wB)
            x = (torch.rand(1, 1, hA, wA, hB, wB, generator=g) - 0.1) * amp
            ref = O.nc_stack(x[0, 0], [w.double() for w in ws], [b.double() for b in bs], sym)
            assert ref.abs().max() > 0
            _check(nc(x.cuda()).cpu()[0, 0], ref)


def test_c_abi_rejects_bad_stacks():
    """p2p_set_nc_stack_weights itself (not the Python checks in front of it) refuses every unsupported stack."""
    import ctypes as C
    from patch2pix_b200 import _lib
    h = _lib.Handle('cuda:0')
    keep = []

    def call(ks, ch, n=None):
        n = len(ks) if n is None else n
        ws, bs = [], []
        for i, (k, c) in enumerate(zip(ks, ch)):
            ws.append(torch.zeros(k, c, 1 if i == 0 else ch[i - 1], k, k, k))
            bs.append(torch.zeros(c))
        keep.append((ws, bs))
        return h.lib.p2p_set_nc_stack_weights(h.h, n, (C.c_int * max(n, 1))(*ks), (C.c_int * max(n, 1))(*ch),
                                              (C.c_void_p * max(n, 1))(*[w.data_ptr() for w in ws]),
                                              (C.c_void_p * max(n, 1))(*[b.data_ptr() for b in bs]), 1)
    assert call([3, 3], [8, 1]) == 0
    for ks, ch in (([4, 3], [8, 1]), ([3, 2], [8, 1]), ([7], [1]), ([1], [1]), ([3, 3], [17, 1]), ([3, 3], [0, 1]),
                   ([3, 3], [8, 2]), ([5], [3])):
        assert call(ks, ch) == -1, (ks, ch)
    assert call([3], [1], n=0) == -1 and call([3] * 17, [1] * 17) == -1
    msg = h.lib.p2p_last_error().decode()
    assert 'n_layers' in msg
    x = torch.rand(1, 1, 3, 3, 3, 3, device='cuda')
    out = torch.empty_like(x)                # the last good stack is still in place after the refusals
    _lib.check(h.lib.p2p_nc_stack(h.h, _lib.ptr(x), 3, 3, 3, 3, _lib.ptr(out), h.stream()))


# ---- against the live reference's outputs (tests/golden/ncnet_golden.npz, make_ncnet_golden.py) ------------------------
def _gold():
    import importlib.util
    import os
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
    spec = importlib.util.spec_from_file_location('ncnet_cases', os.path.join(d, 'ncnet_cases.py'))
    K = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(K)
    return K, dict(np.load(os.path.join(d, 'ncnet_golden.npz')))


def test_nc_stacks_vs_reference_goldens():
    from patch2pix_b200 import synth
    K, gold = _gold()
    for ks, ch, wseed in K.NC_STACKS:
        ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
        for sym in (True, False):
            nc = _module(ks, ch, sym, ws, bs)
            for shape, xseed in K.NC_VOLUMES:
                g = torch.Generator().manual_seed(xseed)
                x = torch.rand(1, 1, *shape, generator=g) - 0.1
                ref = gold[f'nc_{"_".join(map(str, ks))}_{"_".join(map(str, ch))}_{int(sym)}_{xseed}']
                _check(nc(x.cuda()).cpu()[0, 0], torch.from_numpy(ref).double())


def _tie_rows(corr, inv, margin=1e-6):
    """Rows whose best and second-best (softmax) values lie within `margin` (relative) in float64: either index is
    a correct arg-max at fp32 precision."""
    hA, wA, hB, wB = corr.shape
    v = corr.double().reshape(hA * wA, hB * wB)
    v = torch.softmax(v.t() if inv else v, 0)
    top = v.topk(min(2, v.shape[0]), 0).values
    if top.shape[0] < 2:
        return torch.zeros(v.shape[1], dtype=torch.bool)
    return (top[0] - top[1]) <= margin * top[0]


def test_forward_feat_and_corr_to_matches_vs_reference_goldens():
    from patch2pix_b200 import synth
    from patch2pix_b200.ncnet import ImMatchNet, corr_to_matches
    K, gold = _gold()
    ks, ch, wseed = K.FEAT_STACK
    ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
    fa, fb = synth.ncnet_features(K.FEAT_SEED, K.FEAT_C, *K.FEAT_SIZES)
    for reloc in K.RELOCS:
        net = ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=reloc)
        sd = net.state_dict()
        for i, (w, b) in enumerate(zip(ws, bs)):
            sd[f'NeighConsensus.conv.{2 * i}.weight'], sd[f'NeighConsensus.conv.{2 * i}.bias'] = w, b
        net.load_state_dict(sd)
        r = net.forward_feat(fa.cuda(), fb.cuda())
        corr, deltas = (r if reloc > 1 else (r, None))
        _check(corr.cpu()[0, 0], torch.from_numpy(gold[f'ff_r{reloc}_corr'][0, 0]).double())
        if reloc > 1:
            clear = _clear_boxes(fa[0], fb[0], reloc)
            for n, d in zip('ijkl', deltas):
                assert str(d.dtype) == str(gold[f'ff_r{reloc}_d{n}_dtype'])
                assert np.array_equal(d.cpu()[0, 0].numpy()[clear.numpy()], gold[f'ff_r{reloc}_d{n}'][0, 0][clear.numpy()])
        # (d) on the reference's own corr4d / delta4d, so that rows are comparable exactly
        gcorr = torch.from_numpy(gold[f'ff_r{reloc}_corr']).cuda()
        gd = tuple(torch.from_numpy(gold[f'ff_r{reloc}_d{n}']).cuda() for n in 'ijkl') if reloc > 1 else None
        for inv, scale, ri in K.C2M_ARGS:
            key = K.c2m_key(reloc, inv, scale, ri)
            got = corr_to_matches(gcorr, gd, ksize=max(reloc, 1), scale=scale, invert_matching_direction=inv,
                                  return_indices=ri)
            assert [str(t.dtype) for t in got] == list(gold[f'{key}_dtypes']), key
            ok = ~_tie_rows(gcorr[0, 0].cpu(), inv)
            assert ok.float().mean() > 0.9
            for n, t in zip(('a0', 'a1', 'a2', 'a3'), got[:4]):
                t, e = t.cpu()[0].numpy(), gold[f'{key}_{n}'][0]
                if ri:
                    assert np.array_equal(t[ok.numpy()], e[ok.numpy()]), key
                else:
                    np.testing.assert_allclose(t[ok.numpy()], e[ok.numpy()], rtol=0, atol=1e-7)
            np.testing.assert_allclose(got[4].cpu()[0].numpy(), gold[f'{key}_score'][0], rtol=1e-5, atol=1e-7)
        # ImMatchNet's delta tuple and the reference's float / int64 one give the same rows
        if reloc > 1:
            a = corr_to_matches(corr, deltas, ksize=2)
            b = corr_to_matches(corr, tuple(d.long() for d in deltas), ksize=2)
            assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_forward_from_seeded_checkpoint_file_vs_reference_golden(tmp_path):
    """(c): a checkpoint in the reference's file format ('vgg' key prefix, NC configuration in args), then forward()
    on CUDA images with no explicit .cuda() of the model, as INTEGRATION.md shows."""
    from argparse import Namespace
    from patch2pix_b200 import synth
    from patch2pix_b200.ncnet import ImMatchNet
    K, gold = _gold()
    ks, ch = K.CKPT_STACK
    names = [(k, tuple(v.shape)) for k, v in ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch).state_dict().items()]
    sd = synth.ncnet_state_dict(K.CKPT_SEED, names, ks, ch)
    sd = {k.replace('FeatureExtraction.model', 'FeatureExtraction.vgg'): v for k, v in sd.items()}
    path = str(tmp_path / 'ncnet.pth.tar')
    torch.save({'state_dict': sd, 'args': Namespace(ncons_kernel_sizes=ks, ncons_channels=ch)}, path)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = ImMatchNet(checkpoint=path, relocalization_k_size=2)
        ia, ib = synth.ncnet_images(K.IMG_SEED, *K.IMG_SIZES)
        corr, deltas = net({'source_image': ia.cuda(), 'target_image': ib.cuda()})
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    assert [d.dtype for d in deltas] == [torch.float32] * 3 + [torch.int64]
    # the backbone is cuDNN fp32 here and CPU fp32 in the reference: their features differ in the last bits
    ref = torch.from_numpy(gold['fwd_corr'][0, 0]).double()
    scale = ref.abs().max().item()
    np.testing.assert_allclose(corr.cpu()[0, 0].double().numpy(), ref.numpy(), rtol=1e-3, atol=1e-4 * scale)
    clear = gold['fwd_delta_clear']
    for n, d in zip('ijkl', deltas):
        assert np.array_equal(d.cpu()[0, 0].numpy()[clear], gold[f'fwd_d{n}'][0, 0][clear]), n
