"""CPU checks of the NCNet matcher: the float64 oracle against direct definitions, checkpoint parsing, argument
rejections, and a ptxas guard for the stack kernels in nc_stack.cu."""
import os
import re
import shutil
import subprocess
from argparse import Namespace

import pytest
import torch

from oracle import ncnet_oracle as O


def _stack(ks, ch, seed):
    g = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for i, (k, c) in enumerate(zip(ks, ch)):
        cin = 1 if i == 0 else ch[i - 1]
        ws.append((torch.rand(k, c, cin, k, k, k, generator=g, dtype=torch.float64) - 0.35) / (cin * k ** 4) ** 0.5)
        bs.append(0.05 * torch.randn(c, generator=g, dtype=torch.float64))
    return ws, bs


def _conv4d_pointwise(x, W, b, o, a, bb, c, d):
    """One output value of the 'same' 4D cross-correlation straight from its definition."""
    k = W.shape[0]
    p = k // 2
    cin, hA, wA, hB, wB = x.shape
    s = float(b[o])
    for i in range(cin):
        for t1 in range(k):
            for t2 in range(k):
                for t3 in range(k):
                    for t4 in range(k):
                        y = (a + t1 - p, bb + t2 - p, c + t3 - p, d + t4 - p)
                        if all(0 <= y[j] < n for j, n in enumerate((hA, wA, hB, wB))):
                            s += float(W[t1, o, i, t2, t3, t4]) * float(x[i, y[0], y[1], y[2], y[3]])
    return s


@pytest.mark.parametrize('k', [3, 5])
def test_oracle_conv4d_matches_its_definition(k):
    g = torch.Generator().manual_seed(k)
    x = torch.rand(2, 3, 4, 2, 5, generator=g, dtype=torch.float64)
    W = torch.randn(k, 3, 2, k, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(3, generator=g, dtype=torch.float64)
    out = O.conv4d(x, W, b)
    for idx in [(0, 0, 0, 0, 0), (1, 2, 3, 1, 4), (2, 1, 2, 0, 2), (0, 2, 0, 1, 3)]:
        assert abs(out[idx].item() - _conv4d_pointwise(x, W, b, *idx)) < 1e-10


def test_oracle_symmetric_stack_is_transpose_invariant():
    """stack(x) + stack(x^T)^T: transposing the input transposes the output."""
    ws, bs = _stack([3, 5], [4, 1], 1)
    x = torch.rand(3, 4, 5, 2, dtype=torch.float64)
    a = O.nc_stack(x, ws, bs, True)
    b = O.nc_stack(x.permute(2, 3, 0, 1), ws, bs, True).permute(2, 3, 0, 1)
    assert torch.allclose(a, b, rtol=0, atol=1e-12)


def test_oracle_maxpool4d_first_maximum_and_mutual():
    x = torch.zeros(4, 4, 2, 2, dtype=torch.float64)
    x[1, 0, 1, 1] = 2.0
    x[0, 1, 0, 0] = 2.0      # same box, earlier in row-major order of (di, dj, dk, dl): (0, 1, 0, 0) < (1, 0, 1, 1)
    m, di, dj, dk, dl = O.maxpool4d(x, 2)
    assert m[0, 0, 0, 0] == 2.0 and (di[0, 0, 0, 0], dj[0, 0, 0, 0], dk[0, 0, 0, 0], dl[0, 0, 0, 0]) == (0, 1, 0, 0)
    y = torch.rand(2, 3, 4, 1, dtype=torch.float64)
    v = y.reshape(6, 4)
    ref = v * (v / (v.max(1, keepdim=True).values + 1e-5)) * (v / (v.max(0, keepdim=True).values + 1e-5))
    assert torch.allclose(O.mutual(y).reshape(6, 4), ref)


def test_neigh_consensus_rejects_unsupported_stacks():
    from patch2pix_b200.ncnet import NeighConsensus
    for ks, ch in (([4, 3], [8, 1]), ([7], [1]), ([3, 3], [17, 1]), ([3, 3], [0, 1]), ([3, 3], [8, 2]), ([3], [1, 1]),
                   ([], [])):
        with pytest.raises(ValueError):
            NeighConsensus(kernel_sizes=ks, channels=ch)
    with pytest.raises(ValueError):
        NeighConsensus(use_cuda=False, kernel_sizes=[3], channels=[1])
    nc = NeighConsensus(kernel_sizes=[3, 5, 3], channels=[10, 16, 1])
    names = [k for k in nc.state_dict()]
    assert names == ['conv.0.weight', 'conv.0.bias', 'conv.2.weight', 'conv.2.bias', 'conv.4.weight', 'conv.4.bias']
    assert tuple(nc.state_dict()['conv.2.weight'].shape) == (5, 16, 10, 5, 5, 5)
    with pytest.raises(NotImplementedError):
        nc.train()


def test_immatchnet_rejects_unsupported_options():
    from patch2pix_b200.ncnet import ImMatchNet
    bad = [dict(feature_extraction_cnn='vgg'), dict(feature_extraction_cnn='densenet201'),
           dict(feature_extraction_cnn='resnet101fpn'), dict(half_precision=True), dict(use_cuda=False),
           dict(train_fe=True), dict(relocalization_k_size=3), dict(ncons_kernel_sizes=[3, 4], ncons_channels=[8, 1])]
    for kw in bad:
        with pytest.raises(ValueError):
            ImMatchNet(**kw)


def test_immatchnet_without_weights_refuses_to_run():
    from patch2pix_b200.ncnet import ImMatchNet
    net = ImMatchNet(ncons_kernel_sizes=[3, 3], ncons_channels=[4, 1])
    with pytest.raises(RuntimeError, match='no weights'):
        net.forward_feat(torch.zeros(1, 64, 2, 2), torch.zeros(1, 64, 2, 2))
    with pytest.raises(NotImplementedError):
        net.train()


def test_immatchnet_checkpoint_in_the_reference_format(tmp_path):
    """state_dict keys with the old 'vgg' prefix, NC configuration from checkpoint['args']."""
    from patch2pix_b200.ncnet import ImMatchNet
    src = ImMatchNet(ncons_kernel_sizes=[5, 3], ncons_channels=[6, 1])
    g = torch.Generator().manual_seed(3)
    sd = {k.replace('FeatureExtraction.model', 'FeatureExtraction.vgg'): torch.rand(v.shape, generator=g)
          if v.is_floating_point() else v for k, v in src.state_dict().items()}
    path = tmp_path / 'ncnet.pth.tar'
    torch.save({'state_dict': sd, 'args': Namespace(ncons_kernel_sizes=[5, 3], ncons_channels=[6, 1])}, str(path))
    net = ImMatchNet(checkpoint=str(path), relocalization_k_size=2)
    assert net.NeighConsensus.kernel_sizes == [5, 3] and net.NeighConsensus.channels == [6, 1]
    got = net.state_dict()
    for k, v in sd.items():
        k2 = k.replace('vgg', 'model')
        if 'num_batches_tracked' not in k2:
            assert torch.equal(got[k2], v), k2
    assert net._loaded


def test_nc_stack_kernels_pipeline_wgmma_without_spills(tmp_path):
    """Compiled as the library is: no ptxas "wgmma serialized" advisory, no spills, the expected kernels."""
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'nc_stack.cu'),
                                   '-o', str(tmp_path / 'nc_stack.o')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-2000:]
    assert not [ln for ln in log.splitlines() if re.search(r'C75\d\d|wgmma.*serializ', ln)], log
    spills, cur = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', ln)
        if m and cur is not None:
            spills[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    layer = [k for k in spills if 'nc_stack_layer_kernel' in k]
    assert len(layer) == 4, sorted(spills)          # k in {3, 5} x {one net, symmetric pair}
    assert not {k: v for k, v in spills.items() if v}, spills


# ---- the oracle against the live reference's outputs (tests/golden/ncnet_golden.npz, make_ncnet_golden.py) ----------
import importlib.util  # noqa: E402

import numpy as np  # noqa: E402

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _cases():
    spec = importlib.util.spec_from_file_location('ncnet_cases', os.path.join(GOLD_DIR, 'ncnet_cases.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


K = _cases()


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD_DIR, 'ncnet_golden.npz')))


def _close(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    scale = max(np.abs(ref).max(), 1e-30)
    np.testing.assert_allclose(np.asarray(got, dtype=np.float64), ref, rtol=2e-4, atol=5e-6 * scale)


def test_oracle_nc_stacks_vs_reference(gold):
    from patch2pix_b200 import synth
    for ks, ch, wseed in K.NC_STACKS:
        ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
        for sym in (True, False):
            for shape, xseed in K.NC_VOLUMES:
                g = torch.Generator().manual_seed(xseed)
                x = torch.rand(1, 1, *shape, generator=g) - 0.1
                ref = gold[f'nc_{"_".join(map(str, ks))}_{"_".join(map(str, ch))}_{int(sym)}_{xseed}']
                _close(O.nc_stack(x[0, 0], ws, bs, sym).numpy(), ref)


def test_oracle_forward_feat_and_corr_to_matches_vs_reference(gold):
    from patch2pix_b200 import synth
    ks, ch, wseed = K.FEAT_STACK
    ws, bs = synth.ncnet_stack_weights(wseed, ks, ch)
    fa, fb = synth.ncnet_features(K.FEAT_SEED, K.FEAT_C, *K.FEAT_SIZES)
    for reloc in K.RELOCS:
        corr, deltas = O.forward_feat(fa[0], fb[0], ws, bs, reloc if reloc > 1 else 1)
        _close(corr.numpy(), gold[f'ff_r{reloc}_corr'][0, 0])
        if reloc > 1:
            for n, d in zip('ijkl', deltas):
                assert np.array_equal(d.numpy(), gold[f'ff_r{reloc}_d{n}'][0, 0]), n
            assert [str(gold[f'ff_r{reloc}_d{n}_dtype']) for n in 'ijkl'] == ['torch.float32'] * 3 + ['torch.int64']
        gcorr = torch.from_numpy(gold[f'ff_r{reloc}_corr'][0, 0])
        gd = [torch.from_numpy(gold[f'ff_r{reloc}_d{n}'][0, 0]) for n in 'ijkl'] if reloc > 1 else None
        for inv, scale, ri in K.C2M_ARGS:
            key = K.c2m_key(reloc, inv, scale, ri)
            got = O.corr_to_matches(gcorr, gd, max(reloc, 1), True, scale, inv, ri)
            assert list(gold[f'{key}_dtypes']) == (['torch.int64'] * 4 if ri else ['torch.float32'] * 4) + \
                ['torch.float32']
            for n, t in zip(('a0', 'a1', 'a2', 'a3'), got[:4]):
                if ri:
                    assert np.array_equal(t.numpy(), gold[f'{key}_{n}'][0]), key
                else:
                    np.testing.assert_allclose(t.numpy(), gold[f'{key}_{n}'][0], atol=1e-6)
            np.testing.assert_allclose(got[4].numpy(), gold[f'{key}_score'][0], rtol=1e-5)


def test_oracle_forward_from_seeded_checkpoint_vs_reference(gold):
    """(c): the seeded checkpoint's ResNet101 layer3 (this package's torchvision backbone, CPU) + the oracle."""
    from patch2pix_b200 import synth
    from patch2pix_b200.ncnet import ImMatchNet
    ks, ch = K.CKPT_STACK
    net = ImMatchNet(ncons_kernel_sizes=ks, ncons_channels=ch, relocalization_k_size=2)
    sd = synth.ncnet_state_dict(K.CKPT_SEED, [(k, tuple(v.shape)) for k, v in net.state_dict().items()], ks, ch)
    net.load_state_dict(sd)
    fe = net.FeatureExtraction.cpu().eval()
    ia, ib = synth.ncnet_images(K.IMG_SEED, *K.IMG_SIZES)
    with torch.no_grad():
        fa, fb = fe(ia), fe(ib)
    ws = [sd[f'NeighConsensus.conv.{2 * i}.weight'] for i in range(len(ks))]
    bs = [sd[f'NeighConsensus.conv.{2 * i}.bias'] for i in range(len(ks))]
    corr, deltas = O.forward_feat(fa[0], fb[0], ws, bs, 2)
    _close(corr.numpy(), gold['fwd_corr'][0, 0])
    clear = gold['fwd_delta_clear']
    assert clear.sum() >= 200             # boxes whose maximum leads the runner-up by > 1e-4 (relative)
    for n, d in zip('ijkl', deltas):
        assert np.array_equal(d.numpy()[clear], gold[f'fwd_d{n}'][0, 0][clear]), n

