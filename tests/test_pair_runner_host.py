"""The evaluation protocols' shared pair-runner pieces (eval_helper): the decode-ahead generator, the matcher-row
check and the threshold-list check on the host; on the GPU, the device->host copies of eval_hpatches and
eval_relpose."""
import threading

import numpy as np
import pytest
import torch

from patch2pix_b200.eval_helper import MAX_THRESHOLDS, as_rows, check_thresholds, prefetch


# ---- prefetch ----------------------------------------------------------------------------------------------------------
def test_prefetch_in_order_one_item_ahead():
    started, yielded, worker = [], [], set()

    def load(x):
        worker.add(threading.get_ident())
        started.append(x)
        assert x <= len(yielded) + 1, 'a load ran more than one item ahead'
        return x * 10
    for i, got in prefetch(range(6), load):
        assert got == i * 10 and i == len(yielded)
        assert started[-1] <= i + 1
        yielded.append(i)
    assert yielded == list(range(6)) and started == list(range(6))
    assert worker and threading.get_ident() not in worker


def test_prefetch_passes_exceptions_through_and_continues():
    def load(x):
        if x == 2:
            raise KeyError('item 2')
        return x
    out = list(prefetch([0, 1, 2, 3], load))
    assert [i for i, _ in out] == [0, 1, 2, 3]
    assert isinstance(out[2][1], KeyError) and out[2][1].args == ('item 2',)
    assert [got for i, got in out if i != 2] == [0, 1, 3]


def test_prefetch_empty():
    assert list(prefetch([], lambda x: x)) == []


# ---- as_rows -----------------------------------------------------------------------------------------------------------
def test_as_rows_numpy_tensor_tuple_and_empty():
    m = np.arange(12, dtype=np.float32).reshape(3, 4)
    for out in (m, torch.from_numpy(m), (m, 'scores', 'coarse'), (torch.from_numpy(m).long(),), m.tolist()):
        r = as_rows(out, 'cpu')
        assert r.dtype == torch.float64 and r.is_contiguous() and r.shape == (3, 4)
        assert np.array_equal(r.numpy(), m.astype(np.float64))
    for empty in (np.zeros((0, 4)), np.zeros(0), [], torch.zeros(0, 2), (np.zeros((0, 4)), None)):
        assert as_rows(empty, 'cpu').shape == (0, 4)


@pytest.mark.parametrize('bad', [np.zeros((3, 5)), np.zeros(8), np.zeros((2, 2, 4)), torch.zeros(4, 3),
                                 (np.zeros((1, 2)),)])
def test_as_rows_rejects_other_shapes(bad):
    with pytest.raises(ValueError, match=r'\[N, 4\]'):
        as_rows(bad, 'cpu')


# ---- check_thresholds --------------------------------------------------------------------------------------------------
def test_check_thresholds_accepts():
    t = check_thresholds(range(1, MAX_THRESHOLDS + 1))
    assert t.dtype == np.float64 and t.tolist() == list(range(1, 17))
    assert check_thresholds((5e-4,)).tolist() == [5e-4]
    assert MAX_THRESHOLDS == 16


@pytest.mark.parametrize('bad', [[], [2, 1], [1, 1], [0, 1], [-1], [1, float('nan')], [1, float('inf')],
                                 list(range(1, 18))])
def test_check_thresholds_rejects(bad):
    with pytest.raises(ValueError, match='h_thresholds must be 1..16'):
        check_thresholds(bad, 'h_thresholds')


# ---- device->host copies of the protocols ------------------------------------------------------------------------------
def _dtoh(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if 'Memcpy DtoH' in e.name)


@pytest.fixture(scope='module')
def net():
    from patch2pix_b200.eval_helper import load_model
    from patch2pix_b200.synth import make_seeded_state_dict
    return load_model(make_seeded_state_dict(0, nc_init='consensus'))


def _matcher_copies(net, path0, path1):
    """Device->host copies of one match_device call of the net (the mutual-match count it reads)."""
    from patch2pix_b200.eval_helper import PairRunner
    run = PairRunner(net, 2, 'fine', 0.25, 0.0, 1024)
    a, b = run.prepare(run.decode([path0])[0]), run.prepare(run.decode([path1])[0])
    run.match(a, b)
    return _dtoh(lambda: run.match(a, b))


@pytest.mark.gpu
def test_hpatches_device_to_host_copies(net, tmp_path):
    from patch2pix_b200 import hpatches as HP
    from patch2pix_b200.synth import synthetic_hpatches_tree
    root = str(tmp_path)
    synthetic_hpatches_tree(root, 3, [('i_a', (200, 150)), ('v_b', (176, 144))])
    seqs = HP.read_hpatches(root)
    n_pf = _matcher_copies(net, seqs[0].paths[0], seqs[0].paths[1])
    kw = dict(ksize=2, io_thres=0.25, imsize=1024, lprint_=lambda s: None)
    HP.eval_hpatches(net, root, **kw)                                # warm-up
    n = _dtoh(lambda: HP.eval_hpatches(net, root, **kw))
    assert n_pf >= 1 and n == 10 * n_pf + 1, (n_pf, n)


@pytest.mark.gpu
def test_relpose_device_to_host_copies(net, tmp_path):
    from patch2pix_b200 import relpose as RP
    from patch2pix_b200.synth import synthetic_relpose_tree
    root = str(tmp_path)
    path, _ = synthetic_relpose_tree(root, 5, 4)
    pairs = RP.read_pairs(path, root)
    n_pf = _matcher_copies(net, pairs[0].path0, pairs[0].path1)
    kw = dict(ksize=2, io_thres=0.25, imsize=1024, chunk_pairs=2, lprint_=lambda s: None)
    RP.eval_relpose(net, pairs, root, **kw)                          # warm-up
    n = _dtoh(lambda: RP.eval_relpose(net, pairs, root, **kw))
    assert n_pf >= 1 and n == len(pairs) * n_pf + 1, (n_pf, n)
