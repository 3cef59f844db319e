"""Generate tests/golden/nonfinite_golden.npz by running the LIVE reference's corr_to_matches
(networks/ncn/extract_ncmatches.py) on the CPU, on correlation volumes with NaN, +inf and -inf cells and slices.

Run where the reference is checked out (it does not travel with the repository):
    python tests/golden/make_nonfinite_golden.py [/path/to/reference]
The reference is imported unmodified, by main() only: the tests import this module for its cases.  The volumes and
deltas are stored in the file too (vol_<case>, delta_<case>_<i|j|k|l>).  Keys of the outputs:
nonfinite_key(case, inv, sm, ks, ri) + '_a0' .. '_a3' / '_score'.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

SHAPE = (2, 1, 4, 5, 3, 6)          # b, 1, hA, wA, hB, wB
CASES = ('nan_cell', 'nan_slice', 'ninf_slice', 'pinf_cell')
ARGS = [(inv, sm, ks, ri) for inv in (False, True) for sm in (True, False) for ks in (1, 2) for ri in (True, False)]


def nonfinite_key(case, inv, sm, ks, ri):
    return f'{case}_{"inv" if inv else "fwd"}_{"sm" if sm else "raw"}_k{ks}_{"idx" if ri else "xy"}'


def volume(case, seed):
    """[b, 1, hA, wA, hB, wB] float32: uniform [0, 1) with the case's non-finite cells.  Every case marks cells of
    both batch items, so that B-cell slices (the forward direction) and A-cell slices (inverted) are both hit."""
    g = torch.Generator().manual_seed(seed)
    v = torch.rand(*SHAPE, generator=g)
    if case == 'nan_cell':          # one NaN cell each: a first-NaN within a finite slice, both directions
        v[0, 0, 1, 2, 2, 3] = float('nan')
        v[1, 0, 3, 4, 0, 0] = float('nan')
    elif case == 'nan_slice':       # B cell (1, 4) NaN over all of A; A cell (2, 1) NaN over all of B
        v[0, 0, :, :, 1, 4] = float('nan')
        v[1, 0, 2, 1, :, :] = float('nan')
        v[1, 0, 0, 0, 2, 5] = float('nan')
    elif case == 'ninf_slice':      # masked cells: whole slices of -inf, and slices that are -inf but for one cell
        v[0, 0, :, :, 0, 0] = -float('inf')
        v[0, 0, 3, :, :, :] = -float('inf')
        v[1, 0, :, :, 2, 2] = -float('inf')
        v[1, 0, 1, 3, 2, 2] = 0.5
        v[1, 0, 0, 0, :, :] = -float('inf')
    elif case == 'pinf_cell':       # one +inf cell each, and a slice with two +inf (ties to the lower index)
        v[0, 0, 2, 2, 1, 1] = float('inf')
        v[1, 0, 0, 3, 2, 4] = float('inf')
        v[1, 0, 3, 1, 2, 4] = float('inf')
    else:
        raise ValueError(case)
    return v


def deltas(seed, ks):
    """The reference's delta4d: four int64 [b, 1, hA, wA, hB, wB] tensors of offsets in [0, ks)."""
    g = torch.Generator().manual_seed(seed)
    return tuple(torch.randint(0, ks, SHAPE, generator=g) for _ in range(4))


def main():
    sys.path.insert(0, sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
    warnings.filterwarnings('ignore')
    from networks.ncn.extract_ncmatches import corr_to_matches
    out = {}
    torch.set_grad_enabled(False)
    for ci, case in enumerate(CASES):
        v = volume(case, 900 + ci)
        d = deltas(950 + ci, 2)
        out[f'vol_{case}'] = v.numpy()
        for n, t in zip('ijkl', d):
            out[f'delta_{case}_{n}'] = t.numpy()
        for inv, sm, ks, ri in ARGS:
            res = corr_to_matches(v, delta4d=d if ks > 1 else None, ksize=ks, do_softmax=sm, scale='positive',
                                  invert_matching_direction=inv, return_indices=ri)
            key = nonfinite_key(case, inv, sm, ks, ri)
            for n, t in zip(('a0', 'a1', 'a2', 'a3', 'score'), res):
                out[f'{key}_{n}'] = t.detach().numpy()
    np.savez_compressed(os.path.join(HERE, 'nonfinite_golden.npz'), **out)
    print('wrote', os.path.join(HERE, 'nonfinite_golden.npz'), len(out), 'arrays')


if __name__ == '__main__':
    main()
