"""float64 restatement of NCNet's corr_to_matches_topk (the reference's networks/ncn/extract_ncmatches.py) for checking
the CUDA path (topk.cu).  Written from the operation's definition, with this library's tie rule: ranks follow a stable
sort of (-raw value, flat index), so exact ties go to the lowest index."""
import torch


def corr_to_matches_topk(corr, deltas=None, topk=1, ksize=1, do_softmax=True, invert=False):
    """corr [hA, wA, hB, wB] -> (jA, iA, jB, iB, score), each [topk * N]: for every B cell (every A cell with invert)
    the topk cells of the other image, ranked by a stable sort of (-raw value, flat index) -- value descending, exact
    ties to the lowest index -- with the (softmax-normalised over those cells) value as score.  Forward output is
    rank-major (rank r of B cell s at r * N + s), inverted cell-major (s * topk + r).  Indices are refined by the
    maxpool offsets (index * ksize + delta)."""
    hA, wA, hB, wB = corr.shape
    v = corr.double().reshape(hA * wA, hB * wB)
    if invert:
        v = v.t()
    n_slice, n = v.shape
    if not 1 <= topk <= n_slice:
        raise RuntimeError('selected index k out of range')
    order = torch.sort(-v, dim=0, stable=True).indices[:topk]            # [topk, N]
    p = torch.softmax(v, 0) if do_softmax else v
    score = torch.gather(p, 0, order)
    mine = torch.arange(n).expand(topk, n)
    a, bcell = (mine, order) if invert else (order, mine)
    if invert:                                                            # cell-major
        a, bcell, score = a.t(), bcell.t(), score.t()
    a, bcell, score = a.reshape(-1), bcell.reshape(-1), score.reshape(-1)
    iA, jA, iB, jB = a // wA, a % wA, bcell // wB, bcell % wB
    if deltas is not None:
        d = [t.reshape(hA, wA, hB, wB)[iA, jA, iB, jB].long() for t in deltas]
        iA, jA, iB, jB = iA * ksize + d[0], jA * ksize + d[1], iB * ksize + d[2], jB * ksize + d[3]
    return jA, iA, jB, iB, score
