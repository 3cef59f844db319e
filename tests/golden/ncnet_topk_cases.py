"""The corr_to_matches_topk golden cases (tests/golden/ncnet_topk_golden.npz).  Features and NeighConsensus weights are
regenerated from these seeds by patch2pix_b200.synth; the fixture stores the live reference's forward_feat outputs
(so that both sides rank identical volumes) and its corr_to_matches_topk outputs."""

# ImMatchNet.forward_feat on a batch of two different feature pairs (stacked), NC stack [3, 3, 3] / [10, 10, 1]
FEAT_SEEDS, FEAT_C, FEAT_SIZES = (81, 82), 1024, ((8, 10), (12, 6))
STACK = ([3, 3, 3], [10, 10, 1], 83)
RELOCS = (0, 2)
TOPKS = (1, 3, 16, 'all')                 # 'all' = the slice length
# delta tuple formats at relocalisation 2: ImMatchNet's (float, float, float, int64) and all-int64
DELTA_FORMATS = ('mixed', 'int64')


def cases(reloc):
    """-> [(key, invert, do_softmax, topk or 'all', delta format or None)]"""
    out = []
    for inv in (False, True):
        for sm in (True, False):
            for k in TOPKS:
                for fmt in (DELTA_FORMATS if reloc > 1 else (None,)):
                    key = f'topk_r{reloc}_{"inv" if inv else "fwd"}_{"sm" if sm else "raw"}_k{k}' + \
                          (f'_{fmt}' if fmt else '')
                    out.append((key, inv, sm, k, fmt))
    return out
