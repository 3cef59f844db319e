"""The NCNet golden cases (tests/golden/ncnet_golden.npz): every input and weight is regenerated from these seeds by
patch2pix_b200.synth, so the fixture stores only the live reference's outputs."""

# (a) NeighConsensus stacks: (kernel sizes, channels, weight seed), run symmetric and not on each volume
NC_STACKS = [([3, 3, 3], [10, 10, 1], 31), ([5, 5, 5], [16, 16, 1], 32), ([3, 5], [8, 1], 33), ([5], [1], 34)]
NC_VOLUMES = [((3, 4, 2, 6), 41), ((4, 2, 5, 3), 42)]          # (hA, wA, hB, wB), input seed; dimensions below k
# (b) forward_feat: C = 1024 feature maps of different sizes, NC stack [3, 3, 3] / [10, 10, 1]
FEAT_SEED, FEAT_C, FEAT_SIZES = 51, 1024, ((8, 10), (12, 6))
FEAT_STACK = ([3, 3, 3], [10, 10, 1], 52)
RELOCS = (0, 2)
# (c) forward from a seeded checkpoint in the reference's file format
CKPT_SEED, CKPT_STACK = 61, ([3, 3], [16, 1])
IMG_SEED, IMG_SIZES = 62, ((192, 256), (160, 224))
# (d) corr_to_matches on the (b) outputs: both directions, both scales, both return_indices, with and without deltas
C2M_ARGS = [(inv, scale, ri) for inv in (False, True) for scale in ('positive', 'centered') for ri in (True, False)]


def c2m_key(reloc, inv, scale, ri):
    return f'c2m_r{reloc}_{"inv" if inv else "fwd"}_{scale}_{"idx" if ri else "xy"}'
