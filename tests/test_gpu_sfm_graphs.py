"""The track and triangulation stages of csrc/sfm.cu driven directly through p2p_sfm_tracks / p2p_sfm_triangulate, on
match graphs and scenes built here so that their shape is controlled, against oracle/sfm_oracle.py (and scipy for the
connected components).

Graphs: paths of 2^20 keypoints in bit-reversed and in random id order (the slow cases for min-label hooking: on the
bit-reversed path each hook round only halves the number of roots), a star whose hub has the largest id, 10^6 random
edges with duplicate edges, self-edges and invalid endpoints, many 2-node components, a forest of random trees of
1 to 20000 keypoints, empty graphs, and components at and one past the 2^16-observation cap.  The paths, the star and
the random graph are each one component over the cap: they check the labels, the forest and the others the tracks.
Every match is built through kp_of_ep / offsets / E / thr with a random, non-degenerate E per pair and a huge finite
threshold, so every first-in-pair match with two different keypoints is an edge; the test checks each Sampson
denominator is non-zero and each ratio is below the threshold.

Scene: a non-planar cloud seen by 30 SIMPLE_RADIAL / RADIAL images, tracks with 1 to 10 points (so rounds 1-8 each
accept one and a 9th would), two observations in one image, points behind the cameras, baselines below min_angle,
tied hypothesis scores, tracks longer than one triangulation block of 128 threads, and outlier observations.

The hook stage's host loop runs 16 hook / jump / converge rounds per host check, and every launch the library makes
is counted (p2p_launch_count): each further batch adds 48 launches, so the launch count says how many batches a graph
needed, though not how many of a batch's rounds did work."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import sfm_oracle as O

HOOK_BATCH_LAUNCHES = 16 * 3        # hook, jump, converge per round, 16 rounds per host check
REPROJ_PX, MIN_ANGLE = 4.0, 1.5
TRI_THREADS = 128                   # threads of one triangulation block (csrc/sfm.cu kTriThreads)


# ---- graphs ----------------------------------------------------------------------------------------------------------
def bitrev_order(bits):
    """Ids 0 .. 2^bits - 1 with their bits reversed, in counting order."""
    k = np.arange(1 << bits, dtype=np.int64)
    r = np.zeros_like(k)
    for b in range(bits):
        r |= ((k >> b) & 1) << (bits - 1 - b)
    return r


def random_offsets(M, mean, rng):
    """Pair offsets [P + 1] over M matches with pair sizes uniform in 0 .. 2 mean (empty pairs included)."""
    sizes = []
    while sum(sizes) < M:
        sizes.append(int(rng.integers(0, 2 * mean + 1)))
    off = np.concatenate([[0], np.minimum(np.cumsum(sizes), M)]).astype(np.int64)
    return off if len(off) > 1 else np.zeros(2, np.int64)


def packed_offsets(ka, kb, mean, rng):
    """Pair offsets over the matches in order, sizes up to uniform in 1 .. 2 mean, a pair closed early where a
    keypoint would repeat on its side: every match is first in its pair for both keypoints."""
    off, a, b, cap = [0], set(), set(), int(rng.integers(1, 2 * mean + 1))
    for m, (x, y) in enumerate(zip(ka.tolist(), kb.tolist())):
        if m - off[-1] == cap or x in a or y in b:
            off.append(m)
            a, b, cap = set(), set(), int(rng.integers(1, 2 * mean + 1))
        a.add(x)
        b.add(y)
    return np.array(off + [len(ka)], np.int64)


def graph_inputs(ka, kb, n_kp, offsets, rng):
    """The track stage's inputs that make (ka[m], kb[m]) match m: one random E per pair, thr 1e300, kp_n uniform in
    [-1, 1]^2."""
    ka, kb = np.asarray(ka, np.int64), np.asarray(kb, np.int64)
    assert ka.shape == kb.shape and offsets[0] == 0 and offsets[-1] == len(ka) and np.all(np.diff(offsets) >= 0)
    assert np.all((ka >= -1) & (ka < n_kp) & (kb >= -1) & (kb < n_kp))
    P = len(offsets) - 1
    return dict(kp_of_ep=np.stack([ka, kb], 1).reshape(-1).astype(np.int32), offsets=np.asarray(offsets, np.int64),
                E=rng.normal(size=(P, 9)), thr=np.full(P, 1e300), kp_n=rng.uniform(-1, 1, (max(n_kp, 1), 2)),
                n_kp=int(n_kp))


def _first(pair, k):
    """first[m]: match m is the first of its pair, in match order, with its keypoint k[m] (k[m] >= 0)."""
    out = np.zeros(len(k), bool)
    idx = np.nonzero(k >= 0)[0]
    _, first = np.unique((pair[idx] << 32) | k[idx], return_index=True)
    out[idx[first]] = True
    return out


def sampson(inp, m):
    """(numerator^2, denominator) of the Sampson ratio of matches m, in the kernel's order of operations."""
    ka, kb = inp['kp_of_ep'][0::2][m], inp['kp_of_ep'][1::2][m]
    pair = np.repeat(np.arange(len(inp['offsets']) - 1), np.diff(inp['offsets']))[m]
    e = inp['E'][pair].T
    a0, a1 = inp['kp_n'][ka, 0], inp['kp_n'][ka, 1]
    b0, b1 = inp['kp_n'][kb, 0], inp['kp_n'][kb, 1]
    e0 = e[0] * a0 + e[1] * a1 + e[2]
    e1 = e[3] * a0 + e[4] * a1 + e[5]
    e2 = e[6] * a0 + e[7] * a1 + e[8]
    f0 = e[0] * b0 + e[3] * b1 + e[6]
    f1 = e[1] * b0 + e[4] * b1 + e[7]
    num = b0 * e0 + b1 * e1 + e2
    return num * num, e0 * e0 + e1 * e1 + f0 * f0 + f1 * f1


def expected_edges(inp):
    """The edge rule of sfm_oracle.edges, vectorised for graphs of 10^6 matches, with every Sampson test asserted to
    pass -> unique edges [k, 2] sorted, count of first-in-pair matches."""
    ka, kb = inp['kp_of_ep'][0::2].astype(np.int64), inp['kp_of_ep'][1::2].astype(np.int64)
    pair = np.repeat(np.arange(len(inp['offsets']) - 1, dtype=np.int64), np.diff(inp['offsets']))
    both = _first(pair, ka) & _first(pair, kb)
    m = np.nonzero(both)[0]
    num2, den = sampson(inp, m)
    assert np.all(den != 0.0), 'a Sampson denominator is zero'
    with np.errstate(over='ignore'):
        assert np.all(num2 / den <= inp['thr'][pair[m]]), 'a match fails the Sampson test'
    keep = m[ka[m] != kb[m]]
    e = np.stack([np.minimum(ka[keep], kb[keep]), np.maximum(ka[keep], kb[keep])], 1)
    return np.unique(e, axis=0).reshape(-1, 2), len(m)


def random_tree(ids, rng):
    """Edges of a random tree over ids (each node joins a random earlier node), random orientation."""
    ids = rng.permutation(np.asarray(ids, np.int64))
    if len(ids) < 2:
        return np.zeros((0, 2), np.int64)
    par = ids[(rng.random(len(ids) - 1) * np.arange(1, len(ids))).astype(np.int64)]
    e = np.stack([ids[1:], par], 1)
    flip = rng.random(len(e)) < 0.5
    e[flip] = e[flip][:, ::-1]
    return e


def path_graph(order, rng):
    e = np.stack([order[:-1], order[1:]], 1)
    return graph_inputs(e[:, 0], e[:, 1], len(order), random_offsets(len(e), 512, rng), rng)


def star_graph(leaves, rng):
    """Hub = the largest id; pairs of two matches with the hub on side 0 in one and on side 1 in the other."""
    hub = leaves
    leaf = rng.permutation(leaves)
    ka, kb = np.full(leaves, hub), leaf.copy()
    ka[1::2], kb[1::2] = leaf[1::2], hub
    off = np.append(np.arange(0, leaves, 2), leaves)
    return graph_inputs(ka, kb, leaves + 1, off, rng)


def random_multigraph(n_kp, M, rng):
    """M random matches over the keypoints not divisible by 97 (the others are touched by no match), then 10 % of them
    repeated reversed at random places, 1 % self-edges and 1 % invalid endpoints."""
    used = np.nonzero(np.arange(n_kp) % 97)[0]
    ka, kb = used[rng.integers(0, len(used), M)], used[rng.integers(0, len(used), M)]
    dup = rng.integers(0, M, M // 10)
    ka, kb = np.concatenate([ka, kb[dup]]), np.concatenate([kb, ka[dup]])
    perm = rng.permutation(len(ka))
    ka, kb = ka[perm], kb[perm]
    s = rng.integers(0, len(ka), len(ka) // 100)
    kb[s] = ka[s]
    ka[rng.integers(0, len(ka), len(ka) // 200)] = -1
    kb[rng.integers(0, len(kb), len(kb) // 200)] = -1
    return graph_inputs(ka, kb, n_kp, random_offsets(len(ka), 64, rng), rng)


def two_node_graph(n_kp, rng):
    """n_kp / 2 components of two keypoints each, every edge given twice: once per orientation, in different pairs."""
    p = rng.permutation(n_kp).reshape(-1, 2)
    ka, kb = np.concatenate([p[:, 0], p[:, 1]]), np.concatenate([p[:, 1], p[:, 0]])
    return graph_inputs(ka, kb, n_kp, random_offsets(len(ka), 300, rng), rng)


def forest_graph(n_kp, rng):
    """Random trees of 1 .. 20000 keypoints (log-uniform sizes) over n_kp shuffled ids: many tracks of every length."""
    sizes = []
    while sum(sizes) < n_kp:
        sizes.append(min(int(np.exp(rng.uniform(0, np.log(20000)))), n_kp - sum(sizes)))
    parts = np.split(rng.permutation(n_kp), np.cumsum(sizes)[:-1])
    e = np.concatenate([random_tree(p, rng) for p in parts])
    e = e[rng.permutation(len(e))]
    return graph_inputs(e[:, 0], e[:, 1], n_kp, packed_offsets(e[:, 0], e[:, 1], 128, rng), rng)


def first_in_pair_graph(rng):
    """Keypoints that repeat within a pair: pair 0 (0, 5) (0, 6) (1, 5) (2, 7) keeps (0, 5) and (2, 7); pair 1 (0, 6)
    (3, 3) (6, 4) (-1, 8) keeps (0, 6) and (4, 6); pair 2 (4, 6) (6, 4) repeats an edge both ways."""
    ka = [0, 0, 1, 2, 0, 3, 6, -1, 4, 6]
    kb = [5, 6, 5, 7, 6, 3, 4, 8, 6, 4]
    return graph_inputs(ka, kb, 10, np.array([0, 4, 8, 10]), rng)


def cap_graph(rng):
    """Components of 2^16 (kept), 2^16 + 1 and 70000 (both rejected) observations, 3000 of 2-5 and 500 keypoints
    alone, ids shuffled across all of them."""
    sizes = [O.MAX_TRACK, O.MAX_TRACK + 1, 70000] + list(rng.integers(2, 6, 3000)) + [1] * 500
    ids = rng.permutation(int(sum(sizes)))
    parts = np.split(ids, np.cumsum(sizes)[:-1])
    e = np.concatenate([random_tree(p, rng) for p in parts])
    e = e[rng.permutation(len(e))]
    return graph_inputs(e[:, 0], e[:, 1], len(ids), packed_offsets(e[:, 0], e[:, 1], 256, rng), rng), parts


GRAPHS = {
    'bitrev_path': lambda rng: path_graph(bitrev_order(20), rng),
    'random_path': lambda rng: path_graph(rng.permutation(1 << 20), rng),
    'star': lambda rng: star_graph(100000, rng),
    'random_multigraph': lambda rng: random_multigraph(200000, 1000000, rng),
    'two_node': lambda rng: two_node_graph(200000, rng),
    'forest': lambda rng: forest_graph(1000000, rng),
    'first_in_pair': first_in_pair_graph,
}


def reference_tracks(inp):
    """sfm_oracle's components and tracks of inp -> labels, obs_kp, starts, lens, counts [6]."""
    edges, n_first = expected_edges(inp)
    labels = O.components(inp['n_kp'], edges.tolist())
    obs, tr, rej = O.tracks(labels)
    starts = np.array([s for s, _ in tr], np.int64)
    lens = np.array([n for _, n in tr], np.int64)
    return labels, obs, starts, lens, np.array([len(edges), len(tr), lens.sum(), rej, n_first, 0], np.int64), edges


def scipy_labels(n_kp, edges):
    """scipy's connected components, each labelled by its smallest keypoint id."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    if n_kp == 0:
        return np.zeros(0, np.int64)
    g = coo_matrix((np.ones(len(edges)), (edges[:, 0], edges[:, 1])), shape=(n_kp, n_kp))
    nc, lab = connected_components(g, directed=False)
    low = np.full(nc, n_kp, np.int64)
    np.minimum.at(low, lab, np.arange(n_kp))
    return low[lab]


# ---- scene -----------------------------------------------------------------------------------------------------------
def _look_at(C):
    z = -C / np.linalg.norm(C)
    x = np.cross(z, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z])
    t = -R @ C
    return np.concatenate([R.reshape(-1), t, C])


def project(rec, cam, X):
    """Pixels [n, 2] (distorted) and depths [n] of points X [n, 3]."""
    p = np.asarray(X, np.float64).reshape(-1, 3) @ rec[:9].reshape(3, 3).T + rec[9:12]
    with np.errstate(divide='ignore', invalid='ignore'):
        x, y = O.distort_px(cam, p[:, 0] / p[:, 2], p[:, 1] / p[:, 2])
    return np.stack([x, y], 1), p[:, 2]


def angle_deg(rec_a, rec_b, X):
    return math.degrees(math.acos(max(-1.0, min(1.0, O._cos_angle(rec_a, rec_b, X)))))


def build_scene(seed=0):
    """30 images: 28 on a ring of radius 10 around the cloud [-2, 2]^3 looking at its centre, and two more 2 cm beside
    images 0 and 10 (0.1 degree baselines).  6 cameras, SIMPLE_RADIAL and RADIAL.  Keypoints are projections with
    0.3 px noise, each track's keypoints given one group; groups[g] = (kind, meta)."""
    rng = np.random.default_rng(seed)
    ring = 28
    a = 2 * np.pi * np.arange(ring) / ring + rng.uniform(-0.05, 0.05, ring)
    Cs = np.stack([10 * np.cos(a), 10 * np.sin(a), rng.uniform(-1, 1, ring)], 1)
    recs = [_look_at(c) for c in Cs]
    for i in (0, 10):
        r = recs[i].copy()
        r[12:] = r[12:] + 0.02 * r[0:3]                  # 2 cm along the image's x axis
        r[9:12] = -r[:9].reshape(3, 3) @ r[12:]
        recs.append(r)
    recs = np.stack(recs)
    cams = np.array([[2, 900.0, 900.0, 512.0, 384.0, -0.05, 0.0, 0.0],
                     [3, 1000.0, 1000.0, 500.0, 380.0, -0.04, 0.01, 0.0],
                     [2, 1100.0, 1100.0, 520.0, 390.0, 0.03, 0.0, 0.0],
                     [3, 800.0, 800.0, 510.0, 370.0, 0.02, -0.01, 0.0],
                     [2, 950.0, 950.0, 505.0, 385.0, -0.02, 0.0, 0.0],
                     [3, 1050.0, 1050.0, 515.0, 395.0, -0.03, 0.02, 0.0]])
    img_cam = (np.arange(len(recs)) % len(cams)).astype(np.int32)
    cloud = rng.uniform(-2, 2, (1000, 3))
    kps, groups = [], []                                  # kps: (image, x, y, group)

    def add(g, img, X, noise=0.3, reps=1):
        out = []
        for _ in range(reps):
            xy, d = project(recs[img], cams[img_cam[img]], X)
            xy = xy[0] + rng.normal(0, noise, 2)
            out.append(len(kps))
            kps.append((img, xy[0], xy[1], g))
        return out

    def group(kind, **meta):
        groups.append((kind, meta))
        return len(groups) - 1
    free = iter(rng.permutation(len(cloud)))
    ring_px = lambda X: np.stack([project(recs[i], cams[img_cam[i]], X)[0][0] for i in range(ring)])
    # 1 .. 10 points per track, each in 3 ring images and at least 30 px from the track's other points in every ring
    # image (no point takes another's observations): rounds 1-8 each accept one, and a 9th would
    for K in range(1, 11):
        for _ in range(3):
            g = group('multi', K=K)
            placed = []
            while len(placed) < K:
                X = cloud[next(free)]
                px = ring_px(X)
                if any(np.min(np.linalg.norm(px - q, axis=1)) < 30 for q in placed):
                    continue
                placed.append(px)
                for img in rng.choice(ring, 3, replace=False):
                    add(g, img, X)
    # two observations in one image: no pair of different images
    for _ in range(10):
        g = group('one_image')
        img = int(rng.integers(ring))
        add(g, img, cloud[next(free)])
        add(g, img, cloud[next(free)])
    # a point behind both of its images (just outside the ring behind image i, also behind image i + 1)
    for i in (3, 12, 20):
        X = 1.3 * recs[i][12:]
        g = group('behind_all', X=X, imgs=(i, i + 1))
        add(g, i, X, noise=0.0)
        add(g, i + 1, X, noise=0.0)
    # a point behind image i but in front of images i +- 3 and i + 14: a point without the observation of image i
    for i in (5, 17):
        X = 1.15 * recs[i][12:]
        g = group('behind_one', X=X, behind=i)
        for img in sorted({i, (i + 3) % ring, (i - 3) % ring, (i + 14) % ring}):
            add(g, img, X)
    # baselines of 0.1 degree: images 0 and 28, 10 and 29 alone give no point; with a third image they do
    for i, j in ((0, 28), (10, 29)):
        for third in (None, (i + 5) % ring):
            X = cloud[next(free)]
            g = group('narrow' if third is None else 'narrow_wide', X=X, imgs=(i, j))
            for img in sorted({i, j} | ({third} if third is not None else set())):
                add(g, img, X, noise=0.0 if third is None else 0.3)
    # tied scores: points A and B, each exact in two images, A's images before B's; hypotheses (0, 1) and (2, 3) both
    # score 2 and the lower, A, must make the track's first point
    for _ in range(6):
        A, B = cloud[next(free)], cloud[next(free)]
        imgs = np.sort(rng.choice(ring, 4, replace=False))
        g = group('tie', A=A, B=B)
        add(g, imgs[0], A, noise=0.0)
        add(g, imgs[1], A, noise=0.0)
        add(g, imgs[2], B, noise=0.0)
        add(g, imgs[3], B, noise=0.0)
    # longer than one block: one point, 5 observations in each ring image; three points, 2 each; and outliers
    g = group('long', K=1, outliers=0)
    X = cloud[next(free)]
    for img in range(ring):
        add(g, img, X, noise=0.5, reps=5)
    g = group('long', K=3, outliers=12)
    for _ in range(3):
        X = cloud[next(free)]
        for img in range(ring):
            add(g, img, X, noise=0.5, reps=2)
    for _ in range(12):
        kps.append((int(rng.integers(ring)), rng.uniform(0, 1024), rng.uniform(0, 768), g))
    # keypoints in no track
    for _ in range(300):
        kps.append((int(rng.integers(len(recs))), rng.uniform(0, 1024), rng.uniform(0, 768), -1))
    # ids in image order, random within an image; track observations in id order keep each image's together
    img = np.array([k[0] for k in kps], np.int64)
    order = np.lexsort((rng.random(len(kps)), img))
    kp_img = img[order]
    rank = np.arange(len(kps)) - np.searchsorted(kp_img, kp_img)
    kp_key = (kp_img.astype(np.uint64) << np.uint64(44)) | rank.astype(np.uint64)
    kp_xy = np.array([(kps[o][1], kps[o][2]) for o in order])
    kp_group = np.array([kps[o][3] for o in order], np.int64)
    new_id = np.empty(len(kps), np.int64)
    new_id[order] = np.arange(len(kps))
    labels = np.arange(len(kps))
    for gid in range(len(groups)):
        m = kp_group == gid
        labels[m] = np.nonzero(m)[0].min()
    obs_kp, tracks, rej = O.tracks(labels)
    assert rej == 0
    kp_n = O.undistort_keypoints(kp_xy, kp_key, img_cam, cams)
    return dict(recs=recs, cams=cams, img_cam=img_cam, kp_xy=kp_xy, kp_key=kp_key, kp_n=kp_n, obs_kp=obs_kp,
                tracks=tracks, kp_group=kp_group, groups=groups)


def check_scene_structure(sc, points, point_len, kp_point):
    """The geometry each kind of track was built for, on a triangulation of the scene (the oracle's or the kernel's)."""
    recs, cams, img_cam = sc['recs'], sc['cams'], sc['img_cam']
    kp_img = (sc['kp_key'] >> np.uint64(44)).astype(np.int64)
    # every point within reproj_px of each of its observations; point_len counts them
    for p in range(len(points)):
        ks = np.nonzero(kp_point == p)[0]
        assert len(ks) == point_len[p] >= 2
        for k in ks:
            xy, d = project(recs[kp_img[k]], cams[img_cam[kp_img[k]]], points[p])
            assert d[0] > 0 and np.hypot(*(xy[0] - sc['kp_xy'][k])) <= REPROJ_PX * (1 + 1e-12), (p, k)
    seen = set()
    for gid, (kind, meta) in enumerate(sc['groups']):
        ks = np.nonzero(sc['kp_group'] == gid)[0]
        pts = np.unique(kp_point[ks][kp_point[ks] >= 0])
        seen.add(kind)
        if kind == 'multi':
            assert len(pts) == min(meta['K'], 8), (gid, meta['K'], len(pts))     # at most 8 rounds
            if meta['K'] > 8:
                assert np.sum(kp_point[ks] < 0) >= 2
        elif kind in ('one_image', 'behind_all', 'narrow'):
            assert len(pts) == 0, (kind, gid)
        elif kind == 'behind_one':
            assert len(pts) == 1
            behind = ks[kp_img[ks] == meta['behind']]
            assert len(behind) == 1 and kp_point[behind[0]] == -1
            assert np.linalg.norm(points[pts[0]] - meta['X']) < 0.05
        elif kind == 'narrow_wide':
            assert len(pts) == 1 and np.all(kp_point[ks] == pts[0])
        elif kind == 'tie':
            # points are numbered by round: A (hypothesis (0, 1)) first, then B
            assert len(pts) == 2 and kp_point[ks[0]] == kp_point[ks[1]] == pts[0] and \
                kp_point[ks[2]] == kp_point[ks[3]] == pts[1]
            assert np.linalg.norm(points[pts[0]] - meta['A']) < 1e-6 * 12
        elif kind == 'long':
            # outlier observations may pair into points of their own
            assert len(ks) > TRI_THREADS and (len(pts) == meta['K'] if meta['outliers'] == 0 else len(pts) >= meta['K'])
    assert seen == {'multi', 'one_image', 'behind_all', 'behind_one', 'narrow', 'narrow_wide', 'tie', 'long'}


@pytest.fixture(scope='module')
def scene():
    sc = build_scene(0)
    o, tr = sc['obs_kp'], sc['tracks']
    sc['ref'] = O.triangulate(o, tr, sc['kp_xy'], sc['kp_n'], sc['kp_key'], sc['recs'], sc['img_cam'], sc['cams'],
                              REPROJ_PX, MIN_ANGLE)
    return sc


# ---- host checks of the builders and the vectorised edge rule --------------------------------------------------------
def test_expected_edges_is_the_oracle_rule():
    rng = np.random.default_rng(1)
    for trial in range(20):
        n_kp, M = int(rng.integers(1, 30)), int(rng.integers(0, 80))
        ka, kb = rng.integers(-1, n_kp, M), rng.integers(-1, n_kp, M)
        inp = graph_inputs(ka, kb, n_kp, random_offsets(M, 6, rng), rng)
        edges, n_first = expected_edges(inp)
        ref, ref_first = O.edges(inp['kp_of_ep'].astype(np.int64), np.diff(inp['offsets']), inp['E'], inp['thr'],
                                 inp['kp_n'])
        assert [tuple(e) for e in edges.tolist()] == ref and n_first == ref_first, trial
    edges, n_first = expected_edges(first_in_pair_graph(rng))
    assert edges.tolist() == [[0, 5], [0, 6], [2, 7], [4, 6]] and n_first == 7


def test_graph_builders():
    rng = np.random.default_rng(2)
    o = bitrev_order(4)
    assert o.tolist() == [0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15]
    # paths: no keypoint repeats within a pair, so every match is an edge and the graph is the path
    inp = path_graph(bitrev_order(10), rng)
    edges, n_first = expected_edges(inp)
    assert n_first == len(edges) == 1023 and np.array_equal(scipy_labels(1024, edges), np.zeros(1024))
    inp = star_graph(1001, rng)
    edges, n_first = expected_edges(inp)
    assert n_first == len(edges) == 1001 and np.all(edges[:, 1] == 1001)
    inp = random_multigraph(2000, 10000, rng)
    ka, kb = inp['kp_of_ep'][0::2], inp['kp_of_ep'][1::2]
    edges, n_first = expected_edges(inp)
    assert np.sum(ka == kb) > 50 and np.sum(ka < 0) > 20 and np.sum(kb < 0) > 20
    keys = np.minimum(ka, kb).astype(np.int64) << 32 | np.maximum(ka, kb)
    assert len(np.unique(keys[(ka >= 0) & (kb >= 0) & (ka != kb)])) < np.sum((ka >= 0) & (kb >= 0) & (ka != kb)) - 500
    assert not np.isin(np.arange(0, 2000, 97), edges).any()
    inp, parts = cap_graph(rng)
    lab = scipy_labels(inp['n_kp'], expected_edges(inp)[0])
    assert [len(p) for p in parts[:3]] == [65536, 65537, 70000]
    for p in parts[:3]:
        assert np.all(lab[p] == p.min())


def test_scene_builder(scene, monkeypatch):
    """The scene's tracks have the geometry they were built for, and the oracle's triangulation shows it; a 9th round
    would accept a 9th point on the tracks of 9 and 10 points."""
    sc = scene
    monkeypatch.setattr(O, 'MAX_POINTS', 9)
    for s, n in sc['tracks']:
        kind, meta = sc['groups'][sc['kp_group'][sc['obs_kp'][s]]]
        if kind == 'multi' and meta['K'] > 8:
            r = O.triangulate(sc['obs_kp'], [(s, n)], sc['kp_xy'], sc['kp_n'], sc['kp_key'], sc['recs'],
                              sc['img_cam'], sc['cams'], REPROJ_PX, MIN_ANGLE)
            assert len(r[0]) == 9
    monkeypatch.undo()
    for kind, meta in sc['groups']:
        if kind == 'behind_all':
            for i in meta['imgs']:
                assert project(sc['recs'][i], sc['cams'][sc['img_cam'][i]], meta['X'])[1][0] < 0
        if kind == 'behind_one':
            i = meta['behind']
            assert project(sc['recs'][i], sc['cams'][sc['img_cam'][i]], meta['X'])[1][0] < 0
        if kind == 'narrow':
            assert angle_deg(sc['recs'][meta['imgs'][0]], sc['recs'][meta['imgs'][1]], meta['X']) < 0.2
    assert max(n for _, n in sc['tracks']) > TRI_THREADS
    pts, plen, _, kp_point = sc['ref']
    check_scene_structure(sc, pts, plen, kp_point)


# ---- the device entries ----------------------------------------------------------------------------------------------
def _dev_handle():
    from patch2pix_b200 import _lib
    h = _lib.default_handle(torch.device('cuda'))
    return _lib, h


def run_tracks(inp):
    """p2p_sfm_tracks with sfm._triangulate's arguments -> dict(labels, obs_kp, start, tlen, counts, launches)."""
    _lib, h = _dev_handle()
    dev, p = torch.device('cuda'), _lib.ptr
    M, n_kp = len(inp['kp_of_ep']) // 2, inp['n_kp']
    P = len(inp['offsets']) - 1
    kp_of_ep = torch.from_numpy(inp['kp_of_ep'] if M else np.full(2, -1, np.int32)).to(dev)
    off = torch.from_numpy(inp['offsets']).to(dev)
    E, thr, kp_n = (torch.from_numpy(np.ascontiguousarray(inp[k])).to(dev) for k in ('E', 'thr', 'kp_n'))
    nk = max(n_kp, 1)
    labels, obs_kp, start, tlen = (torch.full((nk,), -7, dtype=torch.int32, device=dev) for _ in range(4))
    cnt = torch.zeros(8, dtype=torch.int64, device=dev)
    ct = np.zeros(6, dtype=np.int64)
    n0 = h.launch_count()
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_sfm_tracks(h.h, p(kp_of_ep), M, p(off), P, p(E), p(thr), p(kp_n), n_kp, p(labels),
                                        p(obs_kp), p(start), p(tlen), p(cnt), ct.ctypes.data_as(C.POINTER(C.c_int64)),
                                        h.stream()))
    launches = h.launch_count() - n0
    T = int(ct[1])
    out = dict(labels=labels[:n_kp].cpu().numpy(), obs_kp=obs_kp[:n_kp].cpu().numpy(), start=start[:T].cpu().numpy(),
               tlen=tlen[:T].cpu().numpy(), counts=ct, launches=launches)
    assert np.array_equal(cnt[:6].cpu().numpy(), ct)
    return out


def run_triangulate(sc):
    """p2p_sfm_triangulate with sfm._triangulate's arguments on the scene's track table."""
    _lib, h = _dev_handle()
    dev, p = torch.device('cuda'), _lib.ptr
    n_kp, T = len(sc['kp_xy']), len(sc['tracks'])
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a if dt is None else a.astype(dt))).to(dev)
    obs_kp = t(sc['obs_kp'], np.int32)
    start = t(np.array([s for s, _ in sc['tracks']]), np.int32)
    tlen = t(np.array([n for _, n in sc['tracks']]), np.int32)
    kp_xy, kp_n, kp_key = t(sc['kp_xy']), t(sc['kp_n']), t(sc['kp_key'].view(np.int64))
    recs, cams = t(sc['recs']), t(sc['cams'])
    img_cam = t(np.append(sc['img_cam'], 0), np.int32)
    pts = torch.empty(8 * T, 3, dtype=torch.float64, device=dev)
    plen = torch.empty(8 * T, dtype=torch.int32, device=dev)
    perr = torch.empty(8 * T, dtype=torch.float64, device=dev)
    kp_point = torch.full((n_kp,), -7, dtype=torch.int32, device=dev)
    cnt = torch.zeros(8, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(h.lib.p2p_sfm_triangulate(h.h, p(obs_kp), p(start), p(tlen), T, n_kp, p(kp_xy), p(kp_n), p(kp_key),
                                             p(recs), p(img_cam), p(cams), REPROJ_PX,
                                             math.cos(math.radians(MIN_ANGLE)), p(pts), p(plen), p(perr),
                                             p(kp_point), p(cnt), h.stream()))
        n = int(cnt[0].item())
    return (pts[:n].cpu().numpy(), plen[:n].cpu().numpy().astype(np.int64), perr[:n].cpu().numpy(),
            kp_point.cpu().numpy().astype(np.int64))


@pytest.fixture(scope='module')
def one_batch_launches():
    """Launches of p2p_sfm_tracks on one edge: hooking converges in the first batch."""
    return run_tracks(graph_inputs([0], [1], 2, np.array([0, 1]), np.random.default_rng(0)))['launches']


def hook_batches(got, one_batch_launches):
    extra = got['launches'] - one_batch_launches
    assert extra >= 0 and extra % HOOK_BATCH_LAUNCHES == 0, got['launches']
    return 1 + extra // HOOK_BATCH_LAUNCHES


def assert_tracks_equal(got, ref):
    labels, obs, starts, lens, counts, edges = ref
    np.testing.assert_array_equal(got['labels'], labels)
    np.testing.assert_array_equal(got['obs_kp'], obs)
    np.testing.assert_array_equal(got['start'], starts)
    np.testing.assert_array_equal(got['tlen'], lens)
    np.testing.assert_array_equal(got['counts'], counts)     # edges, tracks, observations, rejected, first-in-pair, 0


@pytest.mark.gpu
@pytest.mark.parametrize('graph', list(GRAPHS))
def test_components_match_oracle_and_scipy(graph, one_batch_launches, record_property):
    """Labels, obs_kp, the track table and the counts bit for bit against sfm_oracle.components / tracks; the labels
    against scipy's connected components too.  counts[0] counts each edge once however often it is matched
    (duplicate-edge skip in the hook stage).  The bit-reversed path needs about 20 hook rounds if each only halves the
    roots, more than one batch of 16; the launch count shows how many batches it took."""
    inp = GRAPHS[graph](np.random.default_rng(10))
    ref = reference_tracks(inp)
    got = run_tracks(inp)
    assert_tracks_equal(got, ref)
    np.testing.assert_array_equal(got['labels'], scipy_labels(inp['n_kp'], ref[5]))
    b = hook_batches(got, one_batch_launches)
    record_property('hook_batches', b)
    print(f'{graph}: {inp["n_kp"]} keypoints, {len(inp["kp_of_ep"]) // 2} matches, {len(ref[5])} edges, '
          f'{len(ref[2])} tracks, hooking in {b} batch(es) of 16 rounds'
          f'{" (crossed a batch boundary)" if b > 1 else ""}')
    if graph == 'random_multigraph':
        assert ref[4][0] < ref[4][4] - 50000      # duplicate edges and self-edges are matched but not counted


@pytest.mark.gpu
def test_empty_graphs():
    """No matches with and without keypoints, keypoints that no edge touches, and matches whose every endpoint was
    dropped (n_kp = 0)."""
    rng = np.random.default_rng(3)
    cases = [graph_inputs([], [], 0, np.zeros(2, np.int64), rng),
             graph_inputs([], [], 7, np.zeros(2, np.int64), rng),
             graph_inputs([0, 2, -1, 3, 5], [0, -1, 4, 3, 5], 7, np.array([0, 2, 5]), rng),
             graph_inputs([-1, -1, -1], [-1, -1, -1], 0, np.array([0, 1, 3]), rng)]
    for i, inp in enumerate(cases):
        got = run_tracks(inp)
        ref = reference_tracks(inp)
        assert_tracks_equal(got, ref)
        assert ref[4][0] == ref[4][1] == 0 and np.array_equal(got['labels'], np.arange(inp['n_kp'])), i


@pytest.mark.gpu
def test_track_cap(one_batch_launches):
    """A component of exactly 2^16 observations is a track; components of 2^16 + 1 and 70000 are each counted in
    counts[3] and make no track.  Each track head is walked by one thread, 2^16 steps here."""
    inp, parts = cap_graph(np.random.default_rng(4))
    ref = reference_tracks(inp)
    got = run_tracks(inp)
    assert_tracks_equal(got, ref)
    big = {int(p.min()): len(p) for p in parts[:3]}
    head_len = dict(zip(got['labels'][got['obs_kp'][got['start']]].tolist(), got['tlen'].tolist()))
    assert head_len[min(parts[0])] == O.MAX_TRACK
    assert all(l not in head_len for l, n in big.items() if n > O.MAX_TRACK)
    assert got['counts'][3] == 2 and got['counts'][1] == 1 + 3000
    assert got['counts'][2] == O.MAX_TRACK + sum(len(p) for p in parts[3:3003])
    hook_batches(got, one_batch_launches)


@pytest.mark.gpu
def test_triangulation_matches_oracle(scene):
    """points, point_len, point_err and kp_point bit for bit against sfm_oracle.triangulate: sfm.cu is compiled without
    fused multiply-add and the oracle repeats each expression in the kernel's order (sums in observation order, the
    IEEE-rounded sqrt and division of both), so no tolerance is needed.  Then the geometry of each kind of track."""
    pts, plen, perr, kp_point = run_triangulate(scene)
    rp, rl, re, rk = scene['ref']
    assert len(rp) > 150 and len(pts) == len(rp), (len(pts), len(rp))
    np.testing.assert_array_equal(kp_point, rk)
    np.testing.assert_array_equal(plen, rl)
    for a, b, name in ((pts, rp, 'points'), (perr, re, 'point_err')):
        assert np.array_equal(a.view(np.int64), b.view(np.int64)), \
            f'{name}: max |diff| {np.abs(a - b).max():.3e}, max rel {np.max(np.abs(a - b) / np.abs(b)):.3e}'
    check_scene_structure(scene, pts, plen, kp_point)


@pytest.mark.gpu
def test_determinism(scene):
    """The largest graph twice, and again with its matches permuted within each pair (a path repeats no keypoint in a
    pair, so the edges do not change): labels and tracks identical.  The scene's triangulation twice: bit-identical."""
    rng = np.random.default_rng(10)
    inp = GRAPHS['bitrev_path'](rng)
    a, b = run_tracks(inp), run_tracks(inp)
    pair = np.repeat(np.arange(len(inp['offsets']) - 1), np.diff(inp['offsets']))
    perm = np.argsort(pair + np.random.default_rng(5).random(len(pair)), kind='stable')
    assert not np.array_equal(perm, np.arange(len(perm)))
    inp_p = dict(inp, kp_of_ep=inp['kp_of_ep'].reshape(-1, 2)[perm].reshape(-1).copy())
    c = run_tracks(inp_p)
    for k in ('labels', 'obs_kp', 'start', 'tlen', 'counts'):
        assert np.array_equal(a[k], b[k]) and np.array_equal(a[k], c[k]), k
    big = GRAPHS['random_multigraph'](np.random.default_rng(10))
    a, b = run_tracks(big), run_tracks(big)
    for k in ('labels', 'obs_kp', 'start', 'tlen', 'counts'):
        assert np.array_equal(a[k], b[k]), k
    r1, r2 = run_triangulate(scene), run_triangulate(scene)
    for x, y in zip(r1, r2):
        assert np.array_equal(x.view(np.int64), y.view(np.int64))
