"""Seeded synthetic inputs for LSDmatcher::SearchByProjection: a frame's key lines with binary descriptors and a local map of
lines projected into it (the fields Frame::isInFrustum(MapLine*) fills), with noisy descriptor copies, occluded / bad
entries, octave mismatches and near-duplicate descriptors so that the ratio test and the occupancy rule fire."""
from __future__ import annotations

import numpy as np


def make_line_search(seed: int, n_frame: int = 40, n_map: int = 120, n_levels: int = 8):
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 613 + 5))
    pt = np.stack([rng.uniform(20, 620, n_frame), rng.uniform(20, 460, n_frame)], 1).astype(np.float32)
    angle = rng.uniform(-np.pi, np.pi, n_frame).astype(np.float32)
    octave = rng.integers(0, 2, n_frame).astype(np.int32)
    desc = rng.integers(0, 256, (n_frame, 32), dtype=np.uint8)
    frame = dict(pt=pt, angle=angle, octave=octave, desc=desc, has_obs=(rng.random(n_frame) < 0.15).astype(np.uint8),
                 scale_factors=(1.2 ** np.arange(n_levels)).astype(np.float32))
    src = rng.integers(0, n_frame, n_map)                       # the frame line each map line really corresponds to
    half = rng.uniform(10, 60, n_map)
    ang = angle[src] + rng.normal(0, 0.3, n_map)
    mid = pt[src] + rng.normal(0, 3.0, (n_map, 2))
    d = np.stack([np.cos(ang), np.sin(ang)], 1) * half[:, None]
    proj = np.concatenate([mid - d, mid + d], 1).astype(np.float32)
    mdesc = desc[src].copy()
    flips = rng.random((n_map, 256)) < rng.choice([0.02, 0.1, 0.3], n_map)[:, None]
    mdesc ^= np.packbits(flips, axis=1)
    dup = rng.random(n_map) < 0.2                               # near-duplicate descriptors of another frame line: ratio test
    mdesc[dup] = desc[(src[dup] + 1) % n_frame]
    level = np.clip(octave[src] + rng.integers(-1, 2, n_map), 0, n_levels - 1).astype(np.int32)
    mp = dict(skip=(rng.random(n_map) < 0.1).astype(np.uint8), level=level, view_cos=rng.uniform(0.99, 1.0, n_map).astype(np.float32), proj=proj,
              desc=np.ascontiguousarray(mdesc), has_obs=(rng.random(n_map) < 0.7).astype(np.uint8))
    return frame, mp


def make_bow_pair(seed: int, n_kf: int = 1000, n_f: int = 1000, n_nodes: int = 300, shared: float = 0.7):
    """A key frame and a frame for ORBmatcher::SearchByBoW: `shared` of the frame features are noisy copies of key-frame features
    (same vocabulary node, rotated by a common in-plane angle plus noise), the rest is clutter; feature vectors as CSR."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 9176 + 3))
    kf_desc = rng.integers(0, 256, (n_kf, 32), dtype=np.uint8)
    kf_node = rng.integers(0, n_nodes, n_kf)
    kf_angle = rng.uniform(0, 360, n_kf).astype(np.float32)
    src = rng.integers(0, n_kf, n_f)
    is_copy = rng.random(n_f) < shared
    f_desc = rng.integers(0, 256, (n_f, 32), dtype=np.uint8)
    flips = rng.random((n_f, 256)) < rng.choice([0.02, 0.06, 0.15], n_f)[:, None]
    f_desc[is_copy] = kf_desc[src[is_copy]] ^ np.packbits(flips, axis=1)[is_copy]
    f_node = np.where(is_copy, kf_node[src], rng.integers(0, n_nodes + 40, n_f))
    rot = 17.0
    f_angle = np.where(is_copy, (kf_angle[src] - rot + rng.normal(0, 4, n_f)) % 360, rng.uniform(0, 360, n_f)).astype(np.float32)
    wrong = is_copy & (rng.random(n_f) < 0.1)
    f_angle[wrong] = rng.uniform(0, 360, int(wrong.sum())).astype(np.float32)          # inconsistent rotation: removed by the histogram

    def csr(node):
        ids = np.unique(node)
        order = np.argsort(node, kind="stable")
        counts = np.array([(node == i).sum() for i in ids])
        return ids.astype(np.int32), np.concatenate([[0], np.cumsum(counts)]).astype(np.int32), order.astype(np.int32)
    kid, koff, kfeat = csr(kf_node)
    fid, foff, ffeat = csr(f_node)
    kf = dict(desc=kf_desc, angle=kf_angle, has_mp=(rng.random(n_kf) < 0.8).astype(np.uint8), node_id=kid, node_off=koff, node_feat=kfeat)
    fr = dict(desc=np.ascontiguousarray(f_desc), angle=f_angle, node_id=fid, node_off=foff, node_feat=ffeat)
    return kf, fr


def make_vocabulary(seed: int, k: int = 10, L: int = 3, stop_frac: float = 0.05):
    """A synthetic DBoW2 vocabulary tree (branching factor k, depth L) as flat arrays in node-id order: 32-byte node descriptors, children CSR,
    word ids for the leaves (in creation order) and word weights (idf-like; a few zero = "stopped" words).  The real ORBvoc has k = 10, L = 6."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 31 + 11))
    desc = [np.zeros(32, np.uint8)]
    children = [[]]
    level = [0]
    frontier = [0]
    for lv in range(1, L + 1):
        nxt = []
        for parent in frontier:
            base = desc[parent]
            for _ in range(k):
                flips = np.packbits(rng.random(256) < (0.5 if lv == 1 else 0.12))
                desc.append(base ^ flips if lv > 1 else rng.integers(0, 256, 32, dtype=np.uint8))
                children.append([])
                level.append(lv)
                children[parent].append(len(desc) - 1)
                nxt.append(len(desc) - 1)
        frontier = nxt
    n = len(desc)
    word_id = np.full(n, -1, np.int32)
    weight = np.zeros(n)
    for w, leaf in enumerate(frontier):
        word_id[leaf] = w
        weight[leaf] = 0.0 if rng.random() < stop_frac else float(rng.uniform(0.5, 9.0))
    child_off = np.concatenate([[0], np.cumsum([len(c) for c in children])]).astype(np.int32)
    child_id = np.array([c for ch in children for c in ch], np.int32)
    return dict(L=L, k=k, desc=np.ascontiguousarray(np.array(desc, np.uint8)), child_off=child_off, child_id=child_id, word_id=word_id, weight=weight,
                leaves=np.array(frontier, np.int32))


def make_vocabulary_full(seed: int, k: int = 10, L: int = 6, stop_frac: float = 0.05):
    """A full DBoW2 vocabulary tree of ORBvoc's shape (k = 10, L = 6: 1,111,111 nodes) built level by level with numpy, in the layout of
    make_vocabulary: level order, the children of a node contiguous, level-1 descriptors random, deeper ones their parent's with about 1/8 of the
    bits flipped; leaves numbered in level order, weights idf-like with `stop_frac` of them 0."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 37 + 13))
    sizes = [k ** lv for lv in range(L + 1)]
    n = sum(sizes)
    desc = np.zeros((n, 32), np.uint8)
    desc[1:1 + k] = rng.integers(0, 256, (k, 32), dtype=np.uint8)
    first = 1                                                   # first node of the current level
    for lv in range(2, L + 1):
        parents = np.repeat(np.arange(first, first + sizes[lv - 1]), k)
        bits = lambda: rng.integers(0, 256, (len(parents), 32), dtype=np.uint8)
        desc[first + sizes[lv - 1]:first + sizes[lv - 1] + sizes[lv]] = desc[parents] ^ (bits() & bits() & bits())
        first += sizes[lv - 1]
    n_inner = n - sizes[L]
    child_off = np.concatenate([np.arange(n_inner + 1, dtype=np.int64) * k, np.full(sizes[L], n_inner * k)]).astype(np.int32)
    child_id = np.arange(1, n, dtype=np.int32)
    leaves = np.arange(n_inner, n, dtype=np.int32)
    word_id = np.full(n, -1, np.int32)
    word_id[leaves] = np.arange(sizes[L], dtype=np.int32)
    weight = np.zeros(n)
    weight[leaves] = np.where(rng.random(sizes[L]) < stop_frac, 0.0, rng.uniform(0.5, 9.0, sizes[L]))
    return dict(L=L, k=k, desc=desc, child_off=child_off, child_id=child_id, word_id=word_id, weight=weight, leaves=leaves)


def make_features_for_vocabulary(seed: int, voc: dict, n: int = 1000):
    """ORB-like descriptors: noisy copies of random leaf descriptors (so that several features fall into the same word / node)."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 77 + 1))
    src = voc["leaves"][rng.integers(0, len(voc["leaves"]) // 3 + 1, n)]
    flips = np.packbits(rng.random((n, 256)) < 0.08, axis=1)
    return np.ascontiguousarray(voc["desc"][src] ^ flips)


def make_line_frustum(seed: int, n: int = 400):
    """A camera pose + n map lines for Frame::isInFrustum(MapLine*): about half in view, the rest behind the camera, outside the image,
    outside the scale-invariance distance range or seen too obliquely.  Returns (frame dict, pos [n][6], normal [n][3], max_distance, min_distance)."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 7919 + 17))
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    ang = rng.uniform(0, 0.6)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
    t = rng.normal(0, 0.5, 3)
    Tcw = np.eye(4, dtype=np.float32); Tcw[:3, :3] = R; Tcw[:3, 3] = t
    fx, fy, cx, cy = 535.4, 539.2, 320.1, 247.6
    frame = dict(Tcw=Tcw, fx=fx, fy=fy, cx=cx, cy=cy, min_x=0.0, max_x=640.0, min_y=0.0, max_y=480.0, log_scale_factor=float(np.log(np.float32(1.2))))
    z = rng.uniform(-1.0, 6.0, n)                              # some behind the camera
    u, v = rng.uniform(-100, 740, n), rng.uniform(-80, 560, n)
    mid_c = np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1)
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    half = rng.uniform(0.05, 0.5, n)[:, None]
    Rt = R.T
    to_w = lambda Pc: (Pc - t) @ Rt.T
    sp, ep = to_w(mid_c - d * half), to_w(mid_c + d * half)
    pos = np.concatenate([sp, ep], 1)
    Ow = -Rt @ t
    view = 0.5 * (sp + ep) - Ow
    view /= np.linalg.norm(view, axis=1, keepdims=True) + 1e-12
    nrm = view + rng.normal(0, 0.6, (n, 3))                    # GetNormal(): mean viewing direction; noisy -> some below cos 0.6
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    dist = np.linalg.norm(0.5 * (sp + ep) - Ow, axis=1)
    max_d = (dist * rng.uniform(0.7, 2.5, n)).astype(np.float32)
    min_d = (max_d / np.float32(1.2 ** 7)).astype(np.float32)
    return frame, pos, nrm, max_d, min_d


def make_bow_database(seed: int, n_kf: int = 400, n_words: int = 5000, words_per_kf: int = 300, n_similar: int = 40, covis: int = 10):
    """A key-frame database for KeyFrameDatabase::DetectLoopCandidates / DetectRelocalizationCandidates: a query BowVector, `n_kf` key-frame BowVectors in the
    order KeyFrameDatabase::add saw them (CSR: off, word ascending, val L1-normalised like DBoW2's TF_IDF + L1_NORM transform), of which `n_similar` share a
    varying fraction of the query's words (a revisited place: consecutive runs, so that covisibility groups accumulate), the covisibility table
    GetBestCovisibilityKeyFrames(10) as database indices (-1 ends a row) and the flags of the key frames connected to the query (never candidates)."""
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 7919 + 5))
    idf = rng.uniform(0.5, 8.0, n_words)

    def bow(words, counts):
        words = np.asarray(words)
        order = np.argsort(words)
        v = counts[order] * idf[words[order]]
        return words[order].astype(np.int32), (v / v.sum()).astype(np.float64)
    qw = rng.choice(n_words, words_per_kf, replace=False)
    qc = rng.integers(1, 4, words_per_kf).astype(np.float64)
    q_word, q_val = bow(qw, qc)
    similar_start = int(rng.integers(0, max(n_kf - n_similar, 1)))
    off, words, vals = [0], [], []
    for k in range(n_kf):
        m = int(rng.integers(words_per_kf // 2, words_per_kf * 3 // 2))
        if similar_start <= k < similar_start + n_similar:
            frac = 0.25 + 0.6 * np.exp(-0.5 * ((k - similar_start - n_similar / 2) / (n_similar / 5)) ** 2) * rng.uniform(0.7, 1.0)
            keep = qw[rng.random(words_per_kf) < frac]
            rest = np.setdiff1d(rng.choice(n_words, m, replace=False), qw)[: max(m - len(keep), 0)]
            w = np.concatenate([keep, rest])
        else:
            w = rng.choice(n_words, m, replace=False)
        wi, vi = bow(w, rng.integers(1, 4, len(w)).astype(np.float64))
        words.append(wi); vals.append(vi); off.append(off[-1] + len(wi))
    table = np.full((n_kf, covis), -1, np.int32)
    for k in range(n_kf):            # temporal neighbours, nearest first, a few rows shorter than 10 and a few empty
        nb = [j for d in range(1, covis) for j in (k - d, k + d) if 0 <= j < n_kf][: int(rng.integers(0, covis + 1))]
        table[k, :len(nb)] = nb
    connected = np.zeros(n_kf, np.uint8)
    connected[rng.integers(0, n_kf, 5)] = 1
    if n_similar:
        connected[similar_start + int(rng.integers(0, n_similar))] = 1        # one of the similar key frames is a covisible neighbour of the query
    return dict(q_word=q_word, q_val=q_val, off=np.asarray(off, np.int32), word=np.concatenate(words).astype(np.int32), val=np.concatenate(vals),
                covis=table, connected=connected)


def make_bow_kf_pair(seed: int, **kw):
    """Two key frames for ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, ...): make_bow_pair plus map-point flags on the second side."""
    kf1, kf2 = make_bow_pair(seed, **kw)
    rng = np.random.Generator(np.random.Philox(key=int(seed) * 613 + 1))
    kf2["has_mp"] = (rng.random(len(kf2["angle"])) < 0.85).astype(np.uint8)
    return kf1, kf2
