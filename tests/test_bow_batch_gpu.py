"""GPU: the batched DBoW2 transform against the resident vocabulary (pslam_bow_set_vocabulary + pslam_bow_transform_batch[_dev]).  Every frame's
BowVector (word ids, double values) and FeatureVector (node ids, offsets, feature lists) and the counts must be byte-identical to the CPU oracle
(oracle/bow_transform.cc), to the single-frame pslam_bow_transform and, where it is built, to the reference's own DBoW2."""
import numpy as np
import pytest

import oracle_lib
import ref_lib
from planarslam_b200 import synth_lines as sl
from planarslam_b200._lib import E_INVALID, Context, PslamError
from planarslam_b200.vocabulary import bow_set_vocabulary, bow_transform_batch, load_orb_vocabulary_txt

pytestmark = pytest.mark.gpu
KEYS = ("word_id", "word_val", "node_id", "node_off", "node_feat")


@pytest.fixture(scope="module")
def ctx():
    c = Context(640, 480, 1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def full_voc():
    return sl.make_vocabulary_full(11, k=10, L=6)


def _frames(seed, voc, nframes, cap, n_lo, n_hi=None):
    rng = np.random.default_rng(seed)
    n = rng.integers(n_lo, (n_hi or cap) + 1, nframes).astype(np.int32)
    desc = np.zeros((nframes, cap, 32), np.uint8)
    for f in range(nframes):
        desc[f, :n[f]] = sl.make_features_for_vocabulary(seed * 100003 + f, voc, int(n[f]))
    desc[np.arange(cap)[None, :] >= n[:, None]] = 0xA5           # padding rows carry garbage the transform must not read
    return desc, n


def _assert_same(got, want, tag):
    for key in KEYS:
        a, b = np.asarray(got[key]), np.asarray(want[key])
        assert a.dtype == b.dtype, (tag, key)
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), (tag, key)


def _check_frames(voc, desc, n, out, levelsup, frames):
    for f in frames:
        _assert_same(out[f], oracle_lib.bow_transform(voc, desc[f, :n[f]], levelsup), (f, levelsup))


def test_full_orbvoc_shape_1584_frames(ctx, full_voc):
    bow_set_vocabulary(ctx, full_voc)
    desc, n = _frames(1, full_voc, 1584, 1100, 900)
    out = bow_transform_batch(ctx, desc, n, 4)
    assert len(out) == 1584
    sample = np.random.default_rng(7).choice(1584, 24, replace=False)
    _check_frames(full_voc, desc, n, out, 4, sorted(sample.tolist()) + [0, 1583])
    assert all(len(out[f]["word_id"]) > 100 for f in sample)
    again = bow_transform_batch(ctx, desc, n, 4)                            # two runs of the same batch: identical bytes
    for a, b in zip(out, again):
        _assert_same(a, b, "repeat")
    for lu in (0, 2, 6, 7):
        o = bow_transform_batch(ctx, desc[:6], n[:6], lu)
        _check_frames(full_voc, desc, n, o, lu, range(6))


@pytest.mark.parametrize("k,L", [(4, 5), (16, 4), (17, 2), (32, 2), (3, 3)])
def test_small_and_odd_shapes(ctx, k, L):
    voc = sl.make_vocabulary_full(k * 10 + L, k=k, L=L) if k == 16 else sl.make_vocabulary(k * 10 + L, k=k, L=L)
    bow_set_vocabulary(ctx, voc)
    desc, n = _frames(k + L, voc, 12, 700, 1)
    for lu in range(L + 2):
        _check_frames(voc, desc, n, bow_transform_batch(ctx, desc, n, lu), lu, range(12))


def test_edge_frames(ctx):
    voc = sl.make_vocabulary(21, k=10, L=3, stop_frac=0.2)
    bow_set_vocabulary(ctx, voc)
    cap = 400
    pool = sl.make_features_for_vocabulary(5, voc, 6000)
    fw = oracle_lib.bow_transform(voc, pool, 4)["feat_word"]
    stopped = pool[voc["weight"][voc["leaves"][fw]] == 0][:cap]               # every feature on a word of weight 0
    assert len(stopped) >= 50
    dup = np.repeat(pool[:7], 40, axis=0)[np.random.default_rng(1).permutation(280)]
    root = voc["child_id"][:10]
    dist = lambda a, b: int(np.unpackbits(a ^ b).sum())
    a, b = next((a, b) for a in range(10) for b in range(a + 1, 10) if dist(voc["desc"][root[a]], voc["desc"][root[b]]) % 2 == 0)
    ca, cb = voc["desc"][root[a]], voc["desc"][root[b]]
    bits = np.unpackbits(ca)
    diff = np.flatnonzero(np.unpackbits(ca ^ cb))
    bits[diff[: len(diff) // 2]] ^= 1
    tie = np.packbits(bits)                                                   # as far from root child a as from root child b
    d = [dist(tie, voc["desc"][c]) for c in root]
    assert d[a] == d[b] < min(d[j] for j in range(10) if j not in (a, b))
    rows = [np.zeros((0, 32), np.uint8), pool[:1], pool[:cap], stopped, dup, np.repeat(tie[None], 3, axis=0)]
    desc = np.zeros((len(rows), cap, 32), np.uint8)
    n = np.array([len(r) for r in rows], np.int32)
    for f, r in enumerate(rows):
        desc[f, :len(r)] = r
    out = bow_transform_batch(ctx, desc, n, 2)
    _check_frames(voc, desc, n, out, 2, range(len(rows)))
    assert len(out[0]["word_id"]) == 0 and out[0]["node_off"].tolist() == [0]
    assert len(out[3]["word_id"]) == 0 and len(out[3]["node_id"]) == 0
    assert oracle_lib.bow_transform(voc, tie[None], 2)["feat_node"][0] == root[a]     # the first of two equidistant children wins
    assert out[5]["node_id"].tolist() == [root[a]]


def test_matches_single_frame_entry_point(ctx):
    from planarslam_b200.matcher import bow_transform
    voc = sl.make_vocabulary(33, k=10, L=4)
    bow_set_vocabulary(ctx, voc)
    desc, n = _frames(3, voc, 6, 2000, 1500)
    out = bow_transform_batch(ctx, desc, n, 4)
    for f in range(6):
        _assert_same(out[f], bow_transform(ctx, voc, desc[f, :n[f]], 4), f)


def test_device_chain_after_orb(ctx, full_voc):
    import torch
    from planarslam_b200 import synth
    nframes = 8
    c = Context(640, 480, nframes, nfeatures=1000)
    try:
        dev = torch.device("cuda", 0)
        L = c.L
        cap = int(L.pslam_orb_max_keypoints(c.h))
        assert cap <= 3072
        frames = np.stack([synth.render_frame(4, 5 * k, 640, 480)[0] for k in range(nframes)])
        d_gray = torch.from_numpy(frames).to(dev)
        d_kps = torch.empty((nframes, cap, 28), dtype=torch.uint8, device=dev)
        d_desc = torch.empty((nframes, cap, 32), dtype=torch.uint8, device=dev)
        d_n = torch.zeros(nframes, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()                                             # the context's own stream does not wait for torch's
        c.check(L.pslam_orb_extract_batch_dev(c.h, d_gray.data_ptr(), nframes, d_kps.data_ptr(), d_desc.data_ptr(), cap, d_n.data_ptr()))
        bow_set_vocabulary(c, full_voc)
        o = dict(word_id=torch.empty((nframes, cap), dtype=torch.int32, device=dev), word_val=torch.empty((nframes, cap), dtype=torch.float64, device=dev),
                 node_id=torch.empty((nframes, cap), dtype=torch.int32, device=dev), node_off=torch.empty((nframes, cap + 1), dtype=torch.int32, device=dev),
                 node_feat=torch.empty((nframes, cap), dtype=torch.int32, device=dev))
        cnt = torch.empty((nframes, 2), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        c.check(L.pslam_bow_transform_batch_dev(c.h, d_desc.data_ptr(), d_n.data_ptr(), cap, nframes, 4, *[o[k].data_ptr() for k in KEYS], cnt.data_ptr()))
        c.synchronize()
        desc, n, cnt = d_desc.cpu().numpy(), d_n.cpu().numpy(), cnt.cpu().numpy()
        h = {k: v.cpu().numpy() for k, v in o.items()}
        assert (n > 500).all()
        for f in range(nframes):
            want = oracle_lib.bow_transform(full_voc, desc[f, :n[f]], 4)
            nw, nn = cnt[f]
            got = dict(word_id=h["word_id"][f, :nw], word_val=h["word_val"][f, :nw], node_id=h["node_id"][f, :nn], node_off=h["node_off"][f, :nn + 1],
                       node_feat=h["node_feat"][f, :h["node_off"][f, nn]])
            _assert_same(got, want, f)
    finally:
        c.close()


@pytest.mark.skipif(ref_lib.bow_lib() is None, reason="oracle/_ref/libbow_ref.so not built")
def test_matches_compiled_reference(ctx, tmp_path):
    for seed, (k, L) in enumerate([(10, 4), (4, 6), (16, 3)]):
        voc = sl.make_vocabulary(50 + seed, k=k, L=L)
        path = str(tmp_path / f"voc{seed}.txt")
        ref_lib.write_vocabulary_txt(voc, path)
        rv = ref_lib.RefVocabulary(path)
        bow_set_vocabulary(ctx, load_orb_vocabulary_txt(path))
        desc, n = _frames(seed + 40, voc, 5, 1000, 200)
        for lu in (4, 1, L):
            out = bow_transform_batch(ctx, desc, n, lu)
            for f in range(5):
                _assert_same(out[f], rv.transform(desc[f, :n[f]], lu), (seed, lu, f))


def test_trailing_node_is_dropped(ctx, tmp_path):
    voc = sl.make_vocabulary(8, k=10, L=3)
    path = str(tmp_path / "voc.txt")
    ref_lib.write_vocabulary_txt(voc, path)
    with open(path, "a") as fh:
        fh.write("\n")
    v = load_orb_vocabulary_txt(path)
    extra = len(v["word_id"]) - 1
    bow_set_vocabulary(ctx, v)
    feats = np.concatenate([np.zeros((2, 32), np.uint8), sl.make_features_for_vocabulary(9, v, 300)])
    desc, n = feats[None], np.array([len(feats)], np.int32)
    out = bow_transform_batch(ctx, desc, n, 2)[0]
    o = oracle_lib.bow_transform(v, feats, 2)
    assert o["feat_node"][0] == extra and o["feat_word"][0] == -1
    _assert_same(out, o, "trailing")
    assert 0 not in out["node_feat"] and 1 not in out["node_feat"] and extra not in out["node_id"]


def test_lifecycle_and_rejections():
    c = Context(640, 480, 1)
    try:
        L = c.L
        desc, n = np.zeros((1, 8, 32), np.uint8), np.array([8], np.int32)
        with pytest.raises(PslamError) as e:
            bow_transform_batch(c, desc, n)
        assert e.value.code == E_INVALID
        a, b = sl.make_vocabulary(1, k=8, L=3), sl.make_vocabulary(2, k=8, L=3)
        feats = sl.make_features_for_vocabulary(3, a, 500)
        bow_set_vocabulary(c, a)
        ra = bow_transform_batch(c, feats[None], [500])[0]
        _assert_same(ra, oracle_lib.bow_transform(a, feats, 4), "a")
        bow_set_vocabulary(c, b)                                                  # replacing changes the results to the new vocabulary's
        rb = bow_transform_batch(c, feats[None], [500])[0]
        _assert_same(rb, oracle_lib.bow_transform(b, feats, 4), "b")
        assert ra["word_val"].tobytes() != rb["word_val"].tobytes()
        bow_set_vocabulary(c, None)                                               # n_nodes = 0 releases it
        with pytest.raises(PslamError) as e:
            bow_transform_batch(c, feats[None], [500])
        assert e.value.code == E_INVALID
        wide = sl.make_vocabulary(4, k=33, L=1)                                   # a node with 33 children
        with pytest.raises(PslamError) as e:
            bow_set_vocabulary(c, wide)
        assert e.value.code == E_INVALID and "32 children" in str(e.value)
        bow_set_vocabulary(c, sl.make_vocabulary(4, k=32, L=1))
        big = np.zeros((1, 3073, 32), np.uint8)
        for args in ((big, [3073]), (big[:, :3072], [3073]), (big[:, :100], [-1])):   # more than 3072 rows, n > cap, n < 0
            with pytest.raises(PslamError) as e:
                bow_transform_batch(c, *args)
            assert e.value.code == E_INVALID
        assert len(bow_transform_batch(c, big[:, :3072], [3072])) == 1
        assert L.pslam_bow_transform_batch(c.h, None, None, 8, 0, 4, None, None, None, None, None, None) == 0      # empty batch
    finally:
        c.close()


def test_feeds_search_by_bow(ctx):
    from planarslam_b200.matcher import search_by_bow
    voc = sl.make_vocabulary(61, k=10, L=4)
    bow_set_vocabulary(ctx, voc)
    rng = np.random.default_rng(3)
    kf_desc = sl.make_features_for_vocabulary(62, voc, 900)
    src = rng.integers(0, 900, 800)
    fr_desc = kf_desc[src] ^ np.packbits(rng.random((800, 256)) < 0.04, axis=1)
    cap = 900
    desc = np.zeros((2, cap, 32), np.uint8)
    desc[0, :900], desc[1, :800] = kf_desc, fr_desc
    out = bow_transform_batch(ctx, desc, [900, 800], 4)
    kf_angle = rng.uniform(0, 360, 900).astype(np.float32)
    fr_angle = ((kf_angle[src] - 20 + rng.normal(0, 3, 800)) % 360).astype(np.float32)
    has_mp = (rng.random(900) < 0.8).astype(np.uint8)
    res = []
    for kfv, frv in ((out[0], out[1]), (oracle_lib.bow_transform(voc, kf_desc, 4), oracle_lib.bow_transform(voc, fr_desc, 4))):
        kf = dict(desc=kf_desc, angle=kf_angle, has_mp=has_mp, node_id=kfv["node_id"], node_off=kfv["node_off"], node_feat=kfv["node_feat"])
        fr = dict(desc=fr_desc, angle=fr_angle, node_id=frv["node_id"], node_off=frv["node_off"], node_feat=frv["node_feat"])
        res.append(search_by_bow(ctx, kf, fr))
    assert res[0][0] == res[1][0] > 100 and np.array_equal(res[0][1], res[1][1])
