"""The DBoW2 ORB vocabulary (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h): the ORBvoc.txt loader and the batched transform
(Frame::ComputeBoW / KeyFrame::ComputeBoW) against a vocabulary kept resident on the GPU."""
from __future__ import annotations

import warnings

import numpy as np

from ._lib import Context

_NODE_TOKENS = 2 + 32 + 1                      # parent, isLeaf, 32 descriptor bytes, weight


def load_orb_vocabulary_txt(path: str) -> dict:
    """The flat arrays TemplatedVocabulary::loadFromTextFile (TemplatedVocabulary.h:1338-1434) builds from an ORBvoc.txt file, in node-id order:
    L, k, desc [n][32] u8, child_off [n + 1] / child_id i32 (children CSR in file order), word_id i32 (leaves numbered in file order, -1 elsewhere),
    weight f64, leaves (the word nodes in word order).

    The header is checked as the reference checks it (k in 0..20, L in 1..10, scoring <= 5, weighting <= 3); only L1 scoring with TF-IDF
    weighting ("0 0") is accepted, the one the transform implements.  Every node line must carry 35 tokens.  An empty line - in particular the
    one after the file's final newline, which the reference's while(!f.eof()) loop reads - becomes what the reference makes of it: a child of the
    root with no children and weight 0 that is not a word.  Its descriptor is left uninitialised by the reference; here it is all zeros and its
    word id -1, so a feature that descends into it is dropped like any weight-0 feature (DESIGN.md section 5)."""
    with open(path, "rb") as fh:
        data = fh.read()
    nl = data.find(b"\n")
    head = (data if nl < 0 else data[:nl]).split()
    try:
        k, L, scoring, weighting = (int(t) for t in head[:4])
    except ValueError:
        raise ValueError(f"{path}: the header must start with four integers 'k L scoring weighting'") from None
    if not (0 <= k <= 20 and 1 <= L <= 10 and 0 <= scoring <= 5 and 0 <= weighting <= 3):
        raise ValueError(f"{path}: not a DBoW2 text vocabulary (header k={k} L={L} scoring={scoring} weighting={weighting})")
    if scoring != 0 or weighting != 0:
        raise ValueError(f"{path}: only L1 scoring with TF-IDF weighting (header '0 0') is supported, got {scoring} {weighting}")

    body = b"" if nl < 0 else data[nl + 1:]
    n_lines = 0 if nl < 0 else body.count(b"\n") + 1      # the piece after the last newline is a line too (the reference reads it)
    b = np.frombuffer(body, np.uint8)
    tok = (b != 32) & ((b < 9) | (b > 13))                 # not isspace() in the C locale: what istream >> skips
    start = np.zeros(len(b) + 1, bool)                      # first byte of each token (+ one past the end for the last, possibly empty line)
    start[:len(b)] = tok
    start[1:len(b)] &= ~tok[:-1]
    line_start = np.concatenate([[0], np.flatnonzero(b == 10) + 1])
    line_end = np.concatenate([line_start[1:] - 1, [len(b)]])
    ntok = np.where(line_end > line_start, np.add.reduceat(start.view(np.int8), line_start, dtype=np.int32), 0) if n_lines else np.zeros(0, np.int32)
    bad = np.flatnonzero((ntok != 0) & (ntok != _NODE_TOKENS))
    if len(bad):
        raise ValueError(f"{path}: line {int(bad[0]) + 2} has {int(ntok[bad[0]])} fields, a node line has {_NODE_TOKENS}")
    full = np.flatnonzero(ntok == _NODE_TOKENS)
    with warnings.catch_warnings():
        warnings.simplefilter("error")                     # numpy warns (instead of raising) on text it cannot parse
        try:
            vals = np.fromstring(body, dtype=np.float64, sep=" ") if len(full) else np.zeros(0)
        except (DeprecationWarning, ValueError) as e:
            raise ValueError(f"{path}: unparsable node line ({e})") from None
    if vals.size != len(full) * _NODE_TOKENS:
        raise ValueError(f"{path}: unparsable node line")
    vals = vals.reshape(-1, _NODE_TOKENS)
    ints = vals[:, :34]
    if not np.array_equal(ints, np.floor(ints)):
        raise ValueError(f"{path}: parent, isLeaf and descriptor fields must be integers")
    if len(full) and (vals[:, 2:34].min() < 0 or vals[:, 2:34].max() > 255):
        raise ValueError(f"{path}: descriptor byte outside 0..255")

    n = n_lines + 1
    ids = full + 1                                          # node id = line number after the header
    parent = np.zeros(n, np.int64)
    parent[ids] = vals[:, 0]
    if np.any(parent[1:] < 0) or np.any(parent[1:] >= np.arange(1, n)):
        raise ValueError(f"{path}: every node's parent must be an earlier node")
    is_word = np.zeros(n, bool)
    is_word[ids] = vals[:, 1] > 0
    word_id = np.full(n, -1, np.int32)
    word_id[is_word] = np.arange(int(is_word.sum()), dtype=np.int32)
    weight = np.zeros(n)
    weight[ids] = vals[:, 34]
    desc = np.zeros((n, 32), np.uint8)
    desc[ids] = vals[:, 2:34].astype(np.uint8)
    child_id = (np.argsort(parent[1:], kind="stable") + 1).astype(np.int32)
    child_off = np.concatenate([[0], np.cumsum(np.bincount(parent[1:], minlength=n))]).astype(np.int32)
    return dict(L=L, k=k, desc=desc, child_off=child_off, child_id=child_id, word_id=word_id, weight=weight,
                leaves=np.flatnonzero(is_word).astype(np.int32))


def bow_set_vocabulary(ctx: Context, voc: dict | None):
    """pslam_bow_set_vocabulary: upload the vocabulary (flat arrays as load_orb_vocabulary_txt or synth_lines.make_vocabulary return them) and keep
    it in HBM for bow_transform_batch; voc=None releases it."""
    if voc is None:
        ctx.check(ctx.L.pslam_bow_set_vocabulary(ctx.h, 0, 0, None, None, None, None, None))
        return
    a = {key: np.ascontiguousarray(voc[key], dt) for key, dt in (("desc", np.uint8), ("child_off", np.int32), ("child_id", np.int32),
                                                                 ("word_id", np.int32), ("weight", np.float64))}
    ctx.check(ctx.L.pslam_bow_set_vocabulary(ctx.h, len(a["word_id"]), int(voc["L"]), a["desc"].ctypes.data, a["child_off"].ctypes.data,
                                             a["child_id"].ctypes.data, a["word_id"].ctypes.data, a["weight"].ctypes.data))


def bow_transform_batch(ctx: Context, desc: np.ndarray, n, levelsup: int = 4) -> list[dict]:
    """pslam_bow_transform_batch: ORBVocabulary::transform(mDescriptors, mBowVec, mFeatVec, levelsup) of every frame against the resident vocabulary.
    desc [nframes][cap][32] u8 with n[f] valid rows.  Returns one dict per frame in the shape matcher.bow_transform returns
    (word_id, word_val, node_id, node_off, node_feat)."""
    d = np.ascontiguousarray(desc, np.uint8)
    if d.ndim != 3 or d.shape[2] != 32:
        raise ValueError("desc must be [nframes][cap][32] uint8")
    nframes, cap = d.shape[:2]
    nn = np.ascontiguousarray(n, np.int32)
    if nn.shape != (nframes,):
        raise ValueError("n must hold one row count per frame")
    o = dict(word_id=np.zeros((nframes, cap), np.int32), word_val=np.zeros((nframes, cap)), node_id=np.zeros((nframes, cap), np.int32),
             node_off=np.zeros((nframes, cap + 1), np.int32), node_feat=np.zeros((nframes, cap), np.int32))
    cnt = np.zeros((nframes, 2), np.int32)
    ctx.check(ctx.L.pslam_bow_transform_batch(ctx.h, d.ctypes.data, nn.ctypes.data, cap, nframes, levelsup, o["word_id"].ctypes.data,
                                              o["word_val"].ctypes.data, o["node_id"].ctypes.data, o["node_off"].ctypes.data,
                                              o["node_feat"].ctypes.data, cnt.ctypes.data))
    out = []
    for f in range(nframes):
        nw, nd = int(cnt[f, 0]), int(cnt[f, 1])
        off = o["node_off"][f, :nd + 1].copy()
        out.append(dict(word_id=o["word_id"][f, :nw].copy(), word_val=o["word_val"][f, :nw].copy(), node_id=o["node_id"][f, :nd].copy(),
                        node_off=off, node_feat=o["node_feat"][f, :int(off[-1])].copy()))
    return out
