"""CPU: the ORBvoc.txt loader (planarslam_b200.vocabulary.load_orb_vocabulary_txt) against the writer of the format, against the reference's
own loadFromTextFile + transform (oracle/_ref/libbow_ref.so) through the oracle transform, and on the trailing-newline node and bad headers."""
import numpy as np
import pytest

import oracle_lib
import ref_lib
from planarslam_b200 import synth_lines as sl
from planarslam_b200.vocabulary import load_orb_vocabulary_txt

KEYS = ("word_id", "word_val", "node_id", "node_off", "node_feat")


def _same_arrays(a, b):
    for key in ("desc", "child_off", "child_id", "word_id", "leaves"):
        assert np.array_equal(a[key], b[key]), key
    assert a["weight"].tobytes() == b["weight"].tobytes()          # bit-equal doubles
    assert (a["L"], a["k"]) == (b["L"], b["k"])


@pytest.mark.parametrize("k,L", [(10, 3), (4, 5), (16, 2), (3, 6)])
def test_loader_round_trip(tmp_path, k, L):
    voc = sl.make_vocabulary(k + L, k=k, L=L)
    rng = np.random.default_rng(k)
    voc["weight"][voc["leaves"]] = np.where(voc["weight"][voc["leaves"]] > 0, rng.random(len(voc["leaves"])) * 10 ** rng.uniform(-8, 3, len(voc["leaves"])), 0.0)
    path = str(tmp_path / "voc.txt")
    ref_lib.write_vocabulary_txt(voc, path)
    _same_arrays(load_orb_vocabulary_txt(path), voc)


def test_loader_full_orbvoc_shape(tmp_path):
    voc = sl.make_vocabulary_full(5, k=10, L=5)
    path = str(tmp_path / "voc.txt")
    ref_lib.write_vocabulary_txt(voc, path)
    _same_arrays(load_orb_vocabulary_txt(path), voc)


def test_trailing_newline_adds_one_root_child(tmp_path):
    voc = sl.make_vocabulary(2, k=6, L=3)
    path = str(tmp_path / "voc.txt")
    ref_lib.write_vocabulary_txt(voc, path)
    with open(path, "a") as f:
        f.write("\n")
    v = load_orb_vocabulary_txt(path)
    n = len(voc["word_id"])
    assert len(v["word_id"]) == n + 1
    extra = n
    root = v["child_id"][v["child_off"][0]:v["child_off"][1]]
    assert list(root) == list(voc["child_id"][:6]) + [extra]                      # the last child of the root
    assert v["child_off"][extra + 1] == v["child_off"][extra]                     # no children
    assert v["word_id"][extra] == -1 and v["weight"][extra] == 0.0 and not v["desc"][extra].any()
    assert np.array_equal(v["leaves"], voc["leaves"])
    for key in ("desc", "word_id", "weight"):
        assert np.array_equal(v[key][:n], voc[key]), key
    # an all-zero descriptor descends into the extra node (distance 0) and is dropped.  The reference leaves that node's descriptor
    # uninitialised, so its own output is not a yardstick here.
    feats = np.concatenate([np.zeros((1, 32), np.uint8), sl.make_features_for_vocabulary(3, voc, 200)])
    o = oracle_lib.bow_transform(v, feats, 2)                                   # node level 1
    assert o["feat_word"][0] == -1 and o["feat_node"][0] == extra
    assert 0 not in o["node_feat"] and extra not in o["node_id"] and len(o["word_id"]) > 10


def test_header_only_file(tmp_path):
    p = tmp_path / "v.txt"
    p.write_text("10 6 0 0")
    v = load_orb_vocabulary_txt(str(p))
    assert len(v["word_id"]) == 1 and v["child_off"].tolist() == [0, 0]
    p.write_text("10 6 0 0\n")
    assert len(load_orb_vocabulary_txt(str(p))["word_id"]) == 2


@pytest.mark.parametrize("header", ["21 6 0 0", "-1 6 0 0", "10 0 0 0", "10 11 0 0", "10 6 6 0", "10 6 0 4", "10 6 -1 0", "10 6", "x 6 0 0",
                                    "10 6 1 0", "10 6 0 1", "10 6 5 3"])
def test_bad_or_unsupported_header_rejected(tmp_path, header):
    p = tmp_path / "v.txt"
    p.write_text(header + "\n0 1 " + " ".join(["7"] * 32) + " 1.5")
    with pytest.raises(ValueError):
        load_orb_vocabulary_txt(str(p))


@pytest.mark.parametrize("line", ["0 1 " + " ".join(["7"] * 31) + " 1.5",            # a field missing
                                  "0 1 " + " ".join(["7"] * 32) + " 1.5 9",          # one too many
                                  "0 1 " + " ".join(["256"] * 32) + " 1.5",          # not a byte
                                  "0 1 " + " ".join(["7"] * 32) + " abc",            # not a number
                                  "1 1 " + " ".join(["7"] * 32) + " 1.5"])           # its own parent
def test_bad_node_line_rejected(tmp_path, line):
    p = tmp_path / "v.txt"
    p.write_text("10 6 0 0\n" + line)
    with pytest.raises(ValueError):
        load_orb_vocabulary_txt(str(p))


@pytest.mark.skipif(ref_lib.bow_lib() is None, reason="oracle/_ref/libbow_ref.so not built and no reference tree to build it from")
@pytest.mark.parametrize("k,L", [(4, 5), (4, 6), (10, 3), (10, 4), (16, 3)])
def test_oracle_on_loaded_arrays_matches_reference(tmp_path, k, L):
    voc = sl.make_vocabulary(100 + k + L, k=k, L=L)
    path = str(tmp_path / "voc.txt")
    ref_lib.write_vocabulary_txt(voc, path)
    v = load_orb_vocabulary_txt(path)
    rv = ref_lib.RefVocabulary(path)
    for lu in range(L + 2):
        feats = sl.make_features_for_vocabulary(lu + 7 * k, v, 600)
        o, r = oracle_lib.bow_transform(v, feats, lu), rv.transform(feats, lu)
        for key in KEYS:
            assert np.array_equal(o[key], r[key]), (k, L, lu, key)
