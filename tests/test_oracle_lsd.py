"""CPU: the oracle line-segment detector (oracle/lsd.cc) pinned against the in-container cv2 4.13
cv2.createLineSegmentDetector - the upstream implementation behind the reference's LSDDetector (opencv_contrib
line_descriptor, not vendored in /root/reference; SURVEY.md §8c).

  * LSD_REFINE_NONE and LSD_REFINE_STD: every segment (float32 end points, order included), width and precision must be
    bit-identical (width: to 1 ulp, it carries a double cos / sin).  This pins the Gaussian 7x7 s=0.75 + INTER_LINEAR_EXACT down-scaling, the level-line field, the
    pseudo-ordering, region growing, the rectangle fit and the density refinement.
  * LSD_REFINE_ADV (what the reference runs), oracle variant 3 (cv2 4.13's rect_nfa pixel enumeration + libm rectangle axes):
    every field - end points, order, width, precision and log-NFA - bit-identical on 16 frames.  Variant 1 (same enumeration,
    the deterministic sincos the CUDA path shares): identical except where a 1-ulp axis difference moves a scan-line bound across
    an integer (about one rectangle in a few thousand).
  * LSD_REFINE_ADV, oracle variant 0 (published LSD rectangle iterator - what the CUDA path of this round implements): the
    accepted sets differ for short segments; what the reference consumes - the 40 longest segments
    (src/LSDextractor.cpp:18-26) - must be identical on the frames listed here.
"""
import cv2
import numpy as np
import pytest

import oracle_lib
from depth_cameras import CASES, frames, ramp_band
from planarslam_b200 import synth


def _frames():
    out = [synth.render_frame(seed=s, frame=3 * s)[0] for s in (0, 3, 7)]
    out.append(synth.polygon_image(11))
    return out


@pytest.mark.parametrize("refine,flag", [(0, cv2.LSD_REFINE_NONE), (1, cv2.LSD_REFINE_STD)])
def test_lsd_oracle_bit_exact_vs_cv2(refine, flag):
    for g in _frames():
        segs, width, prec, _ = oracle_lib.lsd_detect(g, refine)
        ref = cv2.createLineSegmentDetector(flag).detect(g)
        assert ref[0] is not None and len(segs) == len(ref[0]) > 50
        assert np.array_equal(segs, ref[0].reshape(-1, 4))
        # width is a double that carries cos / sin of the rectangle angle: the oracle's deterministic sincos (oracle/detmath.h) and
        # cv2's libm agree to 1 ulp
        assert np.allclose(width, ref[1].ravel(), rtol=1e-13, atol=0) and np.array_equal(prec, ref[2].ravel())


def test_lsd_oracle_small_and_flat_images():
    flat = np.full((120, 160), 77, np.uint8)
    assert len(oracle_lib.lsd_detect(flat, 1)[0]) == 0 and cv2.createLineSegmentDetector(cv2.LSD_REFINE_STD).detect(flat)[0] is None
    box = np.zeros((100, 160), np.uint8)
    box[30:70, 40:120] = 200
    segs, width, _, _ = oracle_lib.lsd_detect(box, 1)
    ref = cv2.createLineSegmentDetector(cv2.LSD_REFINE_STD).detect(box)
    assert np.array_equal(segs, ref[0].reshape(-1, 4)) and np.allclose(width, ref[1].ravel(), rtol=1e-13, atol=0)


def _top(segs, k=40):
    length = np.hypot(segs[:, 2] - segs[:, 0], segs[:, 3] - segs[:, 1])
    return segs[np.argsort(-length, kind="stable")[:k]]


def test_lsd_oracle_adv_bit_exact_vs_cv2():
    det = cv2.createLineSegmentDetector(cv2.LSD_REFINE_ADV)
    frames = [synth.render_frame(seed=s, frame=3 * s)[0] for s in range(16)] + [synth.polygon_image(11)]
    n_total = n_same_det = 0
    for g in frames:
        ref = det.detect(g)
        segs, width, prec, nfa = oracle_lib.lsd_detect(g, 2, rect_enum=3)
        assert len(segs) == len(ref[0]) > 50
        assert np.array_equal(segs, ref[0].reshape(-1, 4))
        assert np.array_equal(width, ref[1].ravel()) and np.array_equal(prec, ref[2].ravel()) and np.array_equal(nfa, ref[3].ravel())
        # same enumeration with the deterministic sincos: the segment lists may differ by the odd borderline rectangle
        segs1 = oracle_lib.lsd_detect(g, 2, rect_enum=1)[0]
        a, b = {s.tobytes() for s in segs1}, {s.tobytes() for s in segs}
        n_total += len(b)
        n_same_det += len(a & b)
        assert np.array_equal(_top(segs1), _top(segs))
    assert n_same_det >= n_total - 8, (n_same_det, n_total)


def test_lsd_oracle_adv_top40_matches_cv2():
    for s in range(16):                                            # default oracle enumeration = cv2 4.x rect_nfa (the CUDA path's default)
        g = synth.render_frame(seed=s, frame=3 * s)[0]
        segs = oracle_lib.lsd_detect(g, 2)[0]
        ref = cv2.createLineSegmentDetector(cv2.LSD_REFINE_ADV).detect(g)[0].reshape(-1, 4)
        assert np.array_equal(_top(segs), _top(ref)), s


def test_extract_line_segments_keylines():
    g = synth.render_frame(seed=7, frame=21)[0]
    kl, lf = oracle_lib.extract_line_segments(g, 40)
    assert len(kl) == 40 and np.array_equal(kl["class_id"], np.arange(40))
    assert (np.diff(kl["response"]) <= 0).all()                      # sorted by response = length / max(w, h)
    ref = cv2.createLineSegmentDetector(cv2.LSD_REFINE_ADV).detect(g)[0].reshape(-1, 4)
    top = _top(ref)
    assert np.array_equal(np.stack([kl["startPointX"], kl["startPointY"], kl["endPointX"], kl["endPointY"]], 1), top)
    # line functions: sp x ep normalised (src/LSDextractor.cpp:30-38)
    sp = np.stack([kl["startPointX"], kl["startPointY"], np.ones(40)], 1).astype(np.float64)
    ep = np.stack([kl["endPointX"], kl["endPointY"], np.ones(40)], 1).astype(np.float64)
    l = np.cross(sp, ep)
    assert np.allclose(lf, l / np.linalg.norm(l, axis=1, keepdims=True), rtol=1e-14, atol=0)
    assert np.allclose(kl["lineLength"], np.hypot(top[:, 0] - top[:, 2], top[:, 1] - top[:, 3]), rtol=1e-6)


def test_lsd_oracle_other_image_sizes_vs_cv2():
    """1280 x 960 (BASELINE config 5), 320 x 240, and sizes whose 0.8-scaled dimensions are not integers (641 x 479, 333 x 251): the down-scaling samples with
    step 1 / 0.8 while the destination size is cvRound(0.8 * size) - cv::resize(..., Size(), 0.8, 0.8, INTER_LINEAR_EXACT).  Also every size of
    depth_cameras.CASES (644 x 482, 640 x 481 and 120 x 117 scale to 515 x 386, 512 x 385 and 96 x 94), and the ramp-band frames whose one rectangle holds
    more than 8192 pixels (the NFA's large-n path), in all three refinement modes."""
    cases = [(synth.render_frame(seed=2, frame=6, width=1280, height=960)[0], 100), (synth.render_frame(seed=3, frame=9, width=320, height=240)[0], 100)]
    base = synth.render_frame(seed=5, frame=15)[0]
    cases += [(np.ascontiguousarray(np.pad(base[:479], ((0, 0), (0, 1)), mode="edge")), 100), (np.ascontiguousarray(base[100:351, 200:533]), 100)]
    for w, h in sorted({c[:2] for c in CASES.values()}):
        cases.append((frames(next(k for k, c in CASES.items() if c[:2] == (w, h)), 1)[0][0], 20 if w * h < 320 * 240 else 100))
    for w, h in ((640, 480), (1280, 960)):
        cases += [(ramp_band(w, h, tilt, noise=noise), 1) for tilt in (0.0, 3.0) for noise in (0.0, 8.0)]
    for g, min_segs in cases:
        for refine, flag in ((0, cv2.LSD_REFINE_NONE), (1, cv2.LSD_REFINE_STD), (2, cv2.LSD_REFINE_ADV)):
            segs, width, prec, nfa = oracle_lib.lsd_detect(g, refine, cap=65536, rect_enum=3)
            ref = cv2.createLineSegmentDetector(flag).detect(g)
            assert len(segs) == len(ref[0]) >= min_segs, g.shape
            assert np.array_equal(segs, ref[0].reshape(-1, 4)) and np.array_equal(width, ref[1].ravel()) and np.array_equal(prec, ref[2].ravel()), g.shape
            if refine == 2:
                assert np.array_equal(nfa, ref[3].ravel()), g.shape


def test_lsd_oracle_fuzz_sizes_and_content_vs_cv2():
    """Random image sizes (24 .. 420 x 24 .. 320) and content (noise, blurred noise, filled polygons, crops of the synthetic room): all three refinement
    modes identical to cv2 in every field (180 such cases were run when the enumeration was pinned; 24 are kept here)."""
    rng = np.random.default_rng(1)
    for it in range(24):
        w, h = int(rng.integers(24, 420)), int(rng.integers(24, 320))
        kind = it % 4
        if kind == 0:
            g = rng.integers(0, 256, (h, w), dtype=np.uint8)
        elif kind == 1:
            g = cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (0, 0), 3)
        elif kind == 2:
            g = np.zeros((h, w), np.uint8)
            for _ in range(6):
                cv2.fillPoly(g, [rng.integers(0, [w, h], (4, 2)).astype(np.int32)], int(rng.integers(40, 255)))
        else:
            g = synth.render_frame(seed=it, frame=it)[0][:h, :w].copy()
        for refine, flag in ((0, cv2.LSD_REFINE_NONE), (1, cv2.LSD_REFINE_STD), (2, cv2.LSD_REFINE_ADV)):
            segs, width, prec, nfa = oracle_lib.lsd_detect(g, refine, cap=65536, rect_enum=3)
            ref = cv2.createLineSegmentDetector(flag).detect(g)
            if ref[0] is None:
                assert len(segs) == 0, (it, refine)
                continue
            assert np.array_equal(segs, ref[0].reshape(-1, 4)) and np.array_equal(width, ref[1].ravel()) and np.array_equal(prec, ref[2].ravel()), (it, refine, w, h)
            if refine == 2:
                assert np.array_equal(nfa, ref[3].ravel()), (it, w, h)
