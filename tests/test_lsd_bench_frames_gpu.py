"""GPU: the line-segment detector on frames of the benchmark's scene (synth seed 2, the sequence bench.py replays) against the CPU oracle, in all three
refinement modes.  Bar as in tests/test_lsd_gpu.py: bit-exact segments, widths and precisions, log-NFA to 1e-9."""
import numpy as np
import pytest

import oracle_lib
from planarslam_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("refine", [0, 1, 2])
def test_lsd_bench_frames_match_oracle(refine):
    from planarslam_b200.lines import LineSegment
    g = np.stack([synth.render_frame(2, f)[0] for f in (0, 57, 131, 250)])
    ls = LineSegment(max_batch=len(g))
    res = ls.detect(g, refine)
    for f in range(len(g)):
        segs, width, prec, nfa = res[f]
        osegs, owidth, oprec, onfa = oracle_lib.lsd_detect(g[f], refine)
        assert len(segs) == len(osegs) > 50, (f, len(segs), len(osegs))
        assert np.array_equal(segs, osegs), f
        assert np.array_equal(width, owidth) and np.array_equal(prec, oprec), f
        assert np.allclose(nfa, onfa, rtol=1e-9, atol=1e-9), f
