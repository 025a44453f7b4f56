"""CPU: the grey-conversion oracle cvtcolor_oracle.py (Tracking::GrabImageRGBD, src/Tracking.cc:157-172) equals cv2.cvtColor on every (R, G, B)
triple, for the four codes the reference selects from Camera.RGB and the channel count; alpha is seeded noise and must not matter."""
import numpy as np
import pytest

import cvtcolor_oracle

cv2 = pytest.importorskip("cv2")


def all_triples() -> np.ndarray:
    """[4096][4096][3] uint8: every (c0, c1, c2) once, c0 slowest."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("rgb", [True, False])
def test_gray_from_color_equals_cv2_on_every_triple(channels, rgb):
    img = all_triples()
    if channels == 4:
        alpha = np.random.default_rng(11).integers(0, 256, img.shape[:2] + (1,), dtype=np.uint8)
        img = np.concatenate([img, alpha], -1)
    code = {(3, True): cv2.COLOR_RGB2GRAY, (3, False): cv2.COLOR_BGR2GRAY, (4, True): cv2.COLOR_RGBA2GRAY, (4, False): cv2.COLOR_BGRA2GRAY}[(channels, rgb)]
    want = cv2.cvtColor(img, code)
    got = cvtcolor_oracle.gray_from_color(img, rgb)
    assert got.shape == want.shape and np.array_equal(got, want)

