"""CPU oracle of the grey conversion of Tracking::GrabImageRGBD (src/Tracking.cc:157-172): cv::cvtColor(RGB / BGR / RGBA / BGRA -> GRAY) on 8-bit
images, restated from OpenCV's published 8-bit path (imgproc color_rgb, RGB2Gray<uchar>): 15-bit fixed-point weights of 0.299 / 0.587 / 0.114, rounded so
that they sum to 2^15, plus one half and a shift; alpha is not read.  Pinned against cv2 4.13 on all 2^24 (R, G, B) triples by
test_oracle_gray_from_color.py.  Test infrastructure only."""
from __future__ import annotations

import numpy as np

R2Y, G2Y, B2Y, SHIFT = 9798, 19235, 3735, 15


def gray_from_color(image: np.ndarray, rgb: bool = True) -> np.ndarray:
    """uint8 [..., 3|4] -> uint8 [...]; rgb = Camera.RGB (True: the first byte of a pixel is R, False: it is B)."""
    image = np.asarray(image)
    assert image.dtype == np.uint8 and image.shape[-1] in (3, 4)
    c = [image[..., k].astype(np.uint32) for k in range(3)]
    r, g, b = (c[0], c[1], c[2]) if rgb else (c[2], c[1], c[0])
    return ((R2Y * r + G2Y * g + B2Y * b + (1 << (SHIFT - 1))) >> SHIFT).astype(np.uint8)
