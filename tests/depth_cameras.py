"""The cameras and image sizes the depth products of the RGB-D Frame constructor (plane post-processing, surface normals, stereo, isLineGood) are tested
at, shared by the CPU statement of the normals and the GPU comparison.  Test infrastructure only.

K values are the float32 numbers a Context holds: the reference's yaml settings (Examples/RGB-D/*.yaml), or TUM3 scaled to the frame width the way
pslam_default_config scales it (535.4f * (width / 640.f)).  A Context needs a width that is a multiple of 4, so the odd shapes are 644x482 (w % 3 = 2,
W3 = 215 and H3 = 161, both odd) and 640x481 (h % 3 = 1, H3 odd); 120x117 is the smallest frame a Context with nlevels=4 accepts (every pyramid level
must be at least 68 pixels on a side; 320x240 runs with nlevels=7 for the same reason).  ramp_band draws the LSD frames whose rectangles leave the NFA
tables (the image-side tests and the oracle's cv2 pin share them)."""
from __future__ import annotations

import numpy as np

from planarslam_b200 import synth

f32 = np.float32


def _scaled_tum3(width: int):
    s = f32(width) / f32(640.0)
    return tuple(float(f32(k) * s) for k in synth.TUM3_K)


def _k(*v):
    return tuple(float(f32(x)) for x in v)


# name: (width, height, (fx, fy, cx, cy), DepthMapFactor, Context overrides)
CASES = {
    "tum3": (640, 480, _k(*synth.TUM3_K), 5000.0, {}),
    "icl": (640, 480, _k(*synth.ICL_K), 5000.0, {}),
    "tum2": (640, 480, _k(520.908620, 521.007327, 325.141442, 249.701764), 5208.0, {}),
    "tamu": (640, 480, _k(525.0, 525.0, 319.5, 239.5), 5000.0, {}),
    "config5": (1280, 960, _scaled_tum3(1280), 5000.0, {"nfeatures": 2000}),
    "odd_644x482": (644, 482, _scaled_tum3(644), 5000.0, {}),
    "odd_640x481": (640, 481, _scaled_tum3(640), 5000.0, {}),
    "small_320x240": (320, 240, _scaled_tum3(320), 5000.0, {"nlevels": 7}),
    "min_120x117": (120, 117, _scaled_tum3(120), 5000.0, {"nlevels": 4}),
}


def scale_of(factor: float) -> float:
    """mDepthMapFactor = 1 / DepthMapFactor, as the float the reference and the Context hold."""
    return float(f32(1.0) / f32(factor))


def frames(case: str, n: int, zero_slot: int | None = None, seed: int = 2):
    """n frames of the room-corner sequence rendered through the case's camera: (gray uint8 [n][h][w], depth uint16 [n][h][w]); the depth frame at
    zero_slot is all zero (no plane, every normal NaN)."""
    w, h, K, _, _ = CASES[case]
    g, d = np.zeros((n, h, w), np.uint8), np.zeros((n, h, w), np.uint16)
    for i in range(n):
        gi, di, _, _ = synth.render_frame(seed, 9 * i + 3, w, h, K=K)
        g[i] = gi
        if i != zero_slot:
            d[i] = di
    return g, d


def ramp_band(w: int, h: int, tilt_deg: float = 0.0, band: float = 40.0, noise: float = 0.0, seed: int = 1) -> np.ndarray:
    """uint8 frame with one straight intensity ramp, 0 -> 255 over `band` pixels, across the whole frame through its centre, tilted by tilt_deg from the
    vertical; flat 0 on one side and 255 on the other, plus seeded Gaussian noise of standard deviation `noise` grey levels.  LSD finds one segment as long
    as the frame whose rectangle covers about (0.8 h) x (0.8 band) pixels of the scaled image: over 8192 at 640x480, so its NFA is evaluated outside the
    n <= 512 table and the n + 1 < 8192 log-gamma table.  Without noise nearly every pixel of the rectangle is aligned, so the three log-gamma terms of
    log C(n, k) almost cancel; noise leaves more of the pixels unaligned, and then an error in those terms shows in the log-NFA."""
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    t = np.deg2rad(tilt_deg)
    d = (u - (w - 1) / 2) * np.cos(t) + (v - (h - 1) / 2) * np.sin(t)
    x = 255.0 * np.clip(d / band + 0.5, 0.0, 1.0)
    if noise:
        x += np.random.default_rng(seed).normal(0.0, noise, x.shape)
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)
