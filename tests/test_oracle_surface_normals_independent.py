"""CPU: the surface normals and the voxel grid of the plane post-processing oracle (oracle/planepost.cc) against plain numpy statements of the same
operations, at every camera and image size of depth_cameras.CASES (and below the smallest size a Context accepts, where the 10-point border covers the
whole sub-sampled grid).

The normals statement restates IntegralImageNormalEstimation (AVERAGE_3D_GRADIENT, max depth change factor 0.05, normal smoothing size 10) without
integral images: the organised cloud of every third pixel, the depth-change mask by the reference loop's neighbour rules, the two chamfer passes in float
(rw = int(min(distance, 10)) is a discrete decision, so the distances keep the float roundings), central-difference gradients that are zero on the image
border, and a direct float64 sum of the finite gradient triples over the window rows / columns [i - rw // 2, i - rw // 2 + rw).  So an off-by-one in the
oracle's rectangle corners, window size or depth-change rules shows up here, even where the CUDA kernels share it.  PARITY UNPINNED against PCL itself."""
import numpy as np
import pytest

import oracle_lib
from depth_cameras import CASES, frames, scale_of

f32 = np.float32


def normals_statement(depth: np.ndarray, K, scale: float) -> np.ndarray:
    """vSurfaceNormal of a uint16 depth frame: float32 [n][8] = normal, camera position, frame position (u, v)."""
    h, w = depth.shape
    fx, fy, cx, cy = (f32(k) for k in K)
    W, H = -(-w // 3), -(-h // 3)
    # organised cloud of pixels (3 r, 3 c), in float as the reference's imDepth (CV_32F) and its back-projection
    z = depth[::3, ::3].astype(f32) * f32(scale)
    x = (np.arange(0, w, 3, dtype=f32)[None, :] - cx) * z / fx
    y = (np.arange(0, h, 3, dtype=f32)[:, None] - cy) * z / fy
    P = np.stack([x, y, z], -1)
    assert P.shape == (H, W, 3) and P.dtype == f32
    # depth-change mask: the loop over (r, c) with r < H - 1, c < W - 1 clears a point and its right (lower) neighbour when that step exceeds the tolerance
    dep = z[:-1, :-1]
    tol = f32(0.05) * (np.abs(dep) + f32(1.0)) * f32(2.0)
    right, down = z[:-1, 1:], z[1:, :-1]
    step_r = (np.abs(dep - right) > tol) | ~np.isfinite(dep) | ~np.isfinite(right)
    step_d = (np.abs(dep - down) > tol) | ~np.isfinite(dep) | ~np.isfinite(down)
    edge = np.zeros((H, W), bool)
    edge[:-1, :-1] |= step_r | step_d
    edge[:-1, 1:] |= step_r
    edge[1:, :-1] |= step_d
    # chamfer distance to the nearest edge, on the flat row-major map as the reference walks it: the forward pass reads the upper-right neighbour of the
    # last column from the next row's first element, the backward pass the lower-left neighbour of the first column from the previous row's last one
    flat = np.where(edge, f32(0.0), f32(W + H)).astype(f32).ravel()
    one, diag = f32(1.0), f32(1.4)
    for r in range(1, H):
        for c in range(1, W):
            i, up = r * W + c, (r - 1) * W + c
            cand = min(flat[up - 1] + diag, flat[up] + one, flat[up + 1] + diag, flat[i - 1] + one)
            if cand < flat[i]:
                flat[i] = cand
    for r in range(H - 2, -1, -1):
        for c in range(W - 2, -1, -1):
            i, lo = r * W + c, (r + 1) * W + c
            cand = min(flat[lo - 1] + diag, flat[lo] + one, flat[lo + 1] + diag, flat[i + 1] + one)
            if cand < flat[i]:
                flat[i] = cand
    dist = flat.reshape(H, W)
    # central differences, zero on the border; a triple with a non-finite component does not enter the sums
    gx, gy = np.zeros_like(P), np.zeros_like(P)
    gx[1:-1, 1:-1] = P[1:-1, 2:] - P[1:-1, :-2]
    gy[1:-1, 1:-1] = P[2:, 1:-1] - P[:-2, 1:-1]
    gx = np.where(np.isfinite(gx).all(-1, keepdims=True), gx, 0).astype(np.float64)
    gy = np.where(np.isfinite(gy).all(-1, keepdims=True), gy, 0).astype(np.float64)
    nrm = np.full((H, W, 3), np.nan, f32)
    border = 10
    smoothing = np.minimum(dist, f32(10.0))
    rw_all = smoothing.astype(np.int64)
    for rr in range(border, H - border):
        for cc in range(border, W - border):
            if not np.isfinite(P[rr, cc, 2]) or not smoothing[rr, cc] > f32(2.0):
                continue
            rw = int(rw_all[rr, cc])
            r0, c0 = rr - rw // 2, cc - rw // 2
            sx = gx[r0:r0 + rw, c0:c0 + rw].sum((0, 1))
            sy = gy[r0:r0 + rw, c0:c0 + rw].sum((0, 1))
            n = np.cross(sy, sx)
            ln = float(n @ n)
            if ln == 0.0:
                continue
            n = (n / np.sqrt(ln)).astype(f32)
            v = -P[rr, cc]
            if (v[0] * n[0] + v[1] * n[1]) + v[2] * n[2] < 0:       # flipped towards the view point (the origin)
                n = -n
            nrm[rr, cc] = n
    out = []
    for m in range(1, H, 2):
        for c in range(1, W, 2):
            out.append(np.concatenate([nrm[m, c], P[m, c], [f32(3 * c), f32(3 * m)]]).astype(f32))
    return np.array(out, f32).reshape(-1, 8)


def _check_normals(depth, K, scale):
    osn = oracle_lib.surface_normals(depth, K, f32(scale))
    ref = normals_statement(depth, K, scale)
    assert osn.shape == ref.shape
    assert np.array_equal(np.isnan(osn), np.isnan(ref))
    ok = np.isfinite(ref)
    assert np.abs(osn[ok] - ref[ok]).max(initial=0.0) <= 1e-6
    assert np.array_equal(osn[:, 3:], ref[:, 3:])                                  # camera and frame positions: identical
    return osn


@pytest.mark.parametrize("case", sorted(CASES))
def test_surface_normals_match_the_numpy_statement(case):
    w, h, K, factor, _ = CASES[case]
    _, depth = frames(case, 3, zero_slot=1)
    H3, W3 = (h + 2) // 3, (w + 2) // 3
    finite = 0
    for f in range(len(depth)):
        osn = _check_normals(depth[f], K, scale_of(factor))
        assert len(osn) == (W3 // 2) * (H3 // 2)
        if f == 1:
            assert np.isnan(osn[:, :3]).all()                                         # all-zero depth: no gradient anywhere
        else:
            finite += int(np.isfinite(osn[:, 0]).sum())
    assert finite > (0.25 if min(W3, H3) > 60 else 0.02) * 2 * len(osn)


@pytest.mark.parametrize("shape", [(64, 48), (62, 59), (68, 68)])
def test_surface_normals_at_the_border_sizes(shape):
    """H3 - 10 <= 10 (64x48, 62x59): the border takes the whole grid and every normal is NaN; 68x68: a 3x3 interior."""
    w, h = shape
    s = f32(w) / f32(640.0)
    K = tuple(float(f32(k) * s) for k in (535.4, 539.2, 320.1, 247.6))
    depth = np.repeat((10000 + 20 * np.arange(w)).astype(np.uint16)[None, :], h, 0)      # a tilted plane without depth edges
    osn = _check_normals(depth, K, scale_of(5000.0))
    H3, W3 = (h + 2) // 3, (w + 2) // 3
    assert len(osn) == (W3 // 2) * (H3 // 2)
    assert np.isnan(osn[:, :3]).all() == (H3 - 10 <= 10)


def voxel_centroids(depth, K, scale, members):
    """pcl::VoxelGrid (leaf 0.1) of the member pixels' float vertices, in ascending voxel index: (centroids as the float64 mean of the coordinates,
    centroids as the exact mean of the coordinates quantised to 2^-20 m rounded to float32, member counts)."""
    h, w = depth.shape
    v, u = np.divmod(members, w)
    zz = depth.ravel()[members].astype(np.float64) * float(f32(scale))
    X = np.stack([(u - float(f32(K[2]))) * zz / float(f32(K[0])), (v - float(f32(K[3]))) * zz / float(f32(K[1])), zz], 1).astype(f32)
    key = np.floor(X * f32(10.0)).astype(np.int64)
    key -= key.min(0)
    dims = key.max(0) + 1
    lin = key[:, 0] + key[:, 1] * dims[0] + key[:, 2] * dims[0] * dims[1]
    order = np.argsort(lin, kind="stable")
    _, start, count = np.unique(lin[order], return_index=True, return_counts=True)
    Xs = X[order]
    mean = np.add.reduceat(Xs.astype(np.float64), start, 0) / count[:, None]
    q = np.add.reduceat(np.rint(Xs.astype(np.float64) * 2.0 ** 20).astype(np.int64), start, 0)
    exact = (q.astype(np.float64) / (count[:, None] * 2.0 ** 20)).astype(f32)
    return mean, exact, count


@pytest.mark.parametrize("case", sorted(CASES))
def test_voxel_grid_against_numpy(case):
    w, h, K, factor, _ = CASES[case]
    _, depth = frames(case, 1)
    scale = scale_of(factor)
    planes = oracle_lib.planes_post(depth[0], K, f32(scale))
    po = oracle_lib.PeacOracle(depth[0], K, f32(scale))
    if w * h >= 320 * 240:
        assert len(planes) >= 2
    for P in planes:
        mean, exact, _ = voxel_centroids(depth[0], K, scale, po.membership[P["src"]])
        assert len(mean) == len(P["points"])
        assert np.abs(mean - P["points"]).max() < 2e-5                              # float vs double accumulation
        assert np.array_equal(exact, P["points"])                                   # the oracle's order-free fixed-point sum, exactly
