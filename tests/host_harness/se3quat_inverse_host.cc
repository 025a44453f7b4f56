// Test-only: T = Converter::toSE3Quat(Tcw).inverse() (MapPlane::UpdateCoefficientsAndPoints(const Frame&, int)) from the oracle's SE3Quat restatement
// (oracle/g2o_math.h), for tests/test_track_planar_mapplanes_gpu.py's host replay of the planar chain's map plane updates.  Eigen is absent, so the
// inverse's order of operations is the parity convention of DESIGN.md section 5: [R'^T | -(R'^T t)], R' = quat_to_matrix(qnormalized_pos(quat_from_matrix(R))).
#include "g2o_math.h"

using namespace oracle::gm;

// Tcw: float [4][4] row-major; out: double [4][4] row-major
extern "C" void host_se3quat_inverse(const float* Tcw, double* out) {
    M3 R;
    for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) R.m[r][q] = (double)Tcw[4 * r + q];
    const V3 t{(double)Tcw[3], (double)Tcw[7], (double)Tcw[11]};
    const SE3 T = se3_from_Rt(R, t);
    const M3 Rt = transpose(quat_to_matrix(T.q));
    const V3 ti = mul(Rt, T.t);
    const double tv[3] = {-ti.x, -ti.y, -ti.z};
    for (int r = 0; r < 3; ++r) {
        for (int q = 0; q < 3; ++q) out[4 * r + q] = Rt.m[r][q];
        out[4 * r + 3] = tv[r];
    }
    out[12] = 0; out[13] = 0; out[14] = 0; out[15] = 1;
}
