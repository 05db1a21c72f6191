// Host build of the multi-camera rig arithmetic (pose_math.cuh's rig_compose / rig_lift, lm_math.cuh's
// lm_point_contrib_ext) for the CPU-side checks of tests/test_rig_host.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/lm_math.cuh"

extern "C" {
void shim_rig_compose(const double* Rc, const double* tc, const double* R, const double* t, double* Ro, double* to) {
    dsac::rig_compose(Rc, tc, R, t, Ro, to);
}
void shim_rig_lift(const double* Rc, const double* tc, const double* R, const double* t, double* Ro, double* to) {
    dsac::rig_lift(Rc, tc, R, t, Ro, to);
}
// v[0..27] of one point at rig pose `param` (rvec, t); Rc == nullptr: lm_point_contrib (no extrinsic)
void shim_point_contrib(const double* param, const double* Rc, const double* tc, const double* X, const double* pix, double f,
                        double cx, double cy, double* v) {
    double R[9], J[27];
    dsac::rodrigues_jac(param, R, J);
    for (int k = 0; k < 28; k++) v[k] = 0;
    if (Rc) dsac::lm_point_contrib_ext(R, J, param, Rc, tc, X[0], X[1], X[2], pix[0], pix[1], f, cx, cy, v);
    else dsac::lm_point_contrib(R, J, param, X[0], X[1], X[2], pix[0], pix[1], f, cx, cy, v);
}
}
