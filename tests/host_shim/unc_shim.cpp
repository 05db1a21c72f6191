// Host build of the pose covariance (dsac_b200/csrc/ift.cuh's ift_fit_covariance, compiled with DSAC_HOST_ONLY) for
// tests/test_pose_uncertainty_host.py and tests/test_gpu_pose_uncertainty.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/ift.cuh"

extern "C" {
int shim_ift_fit_covariance(int m, const double* Y, const double* e, const double* pose, double f, double cx, double cy, int rgbd,
                            double* cov_xi, double* cov_jp6, double* sigma2) {
    return dsac::ift_fit_covariance(m, Y, e, pose, f, cx, cy, rgbd != 0, cov_xi, cov_jp6, sigma2) ? 1 : 0;
}
}
