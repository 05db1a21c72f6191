// Host build of the pose priors' gate (dsac_b200/csrc/prior.cuh, compiled with DSAC_HOST_ONLY) for
// tests/test_pose_priors_host.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/prior.cuh"

extern "C" {
// d2[j] of the cv pose (rvec, tvec) against each of the k priors (poses [k][6], info [k][36]); returns 1, or 0 with d2
// untouched when an entry is refused.
int shim_prior_d2(int k, const double* poses, const double* info, const double* pose, double* d2) {
    double R[9];
    dsac::rodrigues_v2m(pose, R);
    for (int j = 0; j < k; j++) {
        dsac::PriorGate g;
        if (!dsac::prior_entry(poses + j * 6, info + j * 36, g)) return 0;
        d2[j] = dsac::prior_d2(R, pose + 3, g);
    }
    return 1;
}
int shim_prior_gate_pass(int k, const double* poses, const double* info, double chi2, const double* pose) {
    dsac::PriorGate g[dsac::PRIOR_MAX];
    for (int j = 0; j < k; j++)
        if (!dsac::prior_entry(poses + j * 6, info + j * 36, g[j])) return -1;
    return dsac::prior_gate_pass(g, k, chi2, pose, pose + 3) ? 1 : 0;
}
void shim_so3_log(const double* M, double* w) { dsac::so3_log(M, w); }
int shim_prior_cholesky(const double* info, double* L) { return dsac::prior_cholesky(info, L) ? 1 : 0; }
}
