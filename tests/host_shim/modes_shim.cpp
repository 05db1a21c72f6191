// Host build of the pose modes' nearness test and ranking key (dsac_b200/csrc/modes.cuh, compiled with DSAC_HOST_ONLY)
// for tests/test_pose_modes_host.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/modes.cuh"

extern "C" {
double shim_mode_angle(const double* Ra, const double* Rb) { return dsac::mode_angle(Ra, Rb); }
double shim_mode_dist(const double* ta, const double* tb) { return dsac::mode_dist(ta, tb); }
int shim_mode_near(const double* Ra, const double* ta, const double* Rb, const double* tb, double rot, double trans) {
    return dsac::mode_near(Ra, ta, Rb, tb, rot, trans) ? 1 : 0;
}
unsigned long long shim_mode_rank_key(int occupied, double score) { return dsac::mode_rank_key(occupied != 0, score); }
}
