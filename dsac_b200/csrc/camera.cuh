// camera.cuh -- the camera a kernel uses for one frame: the engine's, or the frame's own (dsac_set_cameras).
#pragma once
#include <cuda_runtime.h>

namespace dsac {

// Camera of one frame (getCamMat(), properties.cpp:308-323); the layout of dsac_camera (include/dsac_b200.h).
struct Cam {
    double f, cx, cy;
};

// The camera of `frame` for a kernel whose parameters P hold the engine's camera (f, cx, cy) and the nullable per-frame
// table `cams` of the pass (dsac_set_cameras), indexed like coords.  PER_FRAME selects between two instantiations of the
// kernels that are register- or issue-bound, so that the one launched without a table keeps its camera in the constant
// bank; the job kernels branch once per job instead (the second overload).
template <bool PER_FRAME, typename P>
__device__ __forceinline__ Cam frame_cam(const P& p, int frame) {
    if constexpr (PER_FRAME) return p.cams[frame];
    else return Cam{p.f, p.cx, p.cy};
}
template <typename P>
__device__ __forceinline__ Cam frame_cam(const P& p, int frame) {
    return p.cams ? p.cams[frame] : Cam{p.f, p.cx, p.cy};
}

// The fp32 projection rows (f R0 | f t0), (f R1 | f t1), (R2 | t2) of a pose that k_score reads (hyp_P), as every writer of
// hyp_P builds them (the sampler's selection, k1_focal_rows_cam, k_prior_inject, k_rig_lift): each entry is the fp64
// product rounded once to float.  pose_rows_f: the two rows that depend on the focal length.
__device__ __forceinline__ void pose_rows_f(double f, const double R[9], const double t[3], float* P12) {
    float4* P = reinterpret_cast<float4*>(P12);
    P[0] = make_float4((float)(f * R[0]), (float)(f * R[1]), (float)(f * R[2]), (float)(f * t[0]));
    P[1] = make_float4((float)(f * R[3]), (float)(f * R[4]), (float)(f * R[5]), (float)(f * t[1]));
}
__device__ __forceinline__ void pose_rows(double f, const double R[9], const double t[3], float* P12) {
    pose_rows_f(f, R, t, P12);
    reinterpret_cast<float4*>(P12)[2] = make_float4((float)R[6], (float)R[7], (float)R[8], (float)t[2]);
}

}  // namespace dsac
