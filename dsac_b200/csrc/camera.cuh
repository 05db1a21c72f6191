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

}  // namespace dsac
