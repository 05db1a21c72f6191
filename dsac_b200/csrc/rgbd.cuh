// rgbd.cuh -- RGB-D localisation (dsac_set_cell_depth_device): the per-pass eye coordinates of the cells and the test for
// frames without enough depth.  The acceptance test and the rigid fit are in rigid.cuh, the sampler kernels that use them
// in kernels.cuh (k_sample_t), sampler_split.cuh (k1_slot_rgbd, k1_kabsch) and guided.cuh (k1_gtail_t), the refinement in
// refine.cuh (k_refine_rgbd).
#pragma once
#include <cuda_runtime.h>

#include "camera.cuh"
#include "rigid.cuh"

namespace dsac {

constexpr int KE_THREADS = 256;

// One CTA per frame.  eye [n][N][3]: X_eye = ((u - cx) d / f, (v - cy) d / f, d) in fp64 for a cell whose depth d (mm) is
// finite and > 0, NaN otherwise; (u, v) is the cell's pixel, (f, cx, cy) the frame's camera.  skip [n]: DSAC_ST_NO_DEPTH
// when fewer than 4 cells have depth, | DSAC_ST_BAD_WEIGHTS when the guided sampler's table flags the frame (gbad may be null).
template <bool PER_FRAME>
__global__ void __launch_bounds__(KE_THREADS) k_rgbd_eye_t(const float* __restrict__ depth, const int32_t* __restrict__ pix, int pix_stride,
                                                         Cam cam0, const Cam* __restrict__ cams, const uint32_t* __restrict__ gbad,
                                                         double* __restrict__ eye, uint32_t* __restrict__ skip) {
    const int frame = blockIdx.x;
    const Cam cam = PER_FRAME ? cams[frame] : cam0;
    const float* d = depth + (size_t)frame * DSAC_N_CONST;
    const int32_t* px = pix + (size_t)frame * pix_stride;
    double* e = eye + (size_t)frame * DSAC_N_CONST * 3;
    __shared__ int s_have;
    if (threadIdx.x == 0) s_have = 0;
    __syncthreads();
    int have = 0;
    for (int c = threadIdx.x; c < DSAC_N_CONST; c += KE_THREADS) {
        const float z = d[c];
        double X = NAN, Y = NAN, Z = NAN;
        if (isfinite(z) && z > 0.f) {
            Z = (double)z;
            X = ((double)px[c * 2] - cam.cx) * Z / cam.f;
            Y = ((double)px[c * 2 + 1] - cam.cy) * Z / cam.f;
            have++;
        }
        e[c * 3] = X; e[c * 3 + 1] = Y; e[c * 3 + 2] = Z;
    }
    if (have) atomicAdd(&s_have, have);
    __syncthreads();
    if (threadIdx.x == 0) skip[frame] = (s_have < 4 ? ST_NO_DEPTH : 0u) | ((gbad && gbad[frame]) ? 32u /* DSAC_ST_BAD_WEIGHTS */ : 0u);
}

}  // namespace dsac
