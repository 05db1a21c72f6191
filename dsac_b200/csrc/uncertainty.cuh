// uncertainty.cuh -- pose uncertainty of the refined poses (dsac_pose_uncertainty_device): the Gauss-Newton covariance of
// each refined pose over the cells its last accepted refinement step fitted (ift.cuh's ift_cov_from_info), and the number
// of cells that agree with the pose.
#pragma once
#include <cuda_runtime.h>

#include "camera.cuh"
#include "ift.cuh"
#include "pose_math.cuh"
#include "refine.cuh"

namespace dsac {

struct UncParams {
    const int16_t* coords;      // [n][N][3]
    const int32_t* pix;
    int pix_stride;
    double f, cx, cy;
    const Cam* cams;            // [n] or null
    const double* eye;          // [n][N][3] (RGB-D) or null
    int jobs_per_frame;         // 1 (soft-argmax) or H (DSAC variant): job j belongs to frame j / jobs_per_frame
                                // (RIG: to rig j / jobs_per_frame; M for the modes of a rig's pool)
    float thr;                  // thr2d, k_score's inlier threshold
    const double* pose;         // [jobs][6] cv pose of the recording replay
    const uint16_t* sel;        // [jobs][K4_MAX_INLIERS] cells of its last accepted step
    const int32_t* count;       // [jobs] their number, 0: no step accepted
    // outputs, each nullable (dsac_pose_uncertainty_out)
    double* cov_jp6;            // [jobs][36]
    double* cov_xi;             // [jobs][36]
    double* sigma2;             // [jobs]
    int32_t* n_fit;             // [jobs]
    int32_t* support;           // [jobs]
    int32_t* ok;                // [jobs]
};
constexpr int UNC_THREADS = 64, UNC_WARPS = UNC_THREADS / 32;

// One CTA per job with k_refine_ift's layout: the lanes own the recorded cells and accumulate the 21 information entries
// and sum |r|^2 (ift_point_gn), and 25 of the 1600 cells each for the support count -- the reprojection error of k_score
// (score_pair_error on the pose's fp32 projection rows, built as k1_write_hyp builds them) below thr2d, every cell with
// or without depth.  The 23 sums are reduced with the transposed butterfly, then the warps in order; one lane does the 6x6
// work in fp64.
// RIG (k_pose_uncertainty_rig, dsac_rig_pose_uncertainty_device and dsac_rig_pose_modes_device): job j belongs to rig
// r = j / jobs_per_frame of rig.C cameras, pose a pose of the rig, sel entries cam << 11 | cell at a stride of
// C K4_MAX_INLIERS per job (k_refine_rig_rec).  A cell is set up in its own camera frame at
// the composed pose and mapped to the rig frame (ift_point_to_rig), as k_refine_ift_rig does; the support counts the cells
// of every camera under its composed pose.  A rig with DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR in rig_status gets zeros.
// RIG with RGBD (k_pose_uncertainty_rig_rgbd, RGB-D rigs): the residual is the cell's 3-vector in its own camera frame
// against its eye point (mm), sigma2 over 3m - 6; the support is the reprojection count, with or without depth.
template <bool PER_FRAME, bool RGBD, bool RIG = false>
__device__ __forceinline__ void k_pose_uncertainty_body(const UncParams& p, RigRefine rig = RigRefine{},
                                                        const uint32_t* rig_status = nullptr) {
    __shared__ double s_red[UNC_WARPS][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int job = blockIdx.x;
    const int frame = job / p.jobs_per_frame;
    const Cam cam = frame_cam<PER_FRAME>(p, frame);
    const int cnt = p.count[job];
    const int n_cams = RIG ? rig.C : 1;
    const uint16_t* sel = p.sel + (size_t)job * n_cams * K4_MAX_INLIERS;
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    if constexpr (RIG) {
        if (rig_status[frame] & RIG_ST_SPOILED) {   // (uniform over the CTA)
            if (tid < 36) {
                if (p.cov_xi) p.cov_xi[(size_t)job * 36 + tid] = 0.0;
                if (p.cov_jp6) p.cov_jp6[(size_t)job * 36 + tid] = 0.0;
            }
            if (tid == 0) {
                if (p.sigma2) p.sigma2[job] = 0.0;
                if (p.n_fit) p.n_fit[job] = 0;
                if (p.support) p.support[job] = 0;
                if (p.ok) p.ok[job] = 0;
            }
            return;
        }
    }
    double pose[6], R[9];
    for (int k = 0; k < 6; k++) pose[k] = p.pose[(size_t)job * 6 + k];
    rodrigues_v2m(pose, R);
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = 0;
    for (int i = tid; i < cnt; i += UNC_THREADS) {
        if constexpr (RIG) {
            const int code = sel[i], fr = frame * n_cams + (code >> 11), cell = code & 2047;
            const int16_t* co = p.coords + ((size_t)fr * DSAC_N_CONST + cell) * 3;
            const int32_t* px = p.pix + (size_t)fr * p.pix_stride + cell * 2;
            const double Y[3] = {(double)co[0], (double)co[1], (double)co[2]};
            double e[3] = {(double)px[0], (double)px[1], 0};
            if constexpr (RGBD) {
                const double* ey = p.eye + ((size_t)fr * DSAC_N_CONST + cell) * 3;
                e[0] = ey[0]; e[1] = ey[1]; e[2] = ey[2];
            }
            const double* E = rig.ext + (size_t)fr * 12;
            double Rk[9], tk[3];
            rig_compose(E, E + 9, R, pose + 3, Rk, tk);
            const Cam cm = frame_cam<PER_FRAME>(p, fr);
            IftPoint P;
            ift_point_setup(Rk, tk, Y, e, cm.f, cm.cx, cm.cy, RGBD, P);
            ift_point_to_rig(E, P);
            ift_point_gn(P, v);
            continue;
        }
        const int c = sel[i];
        const double Y[3] = {(double)coords[c * 3], (double)coords[c * 3 + 1], (double)coords[c * 3 + 2]};
        double e[3];
        if constexpr (RGBD) {
            const double* ey = p.eye + ((size_t)frame * DSAC_N_CONST + c) * 3;
            e[0] = ey[0]; e[1] = ey[1]; e[2] = ey[2];
        } else {
            e[0] = (double)pix[c * 2]; e[1] = (double)pix[c * 2 + 1]; e[2] = 0;
        }
        IftPoint P;
        ift_point_setup(R, pose + 3, Y, e, cam.f, cam.cx, cam.cy, RGBD, P);
        ift_point_gn(P, v);
    }
    if constexpr (RIG) {   // support over every camera, under its composed pose (the rows k_rig_lift gives k_score)
        int sup = 0;
        for (int c2 = 0; c2 < n_cams; c2++) {
            const int fr = frame * n_cams + c2;
            const double* E = rig.ext + (size_t)fr * 12;
            double Rk[9], tk[3];
            rig_compose(E, E + 9, R, pose + 3, Rk, tk);
            const Cam cm = frame_cam<PER_FRAME>(p, fr);
            const float r0x = (float)(cm.f * Rk[0]), r0y = (float)(cm.f * Rk[1]), r0z = (float)(cm.f * Rk[2]), r0w = (float)(cm.f * tk[0]);
            const float r1x = (float)(cm.f * Rk[3]), r1y = (float)(cm.f * Rk[4]), r1z = (float)(cm.f * Rk[5]), r1w = (float)(cm.f * tk[1]);
            const float r2x = (float)Rk[6], r2y = (float)Rk[7], r2z = (float)Rk[8], r2w = (float)tk[2];
            const float cxf = (float)cm.cx, cyf = (float)cm.cy;
            const int16_t* co = p.coords + (size_t)fr * DSAC_N_CONST * 3;
            const int32_t* px = p.pix + (size_t)fr * p.pix_stride;
            for (int c = tid; c < DSAC_N_CONST; c += UNC_THREADS) {
                float az;
                const float err = score_pair_error<true>(r0x, r0y, r0z, r0w, r1x, r1y, r1z, r1w, r2x, r2y, r2z, r2w, (float)co[c * 3],
                                                         (float)co[c * 3 + 1], (float)co[c * 3 + 2], (float)px[c * 2] - cxf,
                                                         (float)px[c * 2 + 1] - cyf, &az);
                sup += err < p.thr ? 1 : 0;
            }
        }
        v[22] = (double)sup;
    } else {   // support
        const float r0x = (float)(cam.f * R[0]), r0y = (float)(cam.f * R[1]), r0z = (float)(cam.f * R[2]), r0w = (float)(cam.f * pose[3]);
        const float r1x = (float)(cam.f * R[3]), r1y = (float)(cam.f * R[4]), r1z = (float)(cam.f * R[5]), r1w = (float)(cam.f * pose[4]);
        const float r2x = (float)R[6], r2y = (float)R[7], r2z = (float)R[8], r2w = (float)pose[5];
        const float cxf = (float)cam.cx, cyf = (float)cam.cy;
        int sup = 0;
        for (int c = tid; c < DSAC_N_CONST; c += UNC_THREADS) {
            float az;
            const float err = score_pair_error<true>(r0x, r0y, r0z, r0w, r1x, r1y, r1z, r1w, r2x, r2y, r2z, r2w, (float)coords[c * 3],
                                                     (float)coords[c * 3 + 1], (float)coords[c * 3 + 2], (float)pix[c * 2] - cxf,
                                                     (float)pix[c * 2 + 1] - cyf, &az);
            sup += err < p.thr ? 1 : 0;
        }
        v[22] = (double)sup;
    }
#pragma unroll
    for (int half = 16, off = 16; half >= 1; half >>= 1, off >>= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (i < half) {
                const double send = up ? v[i] : v[i + half];
                const double keep = up ? v[i + half] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
    }
    s_red[warp][lane] = v[0];
    __syncthreads();
    if (tid == 0) {
        double acc[23], cxi[36], cjp[36], s2;
        for (int k = 0; k < 23; k++) {
            double t = 0;
            for (int w = 0; w < UNC_WARPS; w++) t += s_red[w][k];
            acc[k] = t;
        }
        const bool ok = ift_cov_from_info(acc, acc[21], cnt, RGBD, pose, cxi, cjp, &s2);
        if (p.cov_xi)
            for (int k = 0; k < 36; k++) p.cov_xi[(size_t)job * 36 + k] = cxi[k];
        if (p.cov_jp6)
            for (int k = 0; k < 36; k++) p.cov_jp6[(size_t)job * 36 + k] = cjp[k];
        if (p.sigma2) p.sigma2[job] = s2;
        if (p.n_fit) p.n_fit[job] = cnt;
        if (p.support) p.support[job] = (int32_t)acc[22];
        if (p.ok) p.ok[job] = ok ? 1 : 0;
    }
}
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty(UncParams p) { k_pose_uncertainty_body<false, false>(p); }
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_cam(UncParams p) { k_pose_uncertainty_body<true, false>(p); }
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rgbd(UncParams p) { k_pose_uncertainty_body<false, true>(p); }
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rgbd_cam(UncParams p) { k_pose_uncertainty_body<true, true>(p); }
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rig(UncParams p, RigRefine rig, const uint32_t* status) {
    k_pose_uncertainty_body<false, false, true>(p, rig, status);
}
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rig_cam(UncParams p, RigRefine rig, const uint32_t* status) {
    k_pose_uncertainty_body<true, false, true>(p, rig, status);
}
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rig_rgbd(UncParams p, RigRefine rig, const uint32_t* status) {
    k_pose_uncertainty_body<false, true, true>(p, rig, status);
}
__global__ void __launch_bounds__(UNC_THREADS) k_pose_uncertainty_rig_rgbd_cam(UncParams p, RigRefine rig, const uint32_t* status) {
    k_pose_uncertainty_body<true, true, true>(p, rig, status);
}
// [per-frame camera][RGB-D]
constexpr void (*k_pose_uncertainty_rig_tab[2][2])(UncParams, RigRefine, const uint32_t*) = {
    {k_pose_uncertainty_rig, k_pose_uncertainty_rig_rgbd}, {k_pose_uncertainty_rig_cam, k_pose_uncertainty_rig_rgbd_cam}};

inline void launch_pose_uncertainty(const UncParams& p, unsigned jobs, cudaStream_t stream) {
    // [per-frame camera][RGB-D]
    constexpr void (*tab[2][2])(UncParams) = {{k_pose_uncertainty, k_pose_uncertainty_rgbd}, {k_pose_uncertainty_cam, k_pose_uncertainty_rgbd_cam}};
    tab[p.cams != nullptr][p.eye != nullptr]<<<jobs, UNC_THREADS, 0, stream>>>(p);
}

}  // namespace dsac
