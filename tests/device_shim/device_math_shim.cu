// Device build of the product's arithmetic headers (dsac_b200/csrc/*.cuh compiled by nvcc for sm_90a, without
// DSAC_HOST_ONLY): the device twin of tests/host_shim/host_math_shim.cpp.  The host build replaces the device's
// approximate reciprocals and square roots with libm and never contracts a multiply-add; these kernels run the
// functions exactly as the engine's kernels inline them.  One thread per item, arrays in device memory; the launchers
// take device pointers and a stream.  Test infrastructure only; never shipped or used by the product path.
#include <cuda_runtime.h>
#include "../../dsac_b200/csrc/pose_math.cuh"

namespace {
constexpr int kThreads = 128;
inline int blocks(int n) { return (n + kThreads - 1) / kThreads; }

// the sampler filter's verdict: 1 = "needs the full solve", 0 = "certainly rejected"
__global__ void k_needs_full(int n, const float* obj, const float* img, double f, double cx, double cy, int thr,
                             uint8_t* needs_full) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    needs_full[k] = dsac::minimal_set_needs_full(obj + 12 * k, img + 8 * k, f, cx, cy, thr) ? 1 : 0;
}

// the exact solve + 4th-point check: accepted, fragile, pose [n][6] (rvec, tvec)
__global__ void k_minimal_set(int n, const float* obj, const float* img, double f, double cx, double cy, int thr,
                              uint8_t* accepted, uint8_t* fragile, double* pose) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    bool fr = false;
    accepted[k] = dsac::minimal_set_hypothesis(obj + 12 * k, img + 8 * k, f, cx, cy, thr, pose + 6 * k, pose + 6 * k + 3, &fr) ? 1 : 0;
    fragile[k] = fr ? 1 : 0;
}
}  // namespace

extern "C" {
int dev_needs_full(int n, const float* obj, const float* img, double f, double cx, double cy, int thr, uint8_t* needs_full,
                   cudaStream_t stream) {
    if (n > 0) k_needs_full<<<blocks(n), kThreads, 0, stream>>>(n, obj, img, f, cx, cy, thr, needs_full);
    return (int)cudaGetLastError();
}
int dev_minimal_set(int n, const float* obj, const float* img, double f, double cx, double cy, int thr, uint8_t* accepted,
                    uint8_t* fragile, double* pose, cudaStream_t stream) {
    if (n > 0) k_minimal_set<<<blocks(n), kThreads, 0, stream>>>(n, obj, img, f, cx, cy, thr, accepted, fragile, pose);
    return (int)cudaGetLastError();
}
}
