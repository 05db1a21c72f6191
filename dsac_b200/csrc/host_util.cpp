// host_util.cpp -- host-side helpers of the C ABI that carry the reference's RNG contract
// and the synthetic-input generator of SURVEY.md section 8(d).  No device code.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <random>
#include <vector>

#include "../../include/dsac_b200.h"
#define DSAC_HOST_ONLY 1
#include "pose_math.cuh"

namespace {

// xoshiro256** seeded by splitmix64: self-contained so the synthetic data does not depend
// on any library's distribution implementations.
struct Rng {
    uint64_t s[4];
    static uint64_t splitmix(uint64_t& x) {
        uint64_t z = (x += 0x9e3779b97f4a7c15ull);
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        return z ^ (z >> 31);
    }
    explicit Rng(uint64_t seed) {
        for (int i = 0; i < 4; i++) s[i] = splitmix(seed);
    }
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    uint64_t next() {
        uint64_t r = rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return r;
    }
    double uni() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
    double uni(double a, double b) { return a + (b - a) * uni(); }
    double gauss() {
        double u1 = uni(), u2 = uni();
        if (u1 < 1e-300) u1 = 1e-300;
        return std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586 * u2);
    }
};

inline int16_t sat16(double v) {
    double r = std::nearbyint(v);
    if (r > 32767) r = 32767;
    if (r < -32768) r = -32768;
    return (int16_t)r;
}

}  // namespace

extern "C" {

// train_obj.cpp:266-270: iota(n), then std::shuffle with std::mt19937(seed) (the reference's is default-seeded: 5489).
// Compiled by the host compiler so that the permutation is libstdc++'s own.
int dsac_shuffle_permutation(int32_t n, uint32_t seed, int32_t* out) {
    if (n < 1 || !out) return DSAC_ERR_ARG;
    std::vector<int> v((size_t)n);
    for (int i = 0; i < n; i++) v[(size_t)i] = i;
    std::mt19937 gen(seed);
    std::shuffle(v.begin(), v.end(), gen);
    for (int i = 0; i < n; i++) out[i] = v[(size_t)i];
    return DSAC_OK;
}

// train_score.cpp:286,381-384: one std::mt19937(seed) that continues across the training rounds, each round a
// std::shuffle of a fresh iota(n).  Writes the permutations of rounds first_round .. first_round + n_rounds - 1,
// replaying the earlier rounds from the seed.
int dsac_shuffle_permutations(int32_t n, uint32_t seed, int32_t first_round, int32_t n_rounds, int32_t* out) {
    if (n < 1 || first_round < 0 || n_rounds < 1 || !out) return DSAC_ERR_ARG;
    std::mt19937 gen(seed);
    std::vector<int> v((size_t)n);
    for (int32_t r = 0; r < first_round + n_rounds; r++) {
        for (int i = 0; i < n; i++) v[(size_t)i] = i;
        std::shuffle(v.begin(), v.end(), gen);
        if (r >= first_round)
            for (int i = 0; i < n; i++) out[(size_t)(r - first_round) * n + i] = v[(size_t)i];
    }
    return DSAC_OK;
}

// stochasticSubSample (cnn_softam.h:283-309; targetSize 40, patchSize 42) drawing from the
// thread-0 generator of ThreadRand (mt19937 seeded `seed`, thread_rand.cpp:52) through
// fresh uniform_real_distribution<double> objects (drand, thread_rand.cpp:71-81).
int dsac_stochastic_subsample(uint32_t seed, int32_t width, int32_t height, int32_t* pix) {
    if (!pix) return DSAC_ERR_ARG;
    std::mt19937 gen;
    gen.seed(seed);
    const int target = DSAC_GRID, patch = 42;
    float xStride = (width - patch) / (float)target;
    float yStride = (height - patch) / (float)target;
    int sx = 0;
    for (float minX = patch / 2, x = xStride + patch / 2; x <= width - patch / 2 + 1; minX = x, x += xStride) {
        int sy = 0;
        for (float minY = patch / 2, y = yStride + patch / 2; y <= height - patch / 2 + 1; minY = y, y += yStride) {
            std::uniform_real_distribution<double> dx(minX, x);
            int curX = dx(gen);
            std::uniform_real_distribution<double> dy(minY, y);
            int curY = dy(gen);
            if (sx < target && sy < target) {
                pix[(sy * target + sx) * 2] = curX;
                pix[(sy * target + sx) * 2 + 1] = curY;
            }
            sy++;
        }
        sx++;
    }
    return DSAC_OK;
}

int dsac_synth_frames(uint32_t data_seed, uint32_t sampler_seed, int32_t n_streams, int64_t frame0, int32_t n_frames,
                      double rho, double sigma, int32_t traj, double focal, double cx, double cy, int16_t* coords,
                      int32_t* pix, double* gt_cv, double* gt_jp) {
    if (!coords || !pix || n_frames < 0) return DSAC_ERR_ARG;
    const int N = DSAC_N;
    for (int32_t i = 0; i < n_frames; i++) {
        int64_t g = frame0 + i;
        Rng rng((uint64_t)data_seed + (uint64_t)g);
        int32_t* px = pix + (size_t)i * N * 2;
        dsac_stochastic_subsample(sampler_seed + (uint32_t)(g * n_streams), (int)std::lround(2 * cx), (int)std::lround(2 * cy), px);
        double rvec[3], tvec[3];
        if (!traj) {
            for (int k = 0; k < 3; k++) rvec[k] = rng.uni(-0.5, 0.5);
            tvec[0] = rng.uni(-300, 300);
            tvec[1] = rng.uni(-300, 300);
            tvec[2] = rng.uni(1500, 3000);
        } else {
            // smooth hand-held trajectory through a ~3 m room centred at the origin
            double s = (double)g * 0.01;
            rvec[0] = 0.25 * std::sin(0.9 * s) + 0.05 * std::sin(3.1 * s);
            rvec[1] = 0.45 * std::sin(0.5 * s + 0.7);
            rvec[2] = 0.15 * std::cos(0.7 * s);
            double R[9];
            dsac::rodrigues_v2m(rvec, R);
            double C[3] = {900 * std::sin(0.6 * s), 250 * std::sin(1.3 * s + 0.4), -2200 + 500 * std::cos(0.45 * s)};
            for (int k = 0; k < 3; k++) tvec[k] = -(R[k * 3] * C[0] + R[k * 3 + 1] * C[1] + R[k * 3 + 2] * C[2]);
            for (int k = 0; k < 8; k++) rng.next();  // keep the per-frame stream layout
        }
        double R[9];
        dsac::rodrigues_v2m(rvec, R);
        int16_t* co = coords + (size_t)i * N * 3;
        for (int p = 0; p < N; p++) {
            double u = px[p * 2], v = px[p * 2 + 1];
            double d = rng.uni(500, 3500);
            double Xc[3] = {(u - cx) * d / focal - tvec[0], (v - cy) * d / focal - tvec[1], d - tvec[2]};
            double Y[3];
            for (int k = 0; k < 3; k++) Y[k] = R[0 * 3 + k] * Xc[0] + R[1 * 3 + k] * Xc[1] + R[2 * 3 + k] * Xc[2];  // R^T
            bool inl = rng.uni() < rho;
            double n0 = rng.gauss(), n1 = rng.gauss(), n2 = rng.gauss();
            double o0 = rng.uni(-2000, 2000), o1 = rng.uni(-2000, 2000), o2 = rng.uni(-2000, 2000);
            if (inl) {
                co[p * 3] = sat16(Y[0] + sigma * n0);
                co[p * 3 + 1] = sat16(Y[1] + sigma * n1);
                co[p * 3 + 2] = sat16(Y[2] + sigma * n2);
            } else {
                co[p * 3] = sat16(o0);
                co[p * 3 + 1] = sat16(o1);
                co[p * 3 + 2] = sat16(o2);
            }
        }
        if (gt_cv) {
            for (int k = 0; k < 3; k++) {
                gt_cv[(size_t)i * 6 + k] = rvec[k];
                gt_cv[(size_t)i * 6 + 3 + k] = tvec[k];
            }
        }
        if (gt_jp) {  // jp::cv2our, types.h:186-214
            double* o = gt_jp + (size_t)i * 12;
            for (int k = 0; k < 9; k++) o[k] = R[k];
            for (int k = 0; k < 3; k++) {
                o[3 + k] = -o[3 + k];
                o[6 + k] = -o[6 + k];
            }
            o[9] = tvec[0]; o[10] = -tvec[1]; o[11] = -tvec[2];
        }
    }
    return DSAC_OK;
}

}  // extern "C"
