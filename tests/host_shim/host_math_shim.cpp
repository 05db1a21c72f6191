// Host build of the PRODUCT's device arithmetic headers (dsac_b200/csrc/*.cuh compiled with
// DSAC_HOST_ONLY) so that `-m "not gpu"` tests can compare them with the oracle on a box
// without a GPU.  Test infrastructure only; never shipped or used by the product path.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/pose_math.cuh"

extern "C" {
int shim_minimal_set(const float* obj, const float* img, double f, double cx, double cy, int thr, double* rvec,
                     double* tvec, int* fragile) {
    bool fr = false;
    bool ok = dsac::minimal_set_hypothesis(obj, img, f, cx, cy, thr, rvec, tvec, &fr);
    *fragile = fr ? 1 : 0;
    return ok ? 1 : 0;
}
int shim_p3p_best(const float* obj, const float* img, double f, double cx, double cy, double* R, double* t, double* e2) {
    dsac::P3PProblem pr;
    for (int i = 0; i < 4; i++) {
        pr.mu[i] = dsac::p3p_pixel(img[i * 2], cx, f);
        pr.mv[i] = dsac::p3p_pixel(img[i * 2 + 1], cy, f);
        for (int k = 0; k < 3; k++) pr.X[i][k] = obj[i * 3 + k];
    }
    return dsac::p3p_best(pr, f, cx, cy, R, t, e2);
}
void shim_rodrigues_v2m(const double* r, double* R) { dsac::rodrigues_v2m(r, R); }
void shim_rodrigues_m2v(const double* R, double* r) { dsac::rodrigues_m2v(R, r); }
}

#include <vector>
#include "../../dsac_b200/csrc/sampler.cuh"
extern "C" {
// product MT19937 + Lemire + candidate parser, run sequentially on the host
void shim_mt_raw(uint32_t seed, int n, uint32_t* out) {
    uint32_t mt[dsac::MT_N];
    dsac::mt_seed(mt, seed);
    int i = 0;
    while (i < n) {
        dsac::mt_twist_all_seq(mt);
        for (int k = 0; k < dsac::MT_N && i < n; k++) out[i++] = dsac::mt_temper(mt[k]);
    }
}
void shim_candidates(uint32_t seed, uint32_t skip, int n, int32_t* cells, uint32_t* used) {
    size_t words = (size_t)skip + (size_t)n * 16 + 4096;
    size_t cap = 1;
    while (cap < words) cap <<= 1;
    std::vector<uint32_t> buf(cap);
    shim_mt_raw(seed, (int)words, buf.data());
    dsac::WordRing ring{buf.data(), (uint32_t)(cap - 1)};
    uint32_t pos = skip;
    for (int k = 0; k < n; k++) {
        int c[4];
        uint32_t u = dsac::parse_candidate(ring, pos, (uint32_t)words, c);
        for (int j = 0; j < 4; j++) cells[k * 4 + j] = c[j];
        used[k] = u;
        pos += u;
    }
}
void shim_stream_chunk(int H, int T, int s, int* h0, int* cnt) { dsac::stream_chunk(H, T, s, h0, cnt); }
}
extern "C" int shim_needs_full(const float* obj, const float* img, double f, double cx, double cy, int thr) {
    return dsac::minimal_set_needs_full(obj, img, f, cx, cy, thr) ? 1 : 0;
}
// n minimal sets (obj [n][12], img [n][8]): the exact solve's verdict and the conservative filter's, one byte each
extern "C" void shim_filter_batch(int n, const float* obj, const float* img, double f, double cx, double cy, int thr,
                                  uint8_t* accepted, uint8_t* needs_full) {
    for (int k = 0; k < n; k++) {
        double rv[3], tv[3];
        bool fr;
        accepted[k] = dsac::minimal_set_hypothesis(obj + 12 * k, img + 8 * k, f, cx, cy, thr, rv, tv, &fr) ? 1 : 0;
        needs_full[k] = dsac::minimal_set_needs_full(obj + 12 * k, img + 8 * k, f, cx, cy, thr) ? 1 : 0;
    }
}

#include <random>
static long long* g_reasons = nullptr; static int g_miss[64]; static int g_nmiss = 0;
extern "C" void shim_set_reasons(long long* r) { g_reasons = r; }
extern "C" int shim_get_misses(int* out) { for (int i = 0; i < g_nmiss * 4; i++) out[i] = g_miss[i]; int n = g_nmiss; g_nmiss = 0; return n; }
// Filter statistics over the first n candidates of one frame's stream: how many candidates each
// conservative filter hands to the full solve, and (the contract) how many ACCEPTED candidates a
// filter would have dropped -- must be zero.
extern "C" void shim_filter_stats(const int16_t* coords, const int32_t* pix, uint32_t seed, uint32_t skip, int n,
                                  double f, double cx, double cy, int thr, long long out[6]) {
    size_t words = (size_t)skip + (size_t)n * 10 + 4096;
    size_t cap = 1;
    while (cap < words) cap <<= 1;
    std::vector<uint32_t> buf(cap);
    shim_mt_raw(seed, (int)words, buf.data());
    dsac::WordRing ring{buf.data(), (uint32_t)(cap - 1)};
    uint32_t pos = skip;
    for (int k = 0; k < 6; k++) out[k] = 0;
    for (int k = 0; k < n; k++) {
        int c[4];
        uint32_t u = dsac::parse_candidate(ring, pos, (uint32_t)words, c);
        pos += u;
        float obj[12], img[8];
        for (int j = 0; j < 4; j++) {
            img[j * 2] = (float)pix[c[j] * 2];
            img[j * 2 + 1] = (float)pix[c[j] * 2 + 1];
            for (int q = 0; q < 3; q++) obj[j * 3 + q] = (float)coords[c[j] * 3 + q];
        }
        double rv[3], tv[3];
        bool fr;
        bool acc = dsac::minimal_set_hypothesis(obj, img, f, cx, cy, thr, rv, tv, &fr);
        bool q64 = dsac::minimal_set_needs_full(obj, img, f, cx, cy, thr);
        int reason = 0;
        bool q32 = dsac::minimal_set_needs_full_f32(obj, img, f, cx, cy, thr, &reason);
        if (q32 && g_reasons) g_reasons[reason]++;
        if (acc && !q32 && g_nmiss < 16) { for (int j = 0; j < 4; j++) g_miss[g_nmiss * 4 + j] = c[j]; g_nmiss++; }
        out[0]++;
        out[1] += acc;
        out[2] += q64;
        out[3] += q32;
        out[4] += (acc && !q64);
        out[5] += (acc && !q32);
    }
}

// guard counters of the fp64 conservative filter (only with -DDSAC_FILTER_STATS)
extern "C" double shim_filter_fp32_maxdev() {
#ifdef DSAC_FILTER_STATS
    return dsac::g_filter_fp32_maxdev;
#else
    return -1.0;
#endif
}

extern "C" void shim_filter_reasons(long long out[24]) {
#ifdef DSAC_FILTER_STATS
    for (int k = 0; k < 24; k++) out[k] = dsac::g_filter_reason[k];
#else
    for (int k = 0; k < 24; k++) out[k] = -1;
#endif
}

// Inlier test of the refinement (k_refine): the conservative fp32 decision against the reference's exact
// arithmetic on n cells of one pose.  out = {decided 0/1, undecided, wrong decisions (must be 0), exact inliers}.
extern "C" void shim_reproj_check(int n, const double* rvec, const double* tvec, const int16_t* coords, const int32_t* pix,
                                  double f, double cx, double cy, int thr, long long out[4], float* exact_err /* n or null */) {
    double R[9];
    dsac::rodrigues_v2m(rvec, R);
    float P[12];
    for (int row = 0; row < 3; row++)
        for (int col = 0; col < 4; col++) {
            double v = col < 3 ? R[row * 3 + col] : tvec[row];
            P[row * 4 + col] = (float)(row < 2 ? f * v : v);
        }
    const float cxf = (float)cx, cyf = (float)cy, c_abs = fabsf(cxf) + fabsf(cyf), thrf = (float)thr;
    for (int k = 0; k < 4; k++) out[k] = 0;
    for (int i = 0; i < n; i++) {
        const float X = (float)coords[i * 3], Y = (float)coords[i * 3 + 1], Z = (float)coords[i * 3 + 2];
        const float fu = (float)pix[i * 2], fv = (float)pix[i * 2 + 1];
        const float e = dsac::reproj_error_exact(R, tvec, X, Y, Z, f, cx, cy, fu, fv);
        if (exact_err) exact_err[i] = e;
        const bool inl = e < thrf;
        const int r = dsac::reproj_below_thr_fast(P, X, Y, Z, fu - cxf, fv - cyf, c_abs, thrf);
        if (r < 0) out[1]++;
        else {
            out[0]++;
            if ((r != 0) != inl) out[2]++;
        }
        out[3] += inl;
    }
}

// ---- the refinement's Levenberg-Marquardt arithmetic (lm_math.cuh), run sequentially on the host
#include "../../dsac_b200/csrc/lm_math.cuh"
extern "C" {
void shim_lm_solve6_fast(const double* S27, double lambda, double* x) { dsac::lm_solve6_fast(S27, lambda, x); }
void shim_rodrigues_jac(const double* r, double* R, double* J) { dsac::rodrigues_jac(r, R, J); }
void shim_rodrigues_jac_lanes(const double* r, double* R, double* J) {
    for (int lane = 0; lane < 32; lane++) dsac::rodrigues_jac_warp(r, lane, R, J);
}
// k_refine's LM loop with the lanes / threads of the kernel run one after the other: same helper functions, same
// state machine, same buffers.  obj [n][3], img [n][2] floats; pose (rvec, tvec) in/out; returns the iteration count.
int shim_lm_refine(int n, const float* obj, const float* img, double f, double cx, double cy, double* pose, int* n_passes) {
    double s_R[9], s_J[27], s_param[6], s_prev[6], s_sum[2][32];
    for (int k = 0; k < 6; k++) s_param[k] = pose[k];
    for (int lane = 0; lane < 32; lane++) dsac::rodrigues_jac_warp(s_param, lane, s_R, s_J);
    dsac::LMState lm;
    int passes = 0;
    for (;;) {
        double v[32];
        for (int k = 0; k < 32; k++) v[k] = 0;
        for (int i = 0; i < n; i++)
            dsac::lm_point_contrib(s_R, s_J, s_param, obj[i * 3], obj[i * 3 + 1], obj[i * 3 + 2], img[i * 2], img[i * 2 + 1], f, cx, cy, v);
        passes++;
        const int buf = dsac::lm_next_buf(lm);
        for (int k = 0; k < 32; k++) s_sum[buf][k] = v[k];
        const int action = dsac::lm_advance(lm, buf, s_sum[buf][27], s_param, s_prev);
        if (action == dsac::LM_DONE) break;
        if (action == dsac::LM_SOLVE_NEWBASE)
            for (int k = 0; k < 6; k++) s_prev[k] = s_param[k];
        double x[6], trial[6];
        dsac::lm_solve6_fast(s_sum[lm.cur], dsac::c_lm_lambda[lm.lambdaLg10 + 16], x);
        for (int k = 0; k < 6; k++) trial[k] = s_prev[k] - x[k];
        for (int k = 0; k < 6; k++) s_param[k] = trial[k];
        for (int lane = 0; lane < 32; lane++) dsac::rodrigues_jac_warp(trial, lane, s_R, s_J);
    }
    for (int k = 0; k < 6; k++) pose[k] = s_param[k];
    if (n_passes) *n_passes = passes;
    return lm.iters;
}
}

// ---- k_score's fp32 arithmetic (score_pair_error / score_sigmoid_sum5) on the host: one hypothesis against n cells.
// err_f32 / err_exact [n]: the fp32 entry (guarded as the kernel ends up computing it: unguarded unless z == 0) and
// getDiffMap's exact entry; *score = alpha * sum of the soft-inlier sigmoids in k_score's order of 5 cells per thread
// (cells 4t..4t+3 and 1280+t), *score_exact the same sum in double from the exact entries.  n must be 1600.
extern "C" void shim_score_hypothesis(const double* rvec, const double* tvec, const int16_t* coords, const int32_t* pix, double f,
                                      double cx, double cy, double thr, double alpha, double beta, float* err_f32, float* err_exact,
                                      double* score, double* score_exact) {
    const int N = 1600, T = 320;
    double R[9];
    dsac::rodrigues_v2m(rvec, R);
    float P[12];
    for (int row = 0; row < 3; row++)
        for (int col = 0; col < 4; col++) {
            double v = col < 3 ? R[row * 3 + col] : tvec[row];
            P[row * 4 + col] = (float)(row < 2 ? f * v : v);
        }
    const float kbeta = (float)(beta * 1.4426950408889634), tau_k = (float)thr * kbeta, cxf = (float)cx, cyf = (float)cy;
    double se = 0;
    float ssum = 0.f;   // (the kernel reduces per-thread sums over warps in a fixed tree; a float running sum is close enough here)
    for (int t = 0; t < T; t++) {
        float e[5];
        for (int j = 0; j < 5; j++) {
            const int c = j < 4 ? 4 * t + j : 4 * T + t;
            const float X = coords[c * 3], Y = coords[c * 3 + 1], Z = coords[c * 3 + 2];
            const float pu = (float)pix[c * 2] - cxf, pv = (float)pix[c * 2 + 1] - cyf;
            float az;
            e[j] = dsac::score_pair_error<false>(P[0], P[1], P[2], P[3], P[4], P[5], P[6], P[7], P[8], P[9], P[10], P[11], X, Y, Z, pu, pv, &az);
            if (az == 0.f)
                e[j] = dsac::score_pair_error<true>(P[0], P[1], P[2], P[3], P[4], P[5], P[6], P[7], P[8], P[9], P[10], P[11], X, Y, Z, pu, pv, &az);
            err_f32[c] = e[j];
            err_exact[c] = dsac::reproj_error_exact(R, tvec, X, Y, Z, f, cx, cy, (float)pix[c * 2], (float)pix[c * 2 + 1]);
            se += 1.0 / (1.0 + exp(-beta * (thr - (double)err_exact[c])));
        }
        ssum += dsac::score_sigmoid_sum5(e, kbeta, tau_k);
    }
    (void)N;
    *score = alpha * (double)ssum;
    *score_exact = alpha * se;
}

// k_sample's block-parallel MT19937 regeneration (mt_regenerate_words), the 227 threads run one after the other on a
// double-buffered state exactly as the kernel holds it: n_blocks x 624 tempered outputs.
extern "C" void shim_mt_regenerated(uint32_t seed, int n_blocks, uint32_t* out) {
    uint32_t st[2 * dsac::MT_N];
    dsac::mt_seed(st, seed);
    for (int r = 0; r < n_blocks; r++) {
        const uint32_t* so = st + (r & 1) * dsac::MT_N;
        uint32_t* sn = st + ((r & 1) ^ 1) * dsac::MT_N;
        for (int t = dsac::MT_N - dsac::MT_M - 1; t >= 0; t--) {   // any thread order: threads only read the old state
            uint32_t x[3];
            const int nw = dsac::mt_regenerate_words(so, t, x);
            for (int w = 0; w < nw; w++) sn[t + w * (dsac::MT_N - dsac::MT_M)] = x[w];
        }
        for (int k = 0; k < dsac::MT_N; k++) out[r * dsac::MT_N + k] = dsac::mt_temper(sn[k]);
    }
}

// the register-carried, branch-free form of the same regeneration (mt_twist3: k1_slot / k1_spec)
extern "C" void shim_mt_twist3(uint32_t seed, int n_blocks, uint32_t* out) {
    uint32_t st[2 * dsac::MT_N];
    dsac::mt_seed(st, seed);
    const int W = dsac::MT_N - dsac::MT_M;
    uint32_t own[W][3];
    for (int t = 0; t < W; t++)
        for (int w = 0; w < 3; w++) own[t][w] = (t + w * W < dsac::MT_N) ? st[t + w * W] : 0u;
    for (int r = 0; r < n_blocks; r++) {
        const uint32_t* so = st + (r & 1) * dsac::MT_N;
        uint32_t* sn = st + ((r & 1) ^ 1) * dsac::MT_N;
        for (int t = W - 1; t >= 0; t--) {
            uint32_t x[3];
            dsac::mt_twist3(so, t, own[t], x);
            for (int w = 0; w < 3; w++)
                if (t + w * W < dsac::MT_N) { sn[t + w * W] = x[w]; own[t][w] = x[w]; }
        }
        for (int k = 0; k < dsac::MT_N; k++) out[r * dsac::MT_N + k] = dsac::mt_temper(sn[k]);
    }
}

// k_sample's pair-based candidate parser (windows without rejected draws) against the reference loop on the same pairs
// `count` consecutive candidates parsed from pair `sp` on (cand_pairs_len, the generator's own routine): end pair of each;
// returns the number parsed before the window ran out
extern "C" int shim_parse_run(const unsigned short* pr16, int sp, int limit, int count, int* end_pair) {
    int n = 0;
    while (n < count) {
        const int len = dsac::cand_pairs_len(pr16, sp, limit);
        if (len < 0) break;
        sp += len;
        end_pair[n++] = sp;
    }
    return n;
}
extern "C" int shim_cand_pairs_len(const unsigned short* pr16, int sp, int limit) { return dsac::cand_pairs_len(pr16, sp, limit); }
