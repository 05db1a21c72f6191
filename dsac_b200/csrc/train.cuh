// train.cuh -- the device side of a training round that is not a refinement, P3P or score derivative: the DSAC variant's
// draw and expected loss (k_dsac_draw), the backward's hypothesis selection (k_dsac_select) and finite-difference job list
// (k_dsac_jobs_count, k_dsac_scan, k_dsac_jobs), the softmax Jacobian of path II (k_dsac_sog) and the hand-off of
// dLoss/dObj to the coordinate CNN (k_e2e_grad).  Each reproduces a host loop of the reference's drivers in the
// reference's order, so the kernels downstream (k_refine, k_dsac_combine, k_dscore) see the same jobs in the same order.
#pragma once
#include "pose_math.cuh"
#include "prior.cuh"
#include "sampler.cuh"

namespace dsac {

constexpr double DRAW_MIN_P = 1e-8;     // draw() skips hypotheses below EPS (cnn.h:111)
constexpr double SELECT_MIN_SF = 1e-4;  // hypotheses differentiated by path I (train_ransac.cpp:320)

// libstdc++ 13 generate_canonical<double, 53>(mt19937): two words, the first one low; a sum that rounds up to 2^64
// gives the largest double below 1.
DSAC_HD double canonical53(uint32_t w0, uint32_t w1) {
    const double sum = DSAC_DADD((double)w0, DSAC_DMUL((double)w1, 4294967296.0));
    double r = sum / 18446744073709551616.0;   // a power of two: exact
    if (r >= 1.0) r = nextafter(1.0, 0.0);
    return r;
}

// draw() of cnn.h:102-126 over one frame's softmax p[0..H): probSum is the sequential sum of the p >= 1e-8 in h order.
// random_draw: u = uniform_real_distribution<double>(0, probSum) from the canonical value `canon`, pick = the first h
// whose cumulative sum exceeds u (std::map::upper_bound on the cumulative sums), the last eligible h when none does.
// Else the arg-max, first maximum kept.  No eligible h: 0.
DSAC_HD int draw_pick(const double* p, int H, int random_draw, double canon) {
    double probSum = 0, maxProb = -1;
    int maxIdx = 0;
    for (int i = 0; i < H; i++) {
        if (p[i] < DRAW_MIN_P) continue;
        probSum = DSAC_DADD(probSum, p[i]);
        if (maxProb < 0 || p[i] > maxProb) { maxProb = p[i]; maxIdx = i; }
    }
    if (!random_draw) return maxIdx;
    const double u = DSAC_DADD(DSAC_DMUL(canon, probSum - 0.0), 0.0);   // (b - a) * canonical + a
    double cum = 0;
    int pick = 0;
    for (int i = 0; i < H; i++) {
        if (p[i] < DRAW_MIN_P) continue;
        cum = DSAC_DADD(cum, p[i]);
        pick = i;
        if (cum > u) break;
    }
    return pick;
}

// Stream positions of the two words generate_canonical takes after `endpos` words: word w of an mt19937 stream is word
// w % 624 of the state after w / 624 + 1 regenerations.
DSAC_HD void draw_word_blocks(unsigned long long endpos, unsigned long long* block0, int* idx0, unsigned long long* block1, int* idx1) {
    *block0 = endpos / MT_N; *idx0 = (int)(endpos % MT_N);
    *block1 = (endpos + 1) / MT_N; *idx1 = (int)((endpos + 1) % MT_N);
}

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)

struct DrawParams {
    int H, T, random_draw;
    uint32_t seed;
    long long frame0;
    const double* sf;                     // [n][H]
    const int32_t* img_idx;               // [n][H][4]
    const unsigned long long* stream_endpos;   // [n][T]
    const double* loss;                   // [n][H] or null (no ground truth: zero)
    const double* rot_err;                // [n][H] or null
    const double* t_err;                  // [n][H] or null
    const int32_t* correct;               // [n][H] or null
    int32_t* inlier_maps;                 // [n][H][N] or null: the support cells are zeroed (cnn.h:1221-1227)
    int32_t* hyp_idx;                     // [n]
    double* expected_loss;                // [n]
    double* out_rot_err;                  // [n]
    double* out_t_err;                    // [n]
    int32_t* out_correct;                 // [n]
};

constexpr int DRAW_THREADS = 256;         // >= 227 regenerating threads
// One CTA per frame.  Stream 0 of global frame g is mt19937(seed + g T); thread 0 of the reference continues it after
// the sampler (drand, thread_rand.cpp:71-81), so the draw takes the two words at stream_endpos[g T] and after.  The state
// is regenerated block-parallel (mt_regenerate_words) into the other half of a double buffer, once per 624 words.
__global__ void __launch_bounds__(DRAW_THREADS) k_dsac_draw(DrawParams p) {
    __shared__ uint32_t s_mt[2][MT_N];
    __shared__ uint32_t s_words[2];
    const int f = blockIdx.x, tid = threadIdx.x;
    const size_t H = p.H;
    const double* sf = p.sf + f * H;
    if (p.inlier_maps)
        for (int i = tid; i < p.H * 4; i += DRAW_THREADS) {
            const int c = p.img_idx[f * H * 4 + i];
            if (c >= 0) p.inlier_maps[(f * H + i / 4) * DSAC_N_CONST + c] = 0;
        }
    if (p.random_draw) {
        if (tid == 0) mt_seed(s_mt[0], p.seed + (uint32_t)((p.frame0 + f) * (long long)p.T));
        unsigned long long b0, b1;
        int i0, i1;
        draw_word_blocks(p.stream_endpos[(size_t)f * p.T], &b0, &i0, &b1, &i1);
        int cur = 0;
        __syncthreads();
        for (unsigned long long b = 0; b <= b1; b++) {
            if (tid < MT_N - MT_M) {
                uint32_t x[3];
                const int m = mt_regenerate_words(s_mt[cur], tid, x);
                for (int w = 0; w < m; w++) s_mt[cur ^ 1][tid + w * (MT_N - MT_M)] = x[w];
            }
            __syncthreads();
            cur ^= 1;
            if (tid == 0 && b == b0) s_words[0] = mt_temper(s_mt[cur][i0]);
            if (tid == 0 && b == b1) s_words[1] = mt_temper(s_mt[cur][i1]);
        }
    }
    if (tid != 0) return;
    const int pick = draw_pick(sf, p.H, p.random_draw, p.random_draw ? canonical53(s_words[0], s_words[1]) : 0.0);
    double expected = 0;   // expectedMaxLoss, cnn.h:137-151
    for (int h = 0; h < p.H; h++) expected = DSAC_DADD(expected, DSAC_DMUL(sf[h], p.loss ? p.loss[f * H + h] : 0.0));
    p.hyp_idx[f] = pick;
    p.expected_loss[f] = expected;
    p.out_rot_err[f] = p.rot_err ? p.rot_err[f * H + pick] : 0.0;
    p.out_t_err[f] = p.t_err ? p.t_err[f * H + pick] : 0.0;
    p.out_correct[f] = p.correct ? p.correct[f * H + pick] : 0;
}

// Exclusive prefix of `v` over the CTA (blockDim.x a multiple of 32, at most 1024); *total gets the sum.  s_warp: 33 ints.
__device__ __forceinline__ int block_exclusive_sum(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    int incl = v;
    for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
    }
    __syncthreads();   // s_warp may still be read by a previous call
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int w = 0; w < warps; w++) { const int c = s_warp[w]; s_warp[w] = acc; acc += c; }
        s_warp[32] = acc;
    }
    __syncthreads();
    *total = s_warp[32];
    return s_warp[warp] + incl - v;
}

struct SelectParams {
    int n, H, skip;
    int prior_k;                 // pose priors of the pass: slots H - prior_k .. H - 1 of a frame without DSAC_ST_BAD_PRIOR
    const uint32_t* status;      // [n] (read with prior_k > 0)
    const double* sf;            // [n][H]
    const int32_t* img_idx;      // [n][H][4]
    const double* hyp_pose;      // [n][H][6]
    int seeded;                  // a seeded backward: select only hypotheses whose seed is not all zero (none: null seed)
    const double* seed;          // [n][H][6]
    // selection (k_dsac_select): selected hypotheses in (frame, h) order
    int32_t* sel;                // [n H] global hypothesis index
    int32_t* sel_frame;          // [n H] frame, -1 behind the last selected (unused k_refine job slots)
    double* sel_init;            // [n H][6] its pose: the initial pose of its forward refinement
    int32_t* sel_begin;          // [n + 1] first selected of frame f
    int32_t* n_selected;         // [n]
    int32_t* totals;             // [2]: selected hypotheses, refinement jobs
    // job list (k_dsac_jobs_count, k_dsac_scan, k_dsac_jobs)
    int32_t* imaps;              // [n H][N] inlier maps of the selected hypotheses' forward refinement
    const int32_t* n_perm;       // [n H] permutations that refinement consumed
    int32_t* pair_count;         // [n H]
    int32_t* pair_begin;         // [n H]
    int32_t* frame_pair_begin;   // [n + 1]
    int32_t* n_refine_jobs;      // [n]
    int32_t* job_frame;          // [jobs]
    int32_t* job_pert;           // [jobs][2]
    int32_t* job_p3p;            // [jobs][3]
    int32_t* job_max;            // [jobs]
    double* job_init;            // [jobs][6]
    int32_t* pair_hyp;           // [pairs]
    int32_t* pair_col;           // [pairs]
    int32_t* pair_scale;         // [pairs]
};

// The hypotheses with sf > 1e-4 and a minimal set (train_ransac.cpp:320) or a pose prior in their slot, and in a seeded
// backward a nonzero seed (a zero seed contributes nothing to path I), stably compacted; one CTA walks the frames.
constexpr int SELECT_THREADS = 1024;   // = DSAC_MAX_HYPS: one pass per frame
__global__ void __launch_bounds__(SELECT_THREADS) k_dsac_select(SelectParams p) {
    __shared__ int s_warp[33];
    const int tid = threadIdx.x;
    int base = 0;
    for (int f = 0; f < p.n; f++) {
        const size_t g = (size_t)f * p.H + tid;
        const bool prior = p.prior_k > 0 && tid >= p.H - p.prior_k && !(p.status[f] & PRIOR_ST_BAD);
        bool take = tid < p.H && p.sf[g] > SELECT_MIN_SF && (p.img_idx[g * 4] >= 0 || prior);
        if (take && p.seeded) {
            bool nz = false;
            if (p.seed)
                for (int k = 0; k < 6; k++) nz |= p.seed[g * 6 + k] != 0.0;
            take = nz;
        }
        int count;
        const int r = block_exclusive_sum(take ? 1 : 0, s_warp, &count);
        if (take) {
            p.sel[base + r] = (int32_t)g;
            p.sel_frame[base + r] = f;
            for (int k = 0; k < 6; k++) p.sel_init[(size_t)(base + r) * 6 + k] = p.hyp_pose[g * 6 + k];
        }
        if (tid == 0) { p.sel_begin[f] = base; p.n_selected[f] = count; }
        base += count;
    }
    for (int i = base + tid; i < p.n * p.H; i += SELECT_THREADS) p.sel_frame[i] = -1;
    if (tid == 0) { p.sel_begin[p.n] = base; p.totals[0] = base; }
}

// A cell of selected hypothesis s that path I differentiates: nonzero in its inlier map and not one of its support cells
// (which cnn.h:1221-1227 zeroes first).
__device__ __forceinline__ bool job_cell(const int32_t* im, const int32_t* cells, int c) {
    return im[c] != 0 && c != cells[0] && c != cells[1] && c != cells[2] && c != cells[3];
}

// Pairs of hypothesis s: 9 on the minimal set (none for a pose prior, which has no minimal set: img_idx -1), 3 per skip-th
// job cell.  Grid: n H CTAs, those past the selection exit.
constexpr int JOBS_THREADS = 256;
constexpr int JOBS_CELLS = (DSAC_N_CONST + JOBS_THREADS - 1) / JOBS_THREADS;   // 7 cells of the x-outer order per thread
__global__ void __launch_bounds__(JOBS_THREADS) k_dsac_jobs_count(SelectParams p) {
    __shared__ int s_warp[33];
    const int s = blockIdx.x;
    if (s >= p.totals[0]) return;
    const int32_t* im = p.imaps + (size_t)s * DSAC_N_CONST;
    const int32_t* cells = p.img_idx + (size_t)p.sel[s] * 4;
    int nz = 0;
    for (int c = threadIdx.x; c < DSAC_N_CONST; c += JOBS_THREADS) nz += job_cell(im, cells, c) ? 1 : 0;
    int total;
    block_exclusive_sum(nz, s_warp, &total);
    if (threadIdx.x == 0) p.pair_count[s] = (cells[0] >= 0 ? 9 : 0) + 3 * (total / p.skip);
}

// Exclusive scan of the pair counts; per-frame pair ranges and job counts; totals[1] = refinement jobs.  One CTA.
__global__ void __launch_bounds__(SELECT_THREADS) k_dsac_scan(SelectParams p) {
    __shared__ int s_warp[33];
    const int ns = p.totals[0];
    int base = 0;
    for (int s0 = 0; s0 < ns; s0 += SELECT_THREADS) {
        const int s = s0 + threadIdx.x;
        const int v = s < ns ? p.pair_count[s] : 0;
        int total;
        const int r = block_exclusive_sum(v, s_warp, &total);
        if (s < ns) p.pair_begin[s] = base + r;
        base += total;
    }
    __syncthreads();
    for (int f = threadIdx.x; f <= p.n; f += SELECT_THREADS) {
        const int b = p.sel_begin[f];
        p.frame_pair_begin[f] = b < ns ? p.pair_begin[b] : base;
    }
    __syncthreads();
    for (int f = threadIdx.x; f < p.n; f += SELECT_THREADS) p.n_refine_jobs[f] = 2 * (p.frame_pair_begin[f + 1] - p.frame_pair_begin[f]);
    if (threadIdx.x == 0) p.totals[1] = 2 * base;
}

// Central-difference pair q: jobs 2q (+eps) and 2q+1 (-eps) of k_refine, localEstObj(y, x)[ch] +/- 2 (cnn.h:866-990).
__device__ __forceinline__ void write_pair(const SelectParams& p, int q, int g, int f, int cell, int ch, bool minimal, int pt, int n_perm) {
    for (int k = 0; k < 2; k++) {
        const int j = 2 * q + k, delta = k ? -2 : 2;
        p.job_frame[j] = f;
        p.job_pert[j * 2] = cell * 3 + ch; p.job_pert[j * 2 + 1] = delta;
        p.job_p3p[j * 3] = minimal ? g : -1; p.job_p3p[j * 3 + 1] = pt * 3 + ch; p.job_p3p[j * 3 + 2] = delta;
        p.job_max[j] = n_perm;
        for (int i = 0; i < 6; i++) p.job_init[(size_t)j * 6 + i] = p.hyp_pose[(size_t)g * 6 + i];   // k_dsac_job_p3p replaces it for the minimal set
    }
    p.pair_hyp[q] = g; p.pair_col[q] = cell * 3 + ch; p.pair_scale[q] = minimal ? 1 : p.skip;
}

// One CTA per selected hypothesis: its 9 minimal-set pairs (3 points x 3 channels; the 4th point's gradient is zero),
// then every skip-th job cell in x-outer, y-inner order (cnn.h:939-960), 3 channels each.
__global__ void __launch_bounds__(JOBS_THREADS) k_dsac_jobs(SelectParams p) {
    __shared__ int s_warp[33];
    const int s = blockIdx.x, tid = threadIdx.x;
    const int g = p.sel[s], f = p.sel_frame[s], q0 = p.pair_begin[s], nper = p.n_perm[s];
    const int32_t* im = p.imaps + (size_t)s * DSAC_N_CONST;
    const int32_t* cells = p.img_idx + (size_t)g * 4;
    const int n_min = cells[0] >= 0 ? 9 : 0;   // a pose prior: no minimal-set pairs
    if (tid < n_min) write_pair(p, q0 + tid, g, f, cells[tid / 3], tid % 3, true, tid / 3, nper);
    const int o0 = tid * JOBS_CELLS;
    int nz = 0;
    for (int o = o0; o < min(o0 + JOBS_CELLS, DSAC_N_CONST); o++) nz += job_cell(im, cells, (o % DSAC_GRID_CONST) * DSAC_GRID_CONST + o / DSAC_GRID_CONST) ? 1 : 0;
    int total;
    int k = block_exclusive_sum(nz, s_warp, &total);
    for (int o = o0; o < min(o0 + JOBS_CELLS, DSAC_N_CONST); o++) {
        const int cell = (o % DSAC_GRID_CONST) * DSAC_GRID_CONST + o / DSAC_GRID_CONST;   // o = x * 40 + y
        if (!job_cell(im, cells, cell)) continue;
        if (++k % p.skip != 0) continue;
        const int q = q0 + n_min + (k / p.skip - 1) * 3;
        for (int ch = 0; ch < 3; ch++) write_pair(p, q + ch, g, f, cell, ch, false, 0, nper);
    }
}

// scoreOutputGradients of the DSAC variant (cnn.h:733-741): g_i = p_i l_i - sum_j p_i p_j l_j, j in order, no contraction.
__global__ void k_dsac_sog(const double* __restrict__ sf, const double* __restrict__ loss, int n, int H, double* __restrict__ sog) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * H) return;
    const double* pf = sf + (size_t)(i / H) * H;
    const double* lf = loss + (size_t)(i / H) * H;
    const double pi = sf[i];
    double g = DSAC_DMUL(pi, loss[i]);
    for (int j = 0; j < H; j++) g = DSAC_DADD(g, -DSAC_DMUL(DSAC_DMUL(pi, pf[j]), lf[j]));
    sog[i] = g;
}

// dLoss/dObj = a (+ b) into dloss_dobj, and the coordinate CNN's gradient as lua/train_obj_softam.lua:101-105 hands it
// to model:backward: float(g_f * clamp(dLoss/dObj, +-clamp)), g_f = loss_grad[f] (null: 1), clamp <= 0: none.  The
// gradient stays per millimetre of the int16 grid and passes straight through the rounding and saturation of
// k_coords_from_prediction (DESIGN.md quirk Q12).
__global__ void k_e2e_grad(const double* __restrict__ a, const double* __restrict__ b, const double* __restrict__ loss_grad,
                           float clamp, size_t count, double* __restrict__ dloss_dobj, float* __restrict__ dloss_dpred) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const double v = b ? a[i] + b[i] : a[i];
    if (dloss_dobj) dloss_dobj[i] = v;
    if (dloss_dpred) {
        const double c = clamp > 0 ? fmax(-(double)clamp, fmin((double)clamp, v)) : v;
        const double g = loss_grad ? loss_grad[i / ((size_t)DSAC_N_CONST * 3)] : 1.0;
        dloss_dpred[i] = (float)(g * c);
    }
}

#endif

}  // namespace dsac
