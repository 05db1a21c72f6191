// guided.cuh -- guided sampling (dsac_set_sampling_logits_device): minimal sets drawn from learned per-cell weights, and the
// log-probability of the draw with its gradient (Neural-Guided RANSAC, Brachmann & Rother, ICCV 2019).
//
//   k_guided_table  once per setting: softmax of the logits in fp64, the integer weights q_j = floor(w_j * 2^31), their
//                   inclusive prefix sums and the DSAC_ST_BAD_WEIGHTS test, per frame
//   k1_gslot        (sampler_split.cuh) the rounds' generator: k1_slot's selection and round sizing, one candidate per thread
//   k1_gtail        streams the rounds left short: more guided candidates, 256 at a time, until the quota or max_candidates
//   k_guided_logp   log-probability of the used candidates of every frame and its gradient, regenerated from the counters
#pragma once
#include <cuda_runtime.h>

#include "sampler_split.cuh"

namespace dsac {

constexpr uint32_t ST_BAD_WEIGHTS = 32u;   // DSAC_ST_BAD_WEIGHTS
constexpr int KG_THREADS = 256;

// One CTA per frame.  w = softmax(logits) in fp64 (max-subtracted exp, the sum in a fixed order), q_j = floor(w_j 2^31)
// (so Q = sum q < 2^32), cum = inclusive prefix sums of q.  bad[f] = 1 for a NaN or +inf logit, or fewer than 4 cells
// with q > 0 (-inf logits are allowed: q = 0).
__global__ void __launch_bounds__(KG_THREADS) k_guided_table(const float* logits, double* w, uint32_t* q, uint32_t* cum, uint32_t* bad) {
    __shared__ double red[KG_THREADS / 32];
    __shared__ uint32_t sq[DSAC_N_CONST];
    __shared__ double s_max, s_sum;
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* l = logits + (size_t)frame * DSAC_N_CONST;
    double mx = -INFINITY;
    int nonfinite = 0;
    for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) {
        const float v = l[k];
        if (isnan(v) || v == INFINITY) nonfinite = 1;
        else mx = fmax(mx, (double)v);
    }
    nonfinite = __syncthreads_or(nonfinite);
    for (int off = 16; off; off >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        double m = red[0];
        for (int i = 1; i < KG_THREADS / 32; i++) m = fmax(m, red[i]);
        s_max = m;
    }
    __syncthreads();
    mx = s_max;
    double s = 0;
    if (!nonfinite && mx > -INFINITY)
        for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) s += exp((double)l[k] - mx);
    for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    __syncthreads();
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (tid == 0) {
        double t = 0;
        for (int i = 0; i < KG_THREADS / 32; i++) t += red[i];
        s_sum = t;
    }
    __syncthreads();
    const bool usable = !nonfinite && mx > -INFINITY;
    const double inv = 1.0 / s_sum;
    for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) {
        const double wk = usable ? exp((double)l[k] - mx) * inv : 0.0;
        w[(size_t)frame * DSAC_N_CONST + k] = wk;
        const uint32_t qk = (uint32_t)floor(wk * (double)GUIDED_ONE);
        sq[k] = qk;
        q[(size_t)frame * DSAC_N_CONST + k] = qk;
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t c = 0;
        int pos = 0;
        for (int k = 0; k < DSAC_N_CONST; k++) {
            c += sq[k];
            pos += sq[k] > 0;
            sq[k] = c;
        }
        bad[frame] = (!usable || pos < 4) ? 1u : 0u;
    }
    __syncthreads();
    for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) cum[(size_t)frame * DSAC_N_CONST + k] = sq[k];
}

// Streams the rounds left short continue here, one CTA per (stream, frame): 256 guided candidates per step, filtered,
// solved and accepted exactly as in the rounds, the first accepted ones in candidate order, until the stream has its
// quota or max_candidates candidates.  An exhausted stream gets the uniform path's empty hypotheses.  Normally no stream
// is left: the kernel then returns after one look at the state.
// RGBD: the candidates are accepted by rgbd_accept instead.
// GATE: behind the pose priors' covariance gate (prior_gate_ok), as the rounds' acceptance.
template <bool PER_FRAME, bool RGBD = false, bool GATE = false>
__global__ void __launch_bounds__(KG_THREADS) k1_gtail_t(K1SplitParams q, GuidedGen gg) {
    __shared__ uint32_t cum[DSAC_N_CONST];
    __shared__ int warp[2][KG_THREADS / 32];
    const SampleParams& p = q.sp;
    const int tid = threadIdx.x, s = blockIdx.x, frame = blockIdx.y, slot = frame * p.T + s;
    int h0, quota;
    stream_chunk(p.H, p.T, s, &h0, &quota);
    if (quota == 0) return;
    K1SlotState& S = q.state[slot];
    if (S.done) return;
    for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) cum[k] = gg.cum[(size_t)frame * DSAC_N_CONST + k];
    __syncthreads();
    int acc = S.acc;
    long long cand_base = S.cand_base;
    const long long cand_max = p.max_candidates > 0 ? (long long)p.max_candidates : (1ll << 40);
    const Cam cam = frame_cam<PER_FRAME>(p, frame);
    const double inv_f = 1. / cam.f, cx_f = cam.cx * inv_f, cy_f = cam.cy * inv_f;
    const CellRec* cell = q.celltab + (size_t)frame * DSAC_N_CONST;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    const unsigned long long z = (unsigned long long)((p.frame0 + frame) * (long long)p.T + s);
    const uint32_t pos0 = (s == 0) ? p.skip : 0u;
    int par = 0;
    while (acc < quota && cand_base < cand_max) {
        const long long ci = cand_base + tid;
        bool ok = false;
        double rvec[3], tvec[3];
        int cells[4];
        if (ci < cand_max) {
            guided_draw(cum, p.seed, z, (uint32_t)ci, cells);
            if constexpr (RGBD) {
                bool fragile = false;
                ok = rgbd_accept_cells(p.coords + (size_t)frame * DSAC_N_CONST * 3, p.eye + (size_t)frame * DSAC_N_CONST * 3, pix, cells,
                                       cam.f, cam.cx, cam.cy, p.thr, rvec, tvec, &fragile);
                if (fragile) atomicAdd(p.n_fragile, 1ull);
            } else if (k1_filter_candidate(cell, cells, cam.f, cam.cx, cam.cy, inv_f, cx_f, cy_f, (double)p.thr)) {
                P3PProblem pr;
                float obj[12], img[8];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const CellRec r = cell[cells[j]];
                    pr.mu[j] = r.xn * cam.f + cam.cx;
                    pr.mv[j] = r.yn * cam.f + cam.cy;
                    pr.X[j][0] = (double)r.X; pr.X[j][1] = (double)r.Y; pr.X[j][2] = (double)r.Z;
                    obj[j * 3] = (float)pr.X[j][0]; obj[j * 3 + 1] = (float)pr.X[j][1]; obj[j * 3 + 2] = (float)pr.X[j][2];
                    img[j * 2] = (float)__ldg(pix + cells[j] * 2);
                    img[j * 2 + 1] = (float)__ldg(pix + cells[j] * 2 + 1);
                }
                P3PFront fr;
                p3p_front(pr, cam.f, cam.cx, cam.cy, fr);
                double R[9], t[3], e2 = 1.7976931348623157e308;
                const int nsol = p3p_full(pr, fr, cam.f, cam.cx, cam.cy, R, t, &e2, 0, 4);
                bool fragile = false;
                if (nsol > 0) ok = minimal_set_accept(obj, img, cam.f, cam.cx, cam.cy, p.thr, R, t, e2, rvec, tvec, &fragile);
                if (fragile) atomicAdd(p.n_fragile, 1ull);
            }
        }
        if constexpr (GATE) ok = ok && prior_gate_ok<GATE>(p, frame, rvec, tvec);
        int tot;
        const int rank = acc + block_excl_scan<KG_THREADS / 32>(ok ? 1 : 0, &tot, warp[par]);
        par ^= 1;
        if (ok && rank < quota) {
            k1_write_hyp(p, (size_t)frame * p.Hs + h0 + rank, rvec, tvec, cells, ci);
            if (rank == quota - 1) {
                p.stream_ncand[slot] = ci + 1;
                p.stream_endpos[slot] = pos0;
            }
        }
        acc += tot;
        cand_base = min(cand_base + KG_THREADS, cand_max);
    }
    if (acc < quota) {
        k1_empty_hyps(p, frame, h0 + acc, quota - acc, tid, KG_THREADS);
        if (tid == 0) {
            p.stream_ncand[slot] = cand_base;
            p.stream_endpos[slot] = pos0;
            atomicOr(p.status + frame, 1u /* DSAC_ST_SAMPLER_EXHAUSTED */);
        }
    }
}

struct GuidedLogpParams {
    const double* w;                 // [n][N] softmax of the logits
    const uint32_t* cum;             // [n][N] prefix sums of the integer weights
    const uint32_t* bad;             // [n]
    const long long* stream_ncand;   // [n][T] used candidates of every stream
    int T;
    uint32_t seed;
    long long frame0;
    double* logp;                    // [n] or null
    const double* grad_logp;         // [n] or null: no gradient
    float* grad_logits;              // [n][N]
};

// One CTA per frame.  The used candidates of stream s are 0 .. stream_ncand[s] - 1; each is regenerated from its counter.
//   log p = sum over candidates and points k of  log w_{c_k} - log(1 - S_k),   S_k = sum_{i<k} w_{c_i},  R_k = 1 - S_k
//   d log p / d logit_j = cnt_j - w_j (4 M + A) + w_j B_j,   A = sum S_k / R_k,   B_j = sum over (cand, k) with j in c_<k of 1 / R_k
// Deterministic without floating-point atomics: a thread's candidates and the reductions have a fixed order; the per-cell
// sums B_j live in shared memory and a batch of 256 candidates adds to them point by point (the B term of point i is
// sum_{k>i} 1 / R_k), warp after warp, the lanes of a warp that hold the same cell summed in lane order first.  cnt_j is
// an integer.  The work per candidate is constant: 3 x 8 block barriers per batch of 256.
__global__ void __launch_bounds__(KG_THREADS) k_guided_logp(GuidedLogpParams g) {
    __shared__ double w[DSAC_N_CONST];
    __shared__ uint32_t cum[DSAC_N_CONST];
    __shared__ double accB[DSAC_N_CONST];
    __shared__ int cntS[DSAC_N_CONST];
    __shared__ double red[2][KG_THREADS / 32];
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t fo = (size_t)frame * DSAC_N_CONST;
    if (g.bad[frame]) {
        if (g.logp && tid == 0) g.logp[frame] = 0.0;
        if (g.grad_logp)
            for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) g.grad_logits[fo + k] = 0.f;
        return;
    }
    for (int k = tid; k < DSAC_N_CONST; k += KG_THREADS) {
        w[k] = g.w[fo + k]; cum[k] = g.cum[fo + k]; accB[k] = 0.0; cntS[k] = 0;
    }
    __syncthreads();
    const bool grad = g.grad_logp != nullptr;
    double lp = 0, A = 0;
    long long M = 0;
    for (int s = 0; s < g.T; s++) {
        const long long ms = g.stream_ncand[(size_t)frame * g.T + s];
        M += ms;
        const unsigned long long z = (unsigned long long)((g.frame0 + frame) * (long long)g.T + s);
        for (long long i0 = 0; i0 < ms; i0 += KG_THREADS) {
            const long long i = i0 + tid;
            const bool valid = i < ms;
            int c[4] = {0, 0, 0, 0};
            double suf[3] = {0, 0, 0};
            if (valid) {
                guided_draw(cum, g.seed, z, (uint32_t)i, c);
                double S = 0, rinv[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const double R = 1.0 - S;
                    lp += log(w[c[k]]) - log(R);
                    A += S / R;
                    rinv[k] = 1.0 / R;
                    S += w[c[k]];
                }
                suf[2] = rinv[3];
                suf[1] = rinv[3] + rinv[2];
                suf[0] = rinv[3] + rinv[2] + rinv[1];
            }
            if (!grad) continue;
            if (valid)
#pragma unroll
                for (int k = 0; k < 4; k++) atomicAdd(&cntS[c[k]], 1);
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const int key = valid ? c[k] : -1 - lane;   // (an idle lane is a group of its own)
                const unsigned grp = __match_any_sync(0xffffffffu, key);
                double sum = 0;
                for (unsigned m = grp; m; m &= m - 1) sum += __shfl_sync(grp, suf[k], __ffs(m) - 1);
                const bool leader = valid && lane == __ffs(grp) - 1;
                for (int ww = 0; ww < KG_THREADS / 32; ww++) {
                    if (warp == ww && leader) accB[c[k]] += sum;
                    __syncthreads();
                }
            }
        }
    }
    for (int off = 16; off; off >>= 1) {
        lp += __shfl_xor_sync(0xffffffffu, lp, off);
        A += __shfl_xor_sync(0xffffffffu, A, off);
    }
    if (lane == 0) { red[0][warp] = lp; red[1][warp] = A; }
    __syncthreads();
    lp = 0; A = 0;
    for (int i = 0; i < KG_THREADS / 32; i++) { lp += red[0][i]; A += red[1][i]; }
    if (g.logp && tid == 0) g.logp[frame] = lp;
    if (grad) {
        const double gf = g.grad_logp[frame], c4 = 4.0 * (double)M + A;
        for (int j = tid; j < DSAC_N_CONST; j += KG_THREADS)
            g.grad_logits[fo + j] = (float)(gf * ((double)cntS[j] - w[j] * c4 + w[j] * accB[j]));
    }
}

}  // namespace dsac
