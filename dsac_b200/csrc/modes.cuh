// modes.cuh -- pose modes (dsac_pose_modes_device): the distinct refined poses of each frame's hypothesis pool.
//
//   mode_angle       the rotation angle between two rotations, so3_angle of Ra Rb^T (prior.cuh)
//   mode_dist        the distance between two translations
//   mode_near        the nearness test: angle <= rot and distance <= trans
//   k_mode_select    one CTA per frame: rank the occupied slots by score, walk them greedily into at most M seeds with
//                    their mass and member count, and write the seeds' refinement jobs; k_mode_select<true> does the
//                    same for each rig's pool of C H lifted poses (dsac_rig_pose_modes_device)
//   k_mode_merge     one warp per frame, after the refinement and the uncertainty of the seeds: merge seeds whose refined
//                    poses are near an earlier survivor, compact, and gather the outputs
//
// The math compiles for the host as well (DSAC_HOST_ONLY): tests/host_shim/modes_shim.cpp checks it against scipy.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pose_math.cuh"
#include "prior.cuh"
#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
#include "refine.cuh"   // RIG_ST_SPOILED
#endif

namespace dsac {

constexpr int MODE_MAX = 16;   // DSAC_MAX_MODES

// th of M = Ra Rb^T (row-major rotations), with v and c as so3_log forms them, fp64.
DSAC_HD double mode_angle(const double Ra[9], const double Rb[9]) {
    double M[9], v[3], s, c;
    rot_mul_bt(Ra, Rb, M);
    return so3_angle(M, v, &s, &c);
}

// |ta - tb|, the squares summed in the order x, y, z, fp64.
DSAC_HD double mode_dist(const double ta[3], const double tb[3]) {
    const double dx = ta[0] - tb[0], dy = ta[1] - tb[1], dz = ta[2] - tb[2];
    return sqrt(dx * dx + dy * dy + dz * dz);
}

// Two poses are near iff mode_angle <= rot and mode_dist <= trans (NaN: not near).  The later pose of a walk is a, the
// earlier one (a seed) b.
DSAC_HD bool mode_near(const double Ra[9], const double ta[3], const double Rb[9], const double tb[3], double rot, double trans) {
    return mode_dist(ta, tb) <= trans && mode_angle(Ra, Rb) <= rot;
}

// The ranking key of a slot: 0 empty, 1 a NaN score, else the score's bits mapped to an unsigned order (+0 for -0, so
// that the two tie).  A larger key ranks first; equal keys rank by slot.
DSAC_HD uint64_t mode_rank_key(bool occupied, double score) {
    if (!occupied) return 0;
    if (score != score) return 1;
    if (score == 0) score = 0.0;
#ifdef __CUDA_ARCH__
    const uint64_t u = (uint64_t)__double_as_longlong(score);
#else
    uint64_t u;
    memcpy(&u, &score, sizeof(u));
#endif
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)

struct ModeSelectParams {
    const double* hyp_pose;    // [n][H][6]  (RIG: the pools [R][C H][6])
    const int32_t* img_idx;    // [n][H][4]  (RIG: of the n = R C camera frames)
    const double* scores;      // [n][H]     (RIG: [R][C H])
    const double* sf;          // [n][H]     (RIG: [R][C H])
    const uint32_t* status;    // [n]        (RIG: the rig status [R])
    int H, M, prior_k;         // slots per frame, modes per frame, priors of the pass (0: none)
    int C;                     // RIG: cameras per rig
    double rot, trans;         // nearness radii (rad, mm)
    // per job j = f * M + m, seed m of frame f
    int32_t* job_frame;        // f, or -1 for no seed
    double* job_init;          // [jobs][6] the seed's hypothesis pose
    double* ref_pose;          // [jobs][6] zeroed for unused jobs (k_refine skips them)
    int32_t* rec_count;        // [jobs] zeroed for unused jobs
    int32_t* steps_done;       // [jobs] zeroed for unused jobs
    int32_t* hyp;              // [jobs] the seed's slot, -1
    double* score;             // [jobs]
    double* mass;              // [jobs] sum of the members' sf, in rank order
    int32_t* members;          // [jobs]
    int32_t* n_seeds;          // [n]
};
constexpr int MODE_SELECT_THREADS = 256;

// Bitonic sort of the (key, slot) pairs of a frame in shared memory (larger key first, then lower slot), then warp 0 walks
// the ranking 32 slots at a time: each lane tests its slot against the existing seeds in seed order; the lowest-ranked
// slot near none becomes the next seed (while fewer than M exist), and the slots after it are tested against that seed,
// until no candidate is left.  Every slot's rotation is formed once, when its chunk is walked.
// RIG (dsac_rig_pose_modes_device): CTA f is rig f and its slots are the S = C H slots of its pool, slot j = c H + h being
// camera c's hypothesis h lifted to the rig frame (k_rig_lift).  Slot j is occupied when frame f C + c sampled h, or when
// the pass had rig priors and h >= H - prior_k; a rig with DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR has none.  The walk, the
// nearness and the mass are those of a frame, over the rig poses and the pool's sf.
template <bool RIG = false>
__global__ void __launch_bounds__(MODE_SELECT_THREADS, 1) k_mode_select(ModeSelectParams p) {
    __shared__ uint64_t s_key[1024];
    __shared__ uint16_t s_slot[1024];
    __shared__ double s_R[MODE_MAX][9], s_t[MODE_MAX][3];
    __shared__ int s_seed_slot[MODE_MAX];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int H = RIG ? p.C * p.H : p.H;   // slots per pool
    int P = 1;
    while (P < H) P <<= 1;
    const bool prior_ok = RIG ? !(p.status[f] & RIG_ST_SPOILED) : p.prior_k > 0 && !(p.status[f] & PRIOR_ST_BAD);
    for (int i = tid; i < P; i += MODE_SELECT_THREADS) {
        uint64_t k = 0;
        if (i < H) {
            const size_t hi = (size_t)f * H + i;
            bool occupied;
            if constexpr (RIG) {   // prior_ok: the rig is not spoiled
                const int c = i / p.H, h = i - c * p.H;
                occupied = prior_ok && (p.img_idx[(((size_t)f * p.C + c) * p.H + h) * 4] >= 0 || (p.prior_k > 0 && h >= p.H - p.prior_k));
            } else {
                occupied = p.img_idx[hi * 4] >= 0 || (prior_ok && i >= H - p.prior_k);
            }
            k = mode_rank_key(occupied, p.scores[hi]);
        }
        s_key[i] = k;
        s_slot[i] = (uint16_t)i;
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += MODE_SELECT_THREADS) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t ka = s_key[i], kb = s_key[ixj];
                    const uint16_t sa = s_slot[i], sb = s_slot[ixj];
                    const bool b_first = kb > ka || (kb == ka && sb < sa);
                    if (((i & k) == 0) == b_first) {
                        s_key[i] = kb; s_key[ixj] = ka;
                        s_slot[i] = sb; s_slot[ixj] = sa;
                    }
                }
            }
            __syncthreads();
        }
    }
    if (tid >= 32) return;
    const int lane = tid;
    int n_ranked = 0;   // occupied slots lead the ranking
    for (int i = lane; i < P; i += 32) n_ranked += s_key[i] != 0;
    for (int o = 16; o; o >>= 1) n_ranked += __shfl_xor_sync(0xffffffffu, n_ranked, o);

    int nseed = 0;
    double mass = 0;   // of seed `lane`, in rank order
    int members = 0;
    for (int base = 0; base < n_ranked; base += 32) {
        const int r = base + lane;
        const bool act = r < n_ranked;
        const int h = act ? s_slot[r] : 0;
        const size_t hi = (size_t)f * H + h;
        double R[9], t[3];
        if (act) {
            const double* po = p.hyp_pose + hi * 6;
            rodrigues_v2m(po, R);
            t[0] = po[3]; t[1] = po[4]; t[2] = po[5];
        }
        int own = -1;
        for (int s = 0; s < nseed; s++) {
            if (!__any_sync(0xffffffffu, act && own < 0)) break;
            if (act && own < 0 && mode_near(R, t, s_R[s], s_t[s], p.rot, p.trans)) own = s;
        }
        unsigned cand = __ballot_sync(0xffffffffu, act && own < 0);
        while (cand && nseed < p.M) {
            const int l = __ffs(cand) - 1, s = nseed;
            if (lane == l) {
                own = s;
                for (int k = 0; k < 9; k++) s_R[s][k] = R[k];
                for (int k = 0; k < 3; k++) s_t[s][k] = t[k];
                s_seed_slot[s] = h;
            }
            __syncwarp();
            nseed++;
            if (act && own < 0 && mode_near(R, t, s_R[s], s_t[s], p.rot, p.trans)) own = s;
            cand = __ballot_sync(0xffffffffu, act && own < 0);
        }
        // each seed's lane adds its members' sf in rank order
        const double w = act ? p.sf[hi] : 0.0;
        const int m = min(32, n_ranked - base);
        for (int i = 0; i < m; i++) {
            const int o = __shfl_sync(0xffffffffu, own, i);
            const double wi = __shfl_sync(0xffffffffu, w, i);
            if (o == lane) {
                mass += wi;
                members++;
            }
        }
    }
    __syncwarp();
    if (lane < p.M) {
        const size_t j = (size_t)f * p.M + lane;
        const bool seed = lane < nseed;
        const int h = seed ? s_seed_slot[lane] : -1;
        const size_t hi = (size_t)f * H + (seed ? h : 0);
        p.job_frame[j] = seed ? f : -1;
        for (int k = 0; k < 6; k++) p.job_init[j * 6 + k] = seed ? p.hyp_pose[hi * 6 + k] : 0.0;
        if (!seed) {
            for (int k = 0; k < 6; k++) p.ref_pose[j * 6 + k] = 0.0;
            p.rec_count[j] = 0;
            p.steps_done[j] = 0;
        }
        p.hyp[j] = h;
        p.score[j] = seed ? p.scores[hi] : 0.0;
        p.mass[j] = seed ? mass : 0.0;
        p.members[j] = seed ? members : 0;
    }
    if (lane == 0) p.n_seeds[f] = nseed;
}

struct ModeMergeParams {
    int n, M;
    double rot, trans;
    // k_mode_select's seeds, the refinement and k_pose_uncertainty, per job f * M + m
    const int32_t* n_seeds;
    const int32_t* hyp;
    const double* score;
    const double* mass;
    const int32_t* members;
    const double* pose;        // [jobs][6] refined
    const int32_t* steps_done;
    const double* cov_xi;      // [jobs][36]
    const double* sigma2;
    const int32_t* n_fit;
    const int32_t* support;
    const int32_t* ok;
    // outputs (dsac_pose_modes_out), each nullable
    int32_t* o_n_modes;
    int32_t* o_hyp;
    double* o_pose;
    double* o_score;
    double* o_mass;
    int32_t* o_members;
    int32_t* o_steps_done;
    double* o_cov_xi;
    double* o_sigma2;
    int32_t* o_n_fit;
    int32_t* o_support;
    int32_t* o_ok;
};
constexpr int MODE_MERGE_WARPS = 4;

// One warp per frame, lane m for seed m.  Seeds are visited in seed order: a seed whose refined pose is near the refined pose
// of an earlier survivor adds its mass and members to the first such one and is dropped.  The survivors are written to
// 0 .. n_modes - 1 in seed order; the entries after them get hyp -1 and zeros.
__global__ void __launch_bounds__(MODE_MERGE_WARPS * 32) k_mode_merge(ModeMergeParams p) {
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * MODE_MERGE_WARPS + (threadIdx.x >> 5);
    if (f >= p.n) return;
    const int ns = p.n_seeds[f];
    const bool valid = lane < ns;
    const size_t j = (size_t)f * p.M + (valid ? lane : 0);
    double R[9], t[3];
    {
        double po[6] = {0, 0, 0, 0, 0, 0};
        if (valid)
            for (int k = 0; k < 6; k++) po[k] = p.pose[j * 6 + k];
        rodrigues_v2m(po, R);
        t[0] = po[3]; t[1] = po[4]; t[2] = po[5];
    }
    double mass = valid ? p.mass[j] : 0.0;
    int members = valid ? p.members[j] : 0;
    bool alive = valid;
    for (int s = 1; s < ns; s++) {
        double Rs[9], ts[3];
        for (int k = 0; k < 9; k++) Rs[k] = __shfl_sync(0xffffffffu, R[k], s);
        for (int k = 0; k < 3; k++) ts[k] = __shfl_sync(0xffffffffu, t[k], s);
        const bool near = alive && lane < s && mode_near(Rs, ts, R, t, p.rot, p.trans);
        const unsigned nb = __ballot_sync(0xffffffffu, near);
        const double ms = __shfl_sync(0xffffffffu, mass, s);
        const int mb = __shfl_sync(0xffffffffu, members, s);
        if (nb) {
            if (lane == __ffs(nb) - 1) {
                mass += ms;
                members += mb;
            }
            if (lane == s) alive = false;
        }
    }
    const unsigned live = __ballot_sync(0xffffffffu, alive);
    const int n_modes = __popc(live);
    if (lane == 0 && p.o_n_modes) p.o_n_modes[f] = n_modes;
    if (alive) {
        const size_t o = (size_t)f * p.M + __popc(live & ((1u << lane) - 1u));
        if (p.o_hyp) p.o_hyp[o] = p.hyp[j];
        if (p.o_pose)
            for (int k = 0; k < 6; k++) p.o_pose[o * 6 + k] = p.pose[j * 6 + k];
        if (p.o_score) p.o_score[o] = p.score[j];
        if (p.o_mass) p.o_mass[o] = mass;
        if (p.o_members) p.o_members[o] = members;
        if (p.o_steps_done) p.o_steps_done[o] = p.steps_done[j];
        if (p.o_cov_xi)
            for (int k = 0; k < 36; k++) p.o_cov_xi[o * 36 + k] = p.cov_xi[j * 36 + k];
        if (p.o_sigma2) p.o_sigma2[o] = p.sigma2[j];
        if (p.o_n_fit) p.o_n_fit[o] = p.n_fit[j];
        if (p.o_support) p.o_support[o] = p.support[j];
        if (p.o_ok) p.o_ok[o] = p.ok[j];
    }
    if (lane >= n_modes && lane < p.M) {
        const size_t o = (size_t)f * p.M + lane;
        if (p.o_hyp) p.o_hyp[o] = -1;
        if (p.o_pose)
            for (int k = 0; k < 6; k++) p.o_pose[o * 6 + k] = 0.0;
        if (p.o_score) p.o_score[o] = 0.0;
        if (p.o_mass) p.o_mass[o] = 0.0;
        if (p.o_members) p.o_members[o] = 0;
        if (p.o_steps_done) p.o_steps_done[o] = 0;
        if (p.o_cov_xi)
            for (int k = 0; k < 36; k++) p.o_cov_xi[o * 36 + k] = 0.0;
        if (p.o_sigma2) p.o_sigma2[o] = 0.0;
        if (p.o_n_fit) p.o_n_fit[o] = 0;
        if (p.o_support) p.o_support[o] = 0;
        if (p.o_ok) p.o_ok[o] = 0;
    }
}

#endif

}  // namespace dsac
