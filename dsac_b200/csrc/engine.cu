// engine.cu -- C ABI of the H100 hypothesis engine (include/dsac_b200.h): device memory,
// launches and host<->device copies.  No CPU fallback: every compute entry point needs a
// CUDA device and fails loudly otherwise.
#include <cuda_runtime.h>

#include <chrono>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <climits>
#include <cstring>
#include <numeric>
#include <random>
#include <string>
#include <vector>

#include "../../include/dsac_b200.h"
#include "backward.cuh"
#include "kernels.cuh"
#include "refine.cuh"
#include "sampler_split.cuh"
#include "guided.cuh"
#include "rgbd.cuh"
#include "train.cuh"
#include "uncertainty.cuh"
#include "modes.cuh"
#include "rig.cuh"
#include "upstream.cuh"
#include "objtrain.cuh"
#include "scoretrain.cuh"

using namespace dsac;

static_assert(sizeof(Cam) == sizeof(dsac_camera), "Cam mirrors dsac_camera");
static_assert(PRIOR_MAX == DSAC_MAX_PRIORS && PRIOR_ST_BAD == DSAC_ST_BAD_PRIOR, "prior.cuh mirrors dsac_b200.h");
static_assert(MODE_MAX == DSAC_MAX_MODES && DSAC_MAX_HYPS <= 1024, "modes.cuh mirrors dsac_b200.h");
static_assert(RIG_MAX_CAMERAS == DSAC_MAX_RIG_CAMERAS && RIG_ST_BAD == DSAC_ST_BAD_RIG && DSAC_MAX_HYPS <= 2048 &&
                  RIG_ST_SPOILED == (DSAC_ST_BAD_RIG | DSAC_ST_BAD_PRIOR),
              "refine.cuh mirrors dsac_b200.h (a rig's selection codes a cell in 11 bits)");
static_assert(sizeof(ObjCam) == sizeof(dsac_rgbd_camera) && offsetof(ObjCam, sensor_trans) == offsetof(dsac_rgbd_camera, sensor_trans) &&
                  offsetof(ObjCam, raw_data) == offsetof(dsac_rgbd_camera, raw_data),
              "ObjCam mirrors dsac_rgbd_camera");

static std::string g_create_error;

// The instantiations of the forward pass's kernel families, indexed by the pass's variant flags in one order:
// [per-frame camera][RGB-D][prior gate], then a family's own flag (k1_solve: four lanes per candidate, k_score: write the
// diffmaps).  dsac_engine_create sets their attributes through the same tables.
static constexpr void (*k_sample_tab[2][2][2])(SampleParams) = {
    {{k_sample_t<false, false, false>, k_sample_t<false, false, true>}, {k_sample_t<false, true, false>, k_sample_t<false, true, true>}},
    {{k_sample_t<true, false, false>, k_sample_t<true, false, true>}, {k_sample_t<true, true, false>, k_sample_t<true, true, true>}}};
static constexpr void (*k1_gtail_tab[2][2][2])(K1SplitParams, GuidedGen) = {
    {{k1_gtail_t<false, false, false>, k1_gtail_t<false, false, true>}, {k1_gtail_t<false, true, false>, k1_gtail_t<false, true, true>}},
    {{k1_gtail_t<true, false, false>, k1_gtail_t<true, false, true>}, {k1_gtail_t<true, true, false>, k1_gtail_t<true, true, true>}}};
static constexpr void (*k1_solve_tab[2][2][2])(K1SplitParams) = {{{k1_solve, k1_solve4}, {k1_solve_gate, k1_solve4_gate}},
                                                                 {{k1_solve_cam, k1_solve4_cam}, {k1_solve_cam_gate, k1_solve4_cam_gate}}};
static constexpr void (*k1_kabsch_tab[2][2])(K1SplitParams) = {{k1_kabsch_t<false, false>, k1_kabsch_t<false, true>},
                                                               {k1_kabsch_t<true, false>, k1_kabsch_t<true, true>}};
static constexpr void (*k1_filter_tab[2])(K1SplitParams) = {k1_filter, k1_filter_cam};
static constexpr void (*k1_cells_tab[2])(K1SplitParams, int, int) = {k1_cells, k1_cells_cam};
static constexpr void (*k_rgbd_eye_tab[2])(const float*, const int32_t*, int, Cam, const Cam*, const uint32_t*, double*, uint32_t*) = {
    k_rgbd_eye_t<false>, k_rgbd_eye_t<true>};
static constexpr void (*k_score_tab[2][2])(ScoreParams) = {{k_score<false>, k_score<true>}, {k_score_cam<false>, k_score_cam<true>}};
static constexpr void (*k_score_rig_tab[2][2])(ScoreParams) = {{k_score_rig<false, false>, k_score_rig<true, false>},
                                                                {k_score_rig<false, true>, k_score_rig<true, true>}};

// Owners of the engine's CUDA resources, the only code here that frees any.  Each releases what it holds in its
// destructor, is move-only, and converts to the raw pointer or handle for use at call sites.
template <typename T, cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
class Mem {
  public:
    Mem() = default;
    Mem(Mem&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; o.bytes_ = 0; }
    Mem& operator=(Mem&& o) noexcept { std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); return *this; }
    ~Mem() { release(); }
    // Grow-only: a request beyond the capacity frees the old block before it allocates the new one (the contents are not
    // kept, and a block of gigabytes is never held twice), with a quarter more with `headroom`.  On failure the buffer is
    // empty and the CUDA error is returned.
    cudaError_t reserve(size_t bytes, bool headroom = false) {
        if (bytes <= bytes_) return cudaSuccess;
        release();
        const size_t cap = headroom ? bytes + bytes / 4 : bytes;
        void* p = nullptr;
        const cudaError_t st = Alloc(&p, cap);
        if (st != cudaSuccess) return st;
        p_ = static_cast<T*>(p);
        bytes_ = cap;
        return cudaSuccess;
    }
    operator T*() const { return p_; }
    T* get() const { return p_; }
    size_t bytes() const { return bytes_; }

  private:
    void release() {
        if (p_) Free(p_);
        p_ = nullptr;
        bytes_ = 0;
    }
    T* p_ = nullptr;
    size_t bytes_ = 0;
};
template <typename T> using DevMem = Mem<T, cudaMalloc, cudaFree>;
template <typename T> using PinnedMem = Mem<T, cudaMallocHost, cudaFreeHost>;

template <typename H, cudaError_t (*Destroy)(H)>
class Handle {
  public:
    Handle() = default;
    Handle(Handle&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Handle& operator=(Handle&& o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Handle() { release(); }
    // where a cudaStreamCreate* / cudaEventCreate* call writes the new handle (what the owner held is released first)
    H* put() {
        release();
        return &h_;
    }
    operator H() const { return h_; }

  private:
    void release() {
        if (h_) Destroy(h_);
        h_ = nullptr;
    }
    H h_ = nullptr;
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;

// The per-frame settings of the following passes, indices into dsac_engine::set.  SET_RIG_PRIORS and SET_RIG_DEPTH are
// read by the rig pass only; every other forward pass refuses to start while one of them is set.
enum { SET_CAMS, SET_LOGITS, SET_DEPTH, SET_PRIORS, SET_RIG_PRIORS, SET_RIG_DEPTH, SET_COUNT };

// One per-frame setting: the frames it covers (0: off), a generation that changes with every update, and the event
// recorded after an update's copy or kernel, which a pass waits for before it reads the setting's buffers.
struct Setting {
    int n = 0;
    unsigned long long gen = 0;
    Event ev;
};

// The forward pass the engine holds, which the backward passes and the pose queries read: its inputs and the snapshot
// of the settings it ran with.
struct Pass {
    int32_t kind = 0;               // DSAC_PASS_SOFTAM, DSAC_PASS_DSAC, DSAC_PASS_RIG, or 0: none
    int n = 0;
    const int16_t* coords = nullptr;
    const int32_t* pix = nullptr;
    int pix_shared = 0;
    const double* gt = nullptr;
    long long frame0 = 0;
    uint32_t stages = DSAC_STAGE_ALL;   // the stages the pass ran (dsac_set_stages)
    uint32_t seed = 0;
    unsigned long long gen[SET_COUNT] = {};
    int set_n[SET_COUNT] = {};
    int prior_k = 0;                // priors per frame
    // the prior tables the sampler and k_prior_inject read: the pose priors' (dsac_set_pose_priors_device), or a rig pass's
    // composition of the rig pose priors with its extrinsics (k_rig_prior_prep)
    const double* prior_pose = nullptr;     // [n][prior_k][6]
    const PriorGate* prior_tab = nullptr;   // [n][prior_k] (a gate only)
    const uint32_t* prior_bad = nullptr;    // [n]
    bool prior_gate = false;
    double prior_chi2 = 0;
    int rig_c = 0;                  // a rig pass's cameras per rig (its gt: the rig ground truth, null without DSAC_STAGE_EVAL)
    // the cell depth the pass read: the cell depth setting's (d_depth) or, in a rig pass, the rig cell depth's (d_rig_depth);
    // null: an RGB pass
    const float* depth = nullptr;
    bool rgbd() const { return depth != nullptr; }
    // a rig pass scored by the rig score hooks (dsac_set_rig_score_hooks): the pair and user it called, which the rig
    // backward must find registered still; all null: scored in closed form
    dsac_score_hook rig_hook = nullptr;
    dsac_score_backward_hook rig_bw_hook = nullptr;
    void* rig_hook_user = nullptr;
};

struct dsac_engine {
    dsac_config cfg;
    std::string err;
    int64_t launches = 0;
    uint32_t stages = DSAC_STAGE_ALL;
    dsac_score_hook hook = nullptr;
    void* hook_user = nullptr;
    dsac_score_backward_hook bw_hook = nullptr;
    void* bw_hook_user = nullptr;
    DevMem<double> d_ext_g;         // [n][H][N] dScore/dDiffMap from the backward hook, then its clamped input [n][H] (grow-only)
    // the rig score hooks (dsac_set_rig_score_hooks), read by the rig passes and the rig backward only
    dsac_score_hook rig_hook = nullptr;
    dsac_score_backward_hook rig_bw_hook = nullptr;
    void* rig_hook_user = nullptr;
    Event ev_fwd;                   // recorded after the last forward launch: the backward waits on it
    DevMem<double> d_kabsch;        // dsac_kabsch: inputs and outputs in one grow-only block
    DevMem<uint64_t> d_reg_keys;    // dsac_register_depth_device: per-pixel scatter keys, grow-only
    int sm_count = 132;
    // inputs (device copies for the host-buffer entry point)
    DevMem<int16_t> d_coords;
    DevMem<int32_t> d_pix;
    DevMem<double> d_gt;
    Pass pass;                      // the last forward pass
    int k1_slots = 296;             // resident k_sample CTAs on this GPU (SMs x CTAs/SM), set at creation
    Setting set[SET_COUNT];
    // per-frame cameras (dsac_set_cameras): sized once for max_frames; set[SET_CAMS].n == 0: the config's camera.  Its event
    // also guards the staging: it is rewritten only after the copy
    DevMem<Cam> d_cams;
    PinnedMem<dsac_camera> h_cams;  // staging of the copy to d_cams
    // guided sampling (dsac_set_sampling_logits_device): per-frame tables sized once for max_frames on first use; off: the
    // reference's uniform sampler
    DevMem<double> d_g_w;            // [max_frames][N] softmax of the logits
    DevMem<uint32_t> d_g_q, d_g_cum; // [max_frames][N] integer weights and their inclusive prefix sums
    DevMem<uint32_t> d_g_bad;        // [max_frames] DSAC_ST_BAD_WEIGHTS
    // RGB-D localisation (dsac_set_cell_depth_device): buffers sized once for max_frames on first use; off: RGB
    DevMem<float> d_depth;           // [max_frames][N] the setting's per-cell depth (mm)
    DevMem<double> d_eye;            // [max_frames][N][3] eye coordinates of the pass's cells, NaN without depth
    DevMem<uint32_t> d_rgbd_skip;    // [max_frames] status bits of frames that sample nothing (DSAC_ST_NO_DEPTH, ...)
    // pose priors (dsac_set_pose_priors_device): tables sized once for max_frames x DSAC_MAX_PRIORS on first use; off: none.
    // The prior of frame f, index j, takes hypothesis slot n_hyps - prior_k + j.
    DevMem<double> d_prior_pose;     // [n][prior_k][6] cv poses
    DevMem<double> d_prior_info;     // [n][prior_k][36] information matrices (a gate only)
    DevMem<PriorGate> d_prior_tab;   // [n][prior_k] what the gate reads (k_prior_prep)
    DevMem<uint32_t> d_prior_bad;    // [n] DSAC_ST_BAD_PRIOR or 0
    int prior_k = 0;
    bool prior_gate = false;
    double prior_chi2 = 0;
    // rig pose priors (dsac_set_rig_pose_priors_device): k rig poses per rig of rig_prior_c cameras, sized once for max_frames
    // x DSAC_MAX_PRIORS on first use; each rig pass composes them with its extrinsics into its own scratch (e->rig)
    DevMem<double> d_rig_prior_pose;  // [R][k][6] cv rig poses
    DevMem<double> d_rig_prior_info;  // [R][k][36] information matrices in the rig chart (a gate only)
    int rig_prior_k = 0, rig_prior_c = 0;
    bool rig_prior_gate = false;
    double rig_prior_chi2 = 0;
    // RGB-D rigs (dsac_set_rig_cell_depth_device): the rig passes' per-cell depth of rig_depth_c cameras per rig, sized once for
    // max_frames on first use; the passes' eye coordinates go to d_eye as an ordinary RGB-D pass's
    DevMem<float> d_rig_depth;       // [max_frames][N] (mm)
    int rig_depth_c = 0;
    // per-dataset cameras of the pre-training data paths (dsac_set_dataset_cameras), indexed by dataset frame; grow-only.
    // ds_cams_n == 0: no table.  ds_cam0 is entry 0 on the host: the frame size and raw_data every entry shares.
    DevMem<ObjCam> d_ds_cams;
    PinnedMem<ObjCam> h_ds_cams;    // staging of the copy to d_ds_cams
    Event ev_ds_cams;               // recorded after that copy: the staging is rewritten, and a reader starts, only after it
    Event ev_ds_use;                // recorded after the last launch that read the table: a new table is copied after it
    int ds_cams_n = 0;
    ObjCam ds_cam0{};
    // state
    DevMem<uint16_t> d_perm;
    DevMem<double> d_hyp_pose;
    DevMem<float> d_hyp_P;
    DevMem<int32_t> d_img_idx;
    DevMem<int32_t> d_cand_idx;
    DevMem<long long> d_stream_ncand;
    DevMem<unsigned long long> d_stream_endpos;
    // refine-all (DSAC variant) buffers, grown on use; d_ra_frame holds the job -> frame table for ra_jobs jobs
    DevMem<int32_t> d_ra_frame; DevMem<double> d_ra_pose, d_ra_loss, d_ra_rot, d_ra_t;
    DevMem<int32_t> d_ra_correct, d_ra_steps, d_ra_imap;
    size_t ra_jobs = 0;
    // per-frame results of k_dsac_draw: drawn hypothesis, expected loss, its errors
    DevMem<int32_t> d_dsac_pick; DevMem<double> d_dsac_exp, d_dsac_rot, d_dsac_terr;
    DevMem<int32_t> d_dsac_correct;
    PinnedMem<int32_t> h_totals;    // [2]: selected hypotheses and refinement jobs of dsac_backward_dsac_device
    DevMem<uint32_t> d_status;
    DevMem<unsigned long long> d_fragile;
    DevMem<unsigned long long> d_phase;   // K1 per-phase cycle counters (DSAC_K1_TIMERS=1), else null
    DevMem<float> d_diffmaps;
    DevMem<double> d_scores;
    DevMem<double> d_sf;
    DevMem<double> d_entropy;
    DevMem<double> d_avg;
    DevMem<double> d_ref;
    DevMem<int32_t> d_inlier_map;
    DevMem<int32_t> d_steps_done;
    DevMem<int32_t> d_n_perm;
    DevMem<double> d_loss;
    DevMem<double> d_rot_err;
    DevMem<double> d_t_err;
    DevMem<int32_t> d_correct;
    DevMem<unsigned int> d_frame_counter;
    PinnedMem<long long> h_stream_ncand;   // [max_frames][n_streams] (pinned, so that a submitted pass stays asynchronous)
    dsac_forward_out* pending_out = nullptr;   // results of a submitted, not yet awaited pass
    int pending_n = 0, pending_chunks = 0;
    BackwardScratch bw;             // views into bw_buf
    DevMem<char> bw_buf;            // the soft-argmax backward's scratch block, grow-only
    int coord_deriv = DSAC_DERIV_CENTRAL;   // dsac_set_coord_derivatives
    IftScratch ift;                 // views into ift_buf (implicit mode's recording replay)
    DevMem<char> ift_buf;
    // dsac_pose_uncertainty_device: its own recording replay (pose, cells, count per job), shared with no backward so
    // that a call changes no later result; ev_unc is recorded after a call's last launch and the next call waits on it
    IftScratch unc;
    uint32_t* unc_status = nullptr;   // [R] dsac_rig_pose_uncertainty_device: the rig status its replay ORs the abort bit into
    DevMem<char> unc_buf;
    Event ev_unc;
    // dsac_pose_modes_device and dsac_rig_pose_modes_device: their seeds, recording replay and covariances in one grow-only
    // block of their own, ordered by ev_modes as the uncertainty scratch is by ev_unc
    DevMem<char> modes_buf;
    Event ev_modes;
    // dsac_forward_rig_device: the extrinsics, the pool, its rows and scores and the per-rig results, views into rig_buf
    // (grow-only, sized for max_frames frames of the largest pool asked for)
    struct {
        double *ext, *cam_scores, *hyp, *scores, *sf, *entropy, *avg, *ref, *loss, *rot, *terr;
        float* P;
        int32_t *imap, *steps, *correct;
        uint32_t* status;
        double* prior_pose;         // [n][k][6] the rig pose priors composed per frame (k_rig_prior_prep), k of the setting
        PriorGate* prior_tab;       // [n][k]
        uint32_t* prior_bad;        // [n]
        float* dm;                  // [n][P][N] the error images of a hooked rig pass (rig_dm_buf)
    } rig = {};
    DevMem<char> rig_buf;
    DevMem<char> rig_dm_buf;        // grow-only, sized for the n frames and the pool of the largest hooked rig pass
    // dsac_backward_rig(_pose)_device: the soft-argmax backward's arrays over rigs and pools, the recording replay, the
    // composed poses, w and the support vectors, in one grow-only block that no other call writes, ordered by ev_rig_bw as
    // the uncertainty scratch is by ev_unc
    struct {
        BackwardScratch b;
        double *rec_pose, *w, *u, *frame_grad;
        double *ext_g, *hook_sog;   // a hooked rig pass: [n][P][N] dScore/dDiffMap from the backward hook, [n][P] its input
        uint16_t* rec_sel;
        int32_t *rec_count, *n_perm;
        uint32_t* status;
    } rig_bw = {};
    DevMem<char> rig_bw_buf;
    Event ev_rig_bw;
    std::vector<DevMem<char>> bw_pool;   // device buffers of dsac_backward_dsac, kept across calls
    Stream pipe[4];                 // chunked H2D / compute / D2H pipeline of dsac_forward
    // tail split (dsac_set_tail_split): the whole sampler waves of a batch run on a high-priority side stream, the
    // frames of the last, partial wave on the caller's stream, so that scoring / refinement of the first part fill
    // the SMs the partial wave leaves idle
    Stream hi;
    Event ev_fork, ev_join;
    int tail_split = 1;
    // split sampler (sampler_split.cuh): per-stream state and round buffers, sized at creation
    int k1_mode = 1;                // 1: round-based pipeline of flat kernels; 0: monolithic k_sample (DSAC_K1_MODE=mono)
    int k1_rounds = 3, k1_cap = 0;   // rounds 0..2 finish every stream of the benchmark batches; a straggler continues in k_sample (resume). 5 rounds = 6 empty launches per pass
    bool k1_rounds_fixed = false;   // DSAC_K1_ROUNDS given
    int k1_filter_grid = 0, k1_solve_grid = 0;
    unsigned long long k1_calls[4] = {0, 0, 0, 0};   // passes by sampler: [0] uniform, [1] guided, [2] gated uniform, [3] gated
                                                     // guided (parity selects the statistics block)
    DevMem<K1SlotState> d_k1_state;
    DevMem<CellRec> d_k1_celltab;
    DevMem<uint2> d_k1_cells;
    DevMem<uint32_t> d_k1_endw;
    DevMem<uint32_t> d_k1_accbits;
    DevMem<double> d_k1_pose;
    DevMem<uint2> d_k1_wq;
    DevMem<uint32_t> d_k1_fq;
    DevMem<int> d_k1_counters;                    // wq_n[K1S_MAX_ROUNDS], fq_n[K1S_MAX_ROUNDS]
    DevMem<unsigned long long> d_k1_stats;        // [4][2][2]: candidates / hypotheses of finished streams, by sampler (uniform,
                                                  // guided, and each of them gated by pose priors) and call parity: the first round
                                                  // of a pass is sized from the last pass of the same sampler, whose rate can differ
                                                  // from the others' many times over
    DevMem<unsigned long long> d_k1_dbg;          // [K1S_MAX_ROUNDS][4] (DSAC_K1_DEBUG=1 or dsac_sampler_profile), else null
    // dsac_sampler_profile: CUDA events between the sampler's launches of the last forward pass
    int k1_profile = 0;
    std::vector<Event> k1_ev;                     // event i is recorded after launch i (event 0 before the first)
    std::vector<int> k1_ev_kind;                  // 0 cells/slot (integer generation + selection), 1 filter, 2 solve, 3 resume tail
    int k1_ev_n = 0;
    // generator / filter overlap: k1_slot runs on the caller's stream, k1_filter + k1_solve on this side stream
    Stream k1_side;
    Stream k1_side2;                              // k1_solve, when it runs next to the following set's filter (overlap mode 2)
    Event k1_ev_filt[K1S_MAX_SETS];               // filter of launch set i done
    Event k1_ev_solve[K1S_MAX_SETS];              // solve of launch set i done
    Event k1_ev_gen[K1S_MAX_SETS];                // generation of launch set i done
    Event k1_ev_round;                            // last solve of a round done
    // a second, independent set of the per-pass sampler resources: a large batch runs as two concurrent half-batches (forward_split)
    struct K1Lane {
        Stream main, side, side2;
        Event ev_filt[K1S_MAX_SETS], ev_solve[K1S_MAX_SETS], ev_gen[K1S_MAX_SETS], ev_round;
        DevMem<int> counters;
        DevMem<unsigned long long> stats;
        unsigned long long calls[4] = {0, 0, 0, 0};
    } lane1;
    int k1_lanes = 1;                             // DSAC_K1_LANES: 0 = never split a batch into two lanes
    int k1_overlap = 1;
    bool k1_overlap_fixed = false;                // DSAC_K1_OVERLAP given
    int k1_solve_batch = 0;                       // 1: one k1_solve per round over the flagged candidates of all its launch sets (a per-set solve runs beside the next set's generator, a per-round one runs alone; on an H100 SXM at 700 W 3.05 vs 3.09 ms per 1024-frame step)
    DevMem<K1SlotState> d_k1_vstate;              // k1_spec: virtual slots of the speculative first round (few streams)
    DevMem<uint2> d_k1_vcells;
    DevMem<uint32_t> d_k1_vendw;
    DevMem<int> d_k1_spec_result;
    DevMem<int> d_k1_spec_table;
    DevMem<uint32_t> d_k1_chain;                  // k1_pipe: hand-over records of the window chain, [slots][K1Q_MAX_WIN + 1][4]
    unsigned long long k1_epoch = 0;              // k1_pipe: one value per launch, engine-wide (a stale hand-over record never matches)
    int k1_pipe = 0;                              // DSAC_K1_PIPE=1: chained generator for 9 .. ~190 streams (experimental, off by default)
    int k1_slot_capacity = 0;                     // CTAs of k1_pipe / k1_slot (256 threads) the GPU holds at once
    int k1_spec_slots = 0;                        // streams the scratch above was sized for (0: speculative round off)
    int k1_solve_group4 = 1;                      // DSAC_K1_SOLVE4: four lanes per flagged candidate for a few streams
    int k1_slot_threads = 0;                      // DSAC_K1_SLOT_THREADS: 256 / 512 / 1024 (0: by the number of streams)
    int k1_fused = 0;                             // 1: filter of set k and generator of set k+1 in one warp-specialised kernel (k1_fused)
    int k1_wq_stride = 0;
};

static int fail(dsac_engine* e, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (e) e->err = buf;
    else g_create_error = buf;
    return code;
}

#define CU(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t _st = (call);                                                                        \
        if (_st != cudaSuccess)                                                                          \
            return fail(e, DSAC_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_st), __FILE__, __LINE__); \
    } while (0)

extern "C" {

const char* dsac_version(void) { return "dsac_b200 0.1 (sm_90a)"; }

int dsac_default_config(dsac_config* c) {
    if (!c) return DSAC_ERR_ARG;
    memset(c, 0, sizeof(*c));
    c->focal = 525.0;                  // properties.cpp:55
    c->cx = 320.0; c->cy = 240.0;      // properties.cpp:310-311 (iw 640, ih 480, xs = ys = 0)
    c->n_hyps = 256;                   // properties.cpp:45
    c->thr2d = 10;                     // properties.cpp:50, int-truncated at test_ransac_softam.cpp:51
    c->inlier_count = 100;             // properties.cpp:47
    c->ref_steps = 8;                  // properties.cpp:46
    c->sub_sample = 0.01;              // properties.cpp:48
    c->alpha = 0.1; c->beta = 0.5;     // engine defaults (BASELINE.md section 2); not reference values
    c->seed = 1305;                    // thread_rand.h:100
    c->n_streams = 1;
    c->stream_skip = 6400;
    c->max_candidates = 1 << 20;
    c->fix_q4 = 0;
    c->grad_clamp = 0.1;               // train_score_softam.lua:13
    c->write_diffmaps = 1;
    c->device = 0;
    c->max_frames = 1;
    c->hyps_per_cta = 0;
    return DSAC_OK;
}

const char* dsac_last_error(const dsac_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int dsac_engine_config(const dsac_engine* e, dsac_config* out) {
    if (!e || !out) return DSAC_ERR_ARG;
    *out = e->cfg;
    return DSAC_OK;
}

void dsac_engine_destroy(dsac_engine* e) {
    if (!e) return;
    cudaSetDevice(e->cfg.device);
    // nothing is freed while work on the engine's streams may still use it
    const cudaStream_t streams[] = {e->pipe[0], e->pipe[1], e->pipe[2], e->pipe[3], e->hi, e->k1_side, e->k1_side2,
                                    e->lane1.main, e->lane1.side, e->lane1.side2};
    for (cudaStream_t st : streams)
        if (st) cudaStreamSynchronize(st);
    if (e->d_phase) {
        unsigned long long h[16];
        if (cudaMemcpy(h, e->d_phase, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess)
            fprintf(stderr, "[dsac K1 thread-0 cycles] A1 gen %llu  A2 bounds %llu  B filter %llu  C queue %llu  D full %llu  E advance %llu\n"
                            "[dsac k1_slot thread-0 cycles] regenerate+decode %llu  scan %llu  walk %llu  starts %llu  write %llu  leftover %llu\n",
                    h[0], h[1], h[2], h[3], h[4], h[5], h[8], h[9], h[10], h[11], h[12], h[13]);
    }
    if (e->d_k1_dbg && e->d_k1_spec_result && e->k1_spec_slots > 0) {
        int h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (cudaMemcpy(h, e->d_k1_spec_result, std::min(8, e->k1_spec_slots) * sizeof(int), cudaMemcpyDeviceToHost) == cudaSuccess)
            fprintf(stderr, "[dsac k1_spec, last call] windows stitched per stream (0 = speculation abandoned or not used): %d %d %d %d %d %d %d %d\n",
                    h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7]);
    }
    if (e->d_k1_dbg) {
        unsigned long long h[K1S_MAX_ROUNDS * 4];
        if (cudaMemcpy(h, e->d_k1_dbg, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess)
            for (int r = 0; r < K1S_MAX_ROUNDS && (h[r * 4] || r == 0); r++)
                fprintf(stderr, "[dsac K1 split, last call] round %d: %llu active streams, %llu candidates, %llu flagged, %llu accepted\n", r,
                        h[r * 4], h[r * 4 + 1], h[r * 4 + 2], h[r * 4 + 3]);
    }
    delete e;
}

int dsac_engine_create(const dsac_config* cfg, dsac_engine** out) {
    dsac_engine* e = nullptr;
    if (!cfg || !out) return fail(e, DSAC_ERR_ARG, "null argument");
    *out = nullptr;
    if (cfg->n_hyps < 1 || cfg->n_hyps > DSAC_MAX_HYPS) return fail(e, DSAC_ERR_ARG, "n_hyps out of range [1,%d]", DSAC_MAX_HYPS);
    if (cfg->n_streams < 1 || cfg->n_streams > cfg->n_hyps) return fail(e, DSAC_ERR_ARG, "n_streams out of range [1,n_hyps]");
    if (cfg->inlier_count < 1 || cfg->inlier_count > K4_MAX_INLIERS) return fail(e, DSAC_ERR_ARG, "inlier_count out of range [1,%d]", K4_MAX_INLIERS);
    if (cfg->ref_steps < 0 || cfg->ref_steps > DSAC_MAX_REF_STEPS) return fail(e, DSAC_ERR_ARG, "ref_steps out of range [0,%d]", DSAC_MAX_REF_STEPS);
    if (cfg->max_frames < 1) return fail(e, DSAC_ERR_ARG, "max_frames must be >= 1");
    int ndev = 0;
    cudaError_t st = cudaGetDeviceCount(&ndev);
    if (st != cudaSuccess || ndev == 0)
        return fail(e, DSAC_ERR_NODEVICE, "no CUDA device available (%s); the engine has no CPU path",
                    st == cudaSuccess ? "device count 0" : cudaGetErrorString(st));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(e, DSAC_ERR_ARG, "device %d out of range (have %d)", cfg->device, ndev);
    e = new dsac_engine();
    e->cfg = *cfg;
    if (e->cfg.max_candidates <= 0) e->cfg.max_candidates = 1 << 20;
    auto bail = [&](int code) {
        g_create_error = e->err;
        delete e;
        return code;
    };
#define CUC(call)                                                                                   \
    do {                                                                                            \
        cudaError_t _s = (call);                                                                    \
        if (_s != cudaSuccess) {                                                                    \
            fail(e, DSAC_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(_s));                  \
            return bail(DSAC_ERR_CUDA);                                                             \
        }                                                                                           \
    } while (0)
    CUC(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUC(cudaGetDeviceProperties(&prop, cfg->device));
    e->sm_count = prop.multiProcessorCount;
    const size_t n = (size_t)cfg->max_frames, H = (size_t)cfg->n_hyps, N = DSAC_N;
    CUC(e->d_coords.reserve(n * N * 3 * sizeof(int16_t)));
    CUC(e->d_pix.reserve(n * N * 2 * sizeof(int32_t)));
    CUC(e->d_gt.reserve(n * 12 * sizeof(double)));
    CUC(e->d_perm.reserve((size_t)std::max(1, cfg->ref_steps) * N * sizeof(uint16_t)));
    CUC(e->d_hyp_pose.reserve(n * H * 6 * sizeof(double)));
    CUC(e->d_hyp_P.reserve(n * H * 12 * sizeof(float)));
    CUC(e->d_img_idx.reserve(n * H * 4 * sizeof(int32_t)));
    CUC(e->d_cand_idx.reserve(n * H * sizeof(int32_t)));
    CUC(e->d_stream_ncand.reserve(n * cfg->n_streams * sizeof(long long)));
    CUC(e->d_stream_endpos.reserve(n * cfg->n_streams * sizeof(unsigned long long)));
    CUC(e->d_status.reserve(n * sizeof(uint32_t)));
    CUC(e->d_fragile.reserve(sizeof(unsigned long long)));
    if (cfg->write_diffmaps) CUC(e->d_diffmaps.reserve(n * H * N * sizeof(float)));
    CUC(e->d_scores.reserve(n * H * sizeof(double)));
    CUC(e->d_sf.reserve(n * H * sizeof(double)));
    CUC(e->d_entropy.reserve(n * sizeof(double)));
    CUC(e->d_avg.reserve(n * 6 * sizeof(double)));
    CUC(e->d_ref.reserve(n * 6 * sizeof(double)));
    CUC(e->d_inlier_map.reserve(n * N * sizeof(int32_t)));
    CUC(e->d_steps_done.reserve(n * sizeof(int32_t)));
    CUC(e->d_n_perm.reserve(n * sizeof(int32_t)));
    CUC(e->d_loss.reserve(n * sizeof(double)));
    CUC(e->d_rot_err.reserve(n * sizeof(double)));
    CUC(e->d_t_err.reserve(n * sizeof(double)));
    CUC(e->d_correct.reserve(n * sizeof(int32_t)));
    CUC(e->d_frame_counter.reserve(n * sizeof(unsigned int)));
    CUC(e->d_dsac_pick.reserve(n * sizeof(int32_t)));
    CUC(e->d_dsac_exp.reserve(n * sizeof(double)));
    CUC(e->d_dsac_rot.reserve(n * sizeof(double)));
    CUC(e->d_dsac_terr.reserve(n * sizeof(double)));
    CUC(e->d_dsac_correct.reserve(n * sizeof(int32_t)));
    CUC(e->h_totals.reserve(2 * sizeof(int32_t)));
    CUC(e->d_cams.reserve(n * sizeof(Cam)));
    CUC(e->h_cams.reserve(n * sizeof(dsac_camera)));
    for (Setting& s : e->set) CUC(cudaEventCreateWithFlags(s.ev.put(), cudaEventDisableTiming));
    CUC(cudaEventCreateWithFlags(e->ev_ds_cams.put(), cudaEventDisableTiming));
    CUC(cudaEventCreateWithFlags(e->ev_ds_use.put(), cudaEventDisableTiming));
    CUC(cudaMemset(e->d_frame_counter, 0, n * sizeof(unsigned int)));
    CUC(cudaMemset(e->d_fragile, 0, sizeof(unsigned long long)));
    if (getenv("DSAC_K1_TIMERS")) {
        CUC(e->d_phase.reserve(16 * sizeof(unsigned long long)));
        CUC(cudaMemset(e->d_phase, 0, 16 * sizeof(unsigned long long)));
    }
    CUC(cudaMemset(e->d_status, 0, n * sizeof(uint32_t)));
    CUC(cudaMemset(e->d_steps_done, 0, n * sizeof(int32_t)));
    CUC(cudaMemset(e->d_n_perm, 0, n * sizeof(int32_t)));
    CUC(cudaMemset(e->d_inlier_map, 0, n * N * sizeof(int32_t)));
    CUC(cudaMemset(e->d_ref, 0, n * 6 * sizeof(double)));
    CUC(cudaMemset(e->d_loss, 0, n * sizeof(double)));
    CUC(cudaMemset(e->d_rot_err, 0, n * sizeof(double)));
    CUC(cudaMemset(e->d_t_err, 0, n * sizeof(double)));
    CUC(cudaMemset(e->d_correct, 0, n * sizeof(int32_t)));
    // refinement permutations: std::mt19937 randG (default seed) once per frame, iota +
    // std::shuffle per step with the continuing generator (cnn_softam.h:1104,1112-1114) --
    // identical for every frame, so they are built once with the very same libstdc++ calls.
    {
        std::mt19937 randG;
        std::vector<uint16_t> perm((size_t)std::max(1, cfg->ref_steps) * N, 0);
        for (int s = 0; s < cfg->ref_steps; s++) {
            std::vector<int> idx(N);
            for (size_t i = 0; i < N; i++) idx[i] = (int)i;
            std::shuffle(idx.begin(), idx.end(), randG);
            for (size_t i = 0; i < N; i++) perm[(size_t)s * N + i] = (uint16_t)idx[i];
        }
        CUC(cudaMemcpy(e->d_perm, perm.data(), perm.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
    }
    for (const auto& by_rgbd : k_sample_tab)
        for (const auto& by_gate : by_rgbd)
            for (auto kern : by_gate) CUC(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(K1Smem)));
    // k_refine wants 8 CTAs x 26 KB of shared memory per SM: ask for the carve-out explicitly (the default heuristic
    // need not pick the split the launch bounds were written for).  k_sample is left to the default: it spills to
    // local memory, so it wants the L1 that the largest carve-out would take away (DSAC_K1_CARVEOUT overrides).
    for (int cam = 0; cam < 2; cam++) {
        CUC(cudaFuncSetAttribute(k_refine_tab[cam], cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        CUC(cudaFuncSetAttribute(k_refine_rgbd_tab[cam], cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        CUC(cudaFuncSetAttribute(k_refine_rig_tab[cam], cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        // the RGB-D rig refinement stages its Kabsch fit's point pairs in dynamic shared memory (refine.cuh)
        CUC(cudaFuncSetAttribute(k_refine_rig_rgbd_tab[cam], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rig_kabsch_smem(RIG_MAX_CAMERAS)));
        CUC(cudaFuncSetAttribute(k_refine_rig_rgbd_rec_tab[cam], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rig_kabsch_smem(RIG_MAX_CAMERAS)));
        if (const char* co = getenv("DSAC_K1_CARVEOUT"))
            CUC(cudaFuncSetAttribute(k_sample_tab[cam][0][0], cudaFuncAttributePreferredSharedMemoryCarveout, atoi(co)));
    }
    {
        int per_sm = 0, sms = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_sample_tab[0][0][0], K1_THREADS, sizeof(K1Smem));
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
        if (per_sm > 0 && sms > 0) e->k1_slots = per_sm * sms;
    }
    CUC(e->h_stream_ncand.reserve(n * cfg->n_streams * sizeof(long long)));
    if (const char* m = getenv("DSAC_K1_MODE")) e->k1_mode = (strcmp(m, "mono") == 0) ? 0 : 1;
    if (const char* r = getenv("DSAC_K1_ROUNDS")) { e->k1_rounds = std::max(1, std::min(K1S_MAX_ROUNDS - 1, atoi(r))); e->k1_rounds_fixed = true; }
    if (e->k1_mode) {
        const size_t T = (size_t)cfg->n_streams, slots = n * T;
        const int quota_max = (cfg->n_hyps + cfg->n_streams - 1) / cfg->n_streams;
        // few streams (single-frame latency): the first round takes 115 % of the expected need, so the capacity is larger
        const int cap_per_hyp = slots < 128 ? (K1S_CAP_PER_HYP * 3) / 2 : K1S_CAP_PER_HYP;
        int cap = std::min(K1S_MAX_CAP, std::max(1024, cap_per_hyp * quota_max));
        cap = (cap + 1023) & ~1023;     // a round is generated in portions of cap / 4, themselves multiples of 256
        e->k1_cap = cap;
        e->k1_wq_stride = (int)(slots * 128);
        CUC(e->d_k1_state.reserve(slots * sizeof(K1SlotState)));
        CUC(e->d_k1_celltab.reserve(n * N * sizeof(CellRec)));
        CUC(e->d_k1_cells.reserve(slots * cap * sizeof(uint2)));
        CUC(e->d_k1_endw.reserve(slots * cap * sizeof(uint32_t)));
        CUC(e->d_k1_accbits.reserve(slots * (cap / 32) * sizeof(uint32_t)));
        CUC(e->d_k1_pose.reserve(slots * cap * 6 * sizeof(double)));
        CUC(e->d_k1_wq.reserve((size_t)K1S_MAX_SETS * slots * 128 * sizeof(uint2)));
        CUC(e->d_k1_fq.reserve(2 * slots * cap * sizeof(uint32_t)));   // two regions: the filter of set k+1 writes one while the solve of set k reads the other
        CUC(e->d_k1_counters.reserve(2 * K1S_MAX_SETS * sizeof(int)));
        CUC(e->d_k1_chain.reserve(slots * (K1Q_MAX_WIN + 1) * 4 * sizeof(uint32_t)));
        CUC(cudaMemset(e->d_k1_chain, 0, slots * (K1Q_MAX_WIN + 1) * 4 * sizeof(uint32_t)));
        {
            int per_sm = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k1_pipe, K1S_THREADS, 0);
            e->k1_slot_capacity = std::max(1, per_sm) * e->sm_count;
            if (const char* pv = getenv("DSAC_K1_PIPE")) e->k1_pipe = atoi(pv);
        }
        {   // speculative first round for a few streams (sampler_split.cuh: k1_spec / k1_stitch); DSAC_K1_SPEC=0 turns it off
            int want = 1;
            if (const char* sv = getenv("DSAC_K1_SPEC")) want = atoi(sv);
            if (want) {
                const size_t ss = std::min<size_t>(slots, 8);    // 8 frames x 1 stream: 0.513 -> 0.466 ms per step (H100 SXM, 700 W); at 16 frames the 1360 window CTAs are no longer one wave
                CUC(e->d_k1_vstate.reserve(ss * K1P_VPER * sizeof(K1SlotState)));
                CUC(e->d_k1_vcells.reserve(ss * K1P_VPER * K1P_CAPW * sizeof(uint2)));
                CUC(e->d_k1_vendw.reserve(ss * K1P_VPER * K1P_CAPW * sizeof(uint32_t)));
                CUC(e->d_k1_spec_result.reserve(ss * sizeof(int)));
                CUC(cudaMemset(e->d_k1_spec_result, 0, ss * sizeof(int)));
                CUC(e->d_k1_spec_table.reserve(ss * K1P_TABLE * sizeof(int)));
                e->k1_spec_slots = (int)ss;
            }
        }
        {   // the fp64 kernels get the higher priority: when a generator launch and a filter launch become ready together,
            // the persistent filter CTAs are placed first and the generator's CTAs fill the registers they leave free
            int least = 0, greatest = 0;
            CUC(cudaDeviceGetStreamPriorityRange(&least, &greatest));
            int prio = greatest;
            if (const char* pr = getenv("DSAC_K1_SIDE_PRIO")) prio = atoi(pr) ? greatest : least;
            CUC(cudaStreamCreateWithPriority(e->k1_side.put(), cudaStreamNonBlocking, prio));
            CUC(cudaStreamCreateWithPriority(e->k1_side2.put(), cudaStreamNonBlocking, prio));
            for (int i = 0; i < K1S_MAX_SETS; i++) {
                CUC(cudaEventCreateWithFlags(e->k1_ev_filt[i].put(), cudaEventDisableTiming));
                CUC(cudaEventCreateWithFlags(e->k1_ev_solve[i].put(), cudaEventDisableTiming));
            }
        }
        for (int i = 0; i < K1S_MAX_SETS; i++) CUC(cudaEventCreateWithFlags(e->k1_ev_gen[i].put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->k1_ev_round.put(), cudaEventDisableTiming));
        {   // the second lane (forward_split: two concurrent half-batches)
            int least = 0, greatest = 0;
            CUC(cudaDeviceGetStreamPriorityRange(&least, &greatest));
            dsac_engine::K1Lane& L = e->lane1;
            CUC(cudaStreamCreateWithFlags(L.main.put(), cudaStreamNonBlocking));
            CUC(cudaStreamCreateWithPriority(L.side.put(), cudaStreamNonBlocking, greatest));
            CUC(cudaStreamCreateWithPriority(L.side2.put(), cudaStreamNonBlocking, greatest));
            for (int i = 0; i < K1S_MAX_SETS; i++) {
                CUC(cudaEventCreateWithFlags(L.ev_filt[i].put(), cudaEventDisableTiming));
                CUC(cudaEventCreateWithFlags(L.ev_solve[i].put(), cudaEventDisableTiming));
                CUC(cudaEventCreateWithFlags(L.ev_gen[i].put(), cudaEventDisableTiming));
            }
            CUC(cudaEventCreateWithFlags(L.ev_round.put(), cudaEventDisableTiming));
            CUC(L.counters.reserve(2 * K1S_MAX_SETS * sizeof(int)));
            CUC(L.stats.reserve(16 * sizeof(unsigned long long)));
            CUC(cudaMemset(L.stats, 0, 16 * sizeof(unsigned long long)));
            if (const char* ln = getenv("DSAC_K1_LANES")) e->k1_lanes = atoi(ln);
        }
        if (const char* ov = getenv("DSAC_K1_OVERLAP")) { e->k1_overlap = atoi(ov); e->k1_overlap_fixed = true; }
        if (const char* fu = getenv("DSAC_K1_FUSED")) e->k1_fused = atoi(fu);
        if (const char* stt = getenv("DSAC_K1_SLOT_THREADS")) e->k1_slot_threads = atoi(stt);
        if (const char* s4 = getenv("DSAC_K1_SOLVE4")) e->k1_solve_group4 = atoi(s4);
        if (const char* sb = getenv("DSAC_K1_SOLVE_BATCH")) e->k1_solve_batch = atoi(sb);
        CUC(cudaFuncSetAttribute(k1_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(K1XSmem)));
        CUC(e->d_k1_stats.reserve(16 * sizeof(unsigned long long)));
        CUC(cudaMemset(e->d_k1_stats, 0, 16 * sizeof(unsigned long long)));
        if (getenv("DSAC_K1_DEBUG")) CUC(e->d_k1_dbg.reserve(K1S_MAX_ROUNDS * 4 * sizeof(unsigned long long)));
        for (auto kern : k1_filter_tab) CUC(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(K1FSmem)));
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k1_filter, K1F_THREADS, sizeof(K1FSmem));
        e->k1_filter_grid = std::max(1, per_sm) * e->sm_count;
        per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k1_solve, K1V_THREADS, 0);
        e->k1_solve_grid = std::max(1, per_sm) * e->sm_count;
        if (const char* g = getenv("DSAC_K1_FILTER_GRID")) e->k1_filter_grid = std::max(1, atoi(g));
        if (const char* g = getenv("DSAC_K1_SOLVE_GRID")) e->k1_solve_grid = std::max(1, atoi(g));
    }
    for (int i = 0; i < 4; i++) CUC(cudaStreamCreateWithFlags(e->pipe[i].put(), cudaStreamNonBlocking));
    {
        int least = 0, greatest = 0;
        CUC(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        CUC(cudaStreamCreateWithPriority(e->hi.put(), cudaStreamNonBlocking, greatest));
        CUC(cudaEventCreateWithFlags(e->ev_fork.put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->ev_join.put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->ev_fwd.put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->ev_unc.put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->ev_modes.put(), cudaEventDisableTiming));
        CUC(cudaEventCreateWithFlags(e->ev_rig_bw.put(), cudaEventDisableTiming));
        if (const char* ts = getenv("DSAC_TAIL_SPLIT")) e->tail_split = atoi(ts);
    }
#undef CUC
    *out = e;
    return DSAC_OK;
}

int dsac_set_stages(dsac_engine* e, uint32_t mask) {
    if (!e) return DSAC_ERR_ARG;
    e->stages = mask;
    return DSAC_OK;
}

int dsac_set_tail_split(dsac_engine* e, int32_t mode) {
    if (!e) return DSAC_ERR_ARG;
    if (mode < 0 || mode > 2) return fail(e, DSAC_ERR_ARG, "tail split mode %d out of range [0,2]", mode);
    e->tail_split = mode;
    return DSAC_OK;
}

int dsac_set_coord_derivatives(dsac_engine* e, int32_t mode) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_set_coord_derivatives: a submitted pass has not been awaited (dsac_forward_wait)");
    if (mode != DSAC_DERIV_CENTRAL && mode != DSAC_DERIV_IMPLICIT)
        return fail(e, DSAC_ERR_ARG, "dsac_set_coord_derivatives: mode %d is neither DSAC_DERIV_CENTRAL (0) nor DSAC_DERIV_IMPLICIT (1)", mode);
    e->coord_deriv = mode;
    return DSAC_OK;
}

// The steps every setter of a per-frame setting shares.  A clear changes the generation only if the setting was on.
static void setting_clear(Setting& s) {
    if (s.n) s.gen++;
    s.n = 0;
}
// An update turns the setting off until setting_commit, so that a failed copy or launch leaves it off, and `stream` waits
// for the last forward pass, which may still read the setting's buffers.
static int setting_begin(dsac_engine* e, Setting& s, cudaStream_t stream) {
    s.n = 0;
    s.gen++;
    CU(cudaStreamWaitEvent(stream, e->ev_fwd, 0));
    return DSAC_OK;
}
static int setting_commit(dsac_engine* e, Setting& s, int32_t n, cudaStream_t stream) {
    CU(cudaEventRecord(s.ev, stream));
    s.n = n;
    return DSAC_OK;
}

int dsac_set_cameras(dsac_engine* e, int32_t n, const dsac_camera* cams, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_set_cameras: a submitted pass has not been awaited (dsac_forward_wait)");
    Setting& s = e->set[SET_CAMS];
    if (!cams) {
        setting_clear(s);
        return DSAC_OK;
    }
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_ARG, "dsac_set_cameras: n %d out of range [1,%d]", n, e->cfg.max_frames);
    for (int32_t i = 0; i < n; i++) {
        const dsac_camera& c = cams[i];
        if (!std::isfinite(c.focal) || !(c.focal > 0) || !std::isfinite(c.cx) || !std::isfinite(c.cy))
            return fail(e, DSAC_ERR_ARG, "dsac_set_cameras: camera %d is invalid (focal %g must be finite and > 0, cx %g and cy %g finite)", i,
                        c.focal, c.cx, c.cy);
    }
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaEventSynchronize(s.ev));                   // the previous copy has left the staging buffer
    memcpy(e->h_cams.get(), cams, (size_t)n * sizeof(dsac_camera));
    if (int rc = setting_begin(e, s, stream)) return rc;
    CU(cudaMemcpyAsync(e->d_cams.get(), e->h_cams.get(), (size_t)n * sizeof(dsac_camera), cudaMemcpyHostToDevice, stream));
    return setting_commit(e, s, n, stream);
}

// What the pass start reports for a batch that does not match a setting: "n_frames %d differs from the %d <frames>",
// and what a consumer of the pass reports when the setting changed after it: "the <changed> changed".
static const struct {
    const char* setter;
    const char* frames;
    const char* changed;
} k_setting[SET_COUNT] = {
    {"dsac_set_cameras", "cameras set by dsac_set_cameras", "cameras were"},
    {"dsac_set_sampling_logits_device", "frames of the sampling logits (dsac_set_sampling_logits_device)", "sampling logits were"},
    {"dsac_set_cell_depth_device", "frames of the cell depth (dsac_set_cell_depth_device)", "cell depth was"},
    {"dsac_set_pose_priors_device", "frames of the pose priors (dsac_set_pose_priors_device)", "pose priors were"},
    {"dsac_set_rig_pose_priors_device", "frames of the rig pose priors (dsac_set_rig_pose_priors_device)", "rig pose priors were"},
    {"dsac_set_rig_cell_depth_device", "frames of the rig cell depth (dsac_set_rig_cell_depth_device)", "rig cell depth was"},
};

// The start every forward entry point shares: the batch matches each setting in force, each of `streams` waits for the
// settings' updates, and the record of the pass takes its inputs and the settings' snapshot.  A pipeline's entry point
// sets the record's kind once the engine holds a pass of it.  rig: the rig pass, the only one that reads the rig pose
// priors, the rig cell depth and the rig score hooks; any other refuses while one of them is set rather than ignore it.
static int pass_begin(dsac_engine* e, int32_t kind, int32_t n, int64_t frame0, const int16_t* coords, const int32_t* pix,
                      int32_t pix_shared, const double* gt, std::initializer_list<cudaStream_t> streams, bool rig = false) {
    if (e->rig_hook && !rig)
        return fail(e, DSAC_ERR_ARG,
                    "rig score hooks are registered (dsac_set_rig_score_hooks), which only dsac_forward_rig_device calls: clear them first");
    Pass p;
    for (int i = 0; i < SET_COUNT; i++) {
        const Setting& s = e->set[i];
        if (i == SET_RIG_PRIORS && s.n && !rig)
            return fail(e, DSAC_ERR_ARG, "rig pose priors are set (%s), which only dsac_forward_rig_device reads: clear them first",
                        k_setting[i].setter);
        if (i == SET_RIG_DEPTH && s.n && !rig)
            return fail(e, DSAC_ERR_ARG, "rig cell depth is set (%s), which only dsac_forward_rig_device reads: clear it first",
                        k_setting[i].setter);
        if (s.n && n != s.n) return fail(e, DSAC_ERR_ARG, "n_frames %d differs from the %d %s", n, s.n, k_setting[i].frames);
        if (s.n)
            for (cudaStream_t st : streams) CU(cudaStreamWaitEvent(st, s.ev, 0));
        p.gen[i] = s.gen;
        p.set_n[i] = s.n;
    }
    if (e->set[SET_PRIORS].n) {
        p.prior_k = e->prior_k;
        p.prior_pose = e->d_prior_pose; p.prior_tab = e->d_prior_tab; p.prior_bad = e->d_prior_bad;
        p.prior_gate = e->prior_gate; p.prior_chi2 = e->prior_chi2;
    }
    if (e->set[SET_DEPTH].n) p.depth = e->d_depth;
    else if (e->set[SET_RIG_DEPTH].n) p.depth = e->d_rig_depth;   // (a rig pass: any other refused above)
    p.kind = kind;
    p.n = n;
    p.coords = coords; p.pix = pix; p.pix_shared = pix_shared; p.gt = gt;
    p.frame0 = frame0;
    p.stages = e->stages;
    p.seed = e->cfg.seed;
    e->pass = p;
    return DSAC_OK;
}

// What a consumer of the held pass needs.  kinds: a pass of the soft-argmax pipeline, the DSAC one, or either, or a rig
// pass, over the same n frames; or PASS_GUIDED, a guided pass over n frames.  settings (1 << SET_*): those whose change
// since the pass makes it stale for the consumer.
enum { PASS_SOFTAM = 1, PASS_DSAC = 2, PASS_EITHER = 3, PASS_GUIDED = 4, PASS_RIG = 8 };
constexpr unsigned SETTINGS_GEOMETRY = 1u << SET_CAMS | 1u << SET_DEPTH | 1u << SET_PRIORS;
constexpr unsigned SETTINGS_SAMPLING = 1u << SET_LOGITS | 1u << SET_DEPTH | 1u << SET_PRIORS;

static int pass_check(dsac_engine* e, const char* who, int32_t n, unsigned kinds, unsigned settings) {
    const Pass& p = e->pass;
    auto unchanged = [&]() {
        for (int i = 0; i < SET_COUNT; i++) {
            if (!(settings >> i & 1u) || p.gen[i] == e->set[i].gen) continue;
            if (kinds == PASS_GUIDED) return fail(e, DSAC_ERR_ARG, "%s: the %s changed after the last pass", who, k_setting[i].changed);
            return fail(e, DSAC_ERR_ARG, "%s: the %s changed (%s) after the forward pass", who, k_setting[i].changed, k_setting[i].setter);
        }
        return (int)DSAC_OK;
    };
    if (kinds == PASS_GUIDED) {
        const int g_n = p.set_n[SET_LOGITS];
        if (!g_n) return fail(e, DSAC_ERR_ARG, "%s: the last forward pass was not guided", who);
        if (n != g_n) return fail(e, DSAC_ERR_ARG, "%s: n %d differs from the %d frames of the last pass", who, n, g_n);
        return unchanged();
    }
    // the consumers of either pipeline's poses report a stale setting before a missing pass, the backward passes after it
    if (kinds == PASS_EITHER)
        if (int rc = unchanged()) return rc;
    const unsigned held = p.kind == DSAC_PASS_SOFTAM ? PASS_SOFTAM : p.kind == DSAC_PASS_DSAC ? PASS_DSAC
                        : p.kind == DSAC_PASS_RIG ? PASS_RIG : 0;
    if (n < 1 || p.n != n || !(held & kinds))
        return fail(e, DSAC_ERR_ARG, "%s must follow %s over the same %d frames", who,
                    kinds == PASS_SOFTAM ? "a dsac_forward" : kinds == PASS_DSAC ? "a dsac_forward_dsac"
                    : kinds == PASS_RIG ? "a dsac_forward_rig_device" : "a forward pass", n);
    return kinds == PASS_EITHER ? DSAC_OK : unchanged();
}

// The per-frame camera table and the eye coordinates of the held pass (null: the config's camera, an RGB pass).
static const Cam* pass_cams(const dsac_engine* e) { return e->pass.set_n[SET_CAMS] ? e->d_cams.get() : nullptr; }
static const double* pass_eye(const dsac_engine* e) { return e->pass.rgbd() ? e->d_eye.get() : nullptr; }

// The part of RefineParams every refinement shares: the inputs, the permutations, the camera and the thresholds.
static RefineParams refine_params(const dsac_engine* e, const int16_t* coords, const int32_t* pix, int32_t pix_shared, const Cam* cams) {
    const dsac_config& c = e->cfg;
    RefineParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.coords = coords; rp.pix = pix; rp.pix_stride = pix_shared ? 0 : DSAC_N * 2;
    rp.perm = e->d_perm;
    rp.f = c.focal; rp.cx = c.cx; rp.cy = c.cy; rp.cams = cams;
    rp.thr = c.thr2d; rp.inlier_count = c.inlier_count; rp.ref_steps = c.ref_steps;
    return rp;
}
// ... over the inputs of the held pass
static RefineParams pass_refine_params(const dsac_engine* e) {
    return refine_params(e, e->pass.coords, e->pass.pix, e->pass.pix_shared, pass_cams(e));
}
// The part of UncParams the pose queries share, over the inputs of the held pass.
static UncParams pass_unc_params(const dsac_engine* e) {
    const dsac_config& c = e->cfg;
    UncParams up;
    memset(&up, 0, sizeof(up));
    up.coords = e->pass.coords; up.pix = e->pass.pix; up.pix_stride = e->pass.pix_shared ? 0 : DSAC_N * 2;
    up.f = c.focal; up.cx = c.cx; up.cy = c.cy; up.cams = pass_cams(e); up.eye = pass_eye(e);
    up.thr = (float)c.thr2d;
    return up;
}

int dsac_set_sampling_logits_device(dsac_engine* e, int32_t n, const float* d_logits, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_set_sampling_logits_device: a submitted pass has not been awaited (dsac_forward_wait)");
    Setting& s = e->set[SET_LOGITS];
    if (!d_logits) {
        setting_clear(s);
        return DSAC_OK;
    }
    if (n < 1 || n > e->cfg.max_frames)
        return fail(e, DSAC_ERR_ARG, "dsac_set_sampling_logits_device: n %d out of range [1,%d]", n, e->cfg.max_frames);
    if (!e->k1_mode) return fail(e, DSAC_ERR_ARG, "guided sampling needs the split sampler (DSAC_K1_MODE unset)");
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaSetDevice(e->cfg.device));
    const size_t cells = (size_t)e->cfg.max_frames * DSAC_N;
    CU(e->d_g_w.reserve(cells * sizeof(double)));
    CU(e->d_g_q.reserve(cells * sizeof(uint32_t)));
    CU(e->d_g_cum.reserve(cells * sizeof(uint32_t)));
    CU(e->d_g_bad.reserve((size_t)e->cfg.max_frames * sizeof(uint32_t)));
    if (int rc = setting_begin(e, s, stream)) return rc;
    k_guided_table<<<(unsigned)n, KG_THREADS, 0, stream>>>(d_logits, e->d_g_w, e->d_g_q, e->d_g_cum, e->d_g_bad);
    e->launches++;
    CU(cudaGetLastError());
    return setting_commit(e, s, n, stream);
}

int dsac_sampling_table_device(dsac_engine* e, int32_t n, uint32_t* d_q) {
    if (!e || !d_q) return DSAC_ERR_ARG;
    const Setting& s = e->set[SET_LOGITS];
    if (!s.n) return fail(e, DSAC_ERR_ARG, "dsac_sampling_table_device: no sampling logits are set");
    if (n != s.n) return fail(e, DSAC_ERR_ARG, "dsac_sampling_table_device: n %d differs from the %d frames of the setting", n, s.n);
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaEventSynchronize(s.ev));
    CU(cudaMemcpy(d_q, e->d_g_q, (size_t)n * DSAC_N * sizeof(uint32_t), cudaMemcpyDeviceToDevice));
    return DSAC_OK;
}

// dsac_sampling_log_prob_device / _backward_device: the last pass must have been guided by the setting still in force.
static int sampling_log_prob_run(dsac_engine* e, const char* who, int32_t n, double* d_logp, const double* d_grad_logp, float* d_grad,
                                 void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "%s: a submitted pass has not been awaited (dsac_forward_wait)", who);
    // (the rig settings: a rig pass's consumers only)
    const unsigned rig_settings = e->pass.kind == DSAC_PASS_RIG ? 1u << SET_RIG_PRIORS | 1u << SET_RIG_DEPTH : 0u;
    if (int rc = pass_check(e, who, n, PASS_GUIDED, SETTINGS_SAMPLING | rig_settings)) return rc;
    if ((!d_logp && !d_grad_logp) || (d_grad_logp && !d_grad)) return fail(e, DSAC_ERR_ARG, "%s: null output", who);
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaStreamWaitEvent(stream, e->ev_fwd, 0));
    GuidedLogpParams g;
    g.w = e->d_g_w; g.cum = e->d_g_cum; g.bad = e->d_g_bad; g.stream_ncand = e->d_stream_ncand;
    g.T = e->cfg.n_streams; g.seed = e->pass.seed; g.frame0 = e->pass.frame0;
    g.logp = d_logp; g.grad_logp = d_grad_logp; g.grad_logits = d_grad;
    k_guided_logp<<<(unsigned)n, KG_THREADS, 0, stream>>>(g);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_sampling_log_prob_device(dsac_engine* e, int32_t n, double* d_logp, void* stream) {
    if (!d_logp) return e ? fail(e, DSAC_ERR_ARG, "dsac_sampling_log_prob_device: null output") : DSAC_ERR_ARG;
    return sampling_log_prob_run(e, "dsac_sampling_log_prob_device", n, d_logp, nullptr, nullptr, stream);
}

int dsac_sampling_log_prob_backward_device(dsac_engine* e, int32_t n, const double* d_grad_logp, float* d_grad_logits, void* stream) {
    if (!d_grad_logp || !d_grad_logits) return e ? fail(e, DSAC_ERR_ARG, "dsac_sampling_log_prob_backward_device: null argument") : DSAC_ERR_ARG;
    return sampling_log_prob_run(e, "dsac_sampling_log_prob_backward_device", n, nullptr, d_grad_logp, d_grad_logits, stream);
}

// The update both cell depth settings share: the copy of n frames of depth into `buf` (sized once for max_frames), and the
// eye coordinates and skip bits of the passes that read it.
static int depth_update(dsac_engine* e, Setting& s, DevMem<float>& buf, int32_t n, const float* d_depth, cudaStream_t stream) {
    CU(cudaSetDevice(e->cfg.device));
    const size_t cells = (size_t)e->cfg.max_frames * DSAC_N;
    CU(buf.reserve(cells * sizeof(float)));
    CU(e->d_eye.reserve(cells * 3 * sizeof(double)));
    CU(e->d_rgbd_skip.reserve((size_t)e->cfg.max_frames * sizeof(uint32_t)));
    if (int rc = setting_begin(e, s, stream)) return rc;
    CU(cudaMemcpyAsync(buf.get(), d_depth, (size_t)n * DSAC_N * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return setting_commit(e, s, n, stream);
}

int dsac_set_cell_depth_device(dsac_engine* e, int32_t n, const float* d_depth, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_set_cell_depth_device: a submitted pass has not been awaited (dsac_forward_wait)");
    Setting& s = e->set[SET_DEPTH];
    if (!d_depth) {
        setting_clear(s);
        return DSAC_OK;
    }
    if (n < 1 || n > e->cfg.max_frames)
        return fail(e, DSAC_ERR_ARG, "dsac_set_cell_depth_device: n %d out of range [1,%d]", n, e->cfg.max_frames);
    return depth_update(e, s, e->d_depth, n, d_depth, (cudaStream_t)stream_v);
}

int dsac_set_pose_priors_device(dsac_engine* e, int32_t n, int32_t k, const double* d_poses, const double* d_info, double gate,
                                void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    static const char* who = "dsac_set_pose_priors_device";
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "%s: a submitted pass has not been awaited (dsac_forward_wait)", who);
    Setting& s = e->set[SET_PRIORS];
    if (!d_poses) {
        setting_clear(s);
        return DSAC_OK;
    }
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_ARG, "%s: n %d out of range [1,%d]", who, n, e->cfg.max_frames);
    const int k_max = std::min(e->cfg.n_hyps, DSAC_MAX_PRIORS);
    if (k < 1 || k > k_max) return fail(e, DSAC_ERR_ARG, "%s: k %d out of range [1,%d]", who, k, k_max);
    if (d_info && !(std::isfinite(gate) && gate > 0)) return fail(e, DSAC_ERR_ARG, "%s: gate %g must be finite and > 0", who, gate);
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaSetDevice(e->cfg.device));
    const size_t slots = (size_t)e->cfg.max_frames * DSAC_MAX_PRIORS;
    CU(e->d_prior_pose.reserve(slots * 6 * sizeof(double)));
    CU(e->d_prior_info.reserve(slots * 36 * sizeof(double)));
    CU(e->d_prior_tab.reserve(slots * sizeof(PriorGate)));
    CU(e->d_prior_bad.reserve((size_t)e->cfg.max_frames * sizeof(uint32_t)));
    if (int rc = setting_begin(e, s, stream)) return rc;
    const size_t nk = (size_t)n * k;
    CU(cudaMemcpyAsync(e->d_prior_pose.get(), d_poses, nk * 6 * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    if (d_info) CU(cudaMemcpyAsync(e->d_prior_info.get(), d_info, nk * 36 * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    k_prior_prep<<<(unsigned)n, 32, 0, stream>>>(e->d_prior_pose, d_info ? e->d_prior_info.get() : nullptr, k, e->d_prior_tab, e->d_prior_bad);
    e->launches++;
    CU(cudaGetLastError());
    if (int rc = setting_commit(e, s, n, stream)) return rc;
    e->prior_k = k;
    e->prior_gate = d_info != nullptr;
    e->prior_chi2 = d_info ? gate : 0.0;
    return DSAC_OK;
}

int64_t dsac_launch_count(const dsac_engine* e) { return e ? e->launches : 0; }

int dsac_sampler_profile(dsac_engine* e, int32_t enable) {
    if (!e) return DSAC_ERR_ARG;
    if (!e->k1_mode) return fail(e, DSAC_ERR_ARG, "dsac_sampler_profile needs the split sampler (DSAC_K1_MODE unset)");
    CU(cudaSetDevice(e->cfg.device));
    if (enable) CU(e->d_k1_dbg.reserve(K1S_MAX_ROUNDS * 4 * sizeof(unsigned long long)));
    e->k1_profile = enable ? 1 : 0;
    return DSAC_OK;
}

int dsac_debug_spec_result(dsac_engine* e, int32_t out8[8]) {
    if (!e || !out8) return DSAC_ERR_ARG;
    for (int i = 0; i < 8; i++) out8[i] = 0;
    if (!e->d_k1_spec_result || e->k1_spec_slots <= 0) return DSAC_OK;
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(out8, e->d_k1_spec_result, std::min(8, e->k1_spec_slots) * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return DSAC_OK;
}

int dsac_sampler_profile_read(dsac_engine* e, double ms[4], uint64_t counts[4]) {
    if (!e || !ms || !counts) return DSAC_ERR_ARG;
    if (!e->k1_profile || e->k1_ev_n < 2) return fail(e, DSAC_ERR_ARG, "dsac_sampler_profile_read: no profiled forward pass");
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaEventSynchronize(e->k1_ev[e->k1_ev_n - 1]));
    for (int k = 0; k < 4; k++) { ms[k] = 0; counts[k] = 0; }
    for (int i = 1; i < e->k1_ev_n; i++) {
        float t = 0;
        CU(cudaEventElapsedTime(&t, e->k1_ev[i - 1], e->k1_ev[i]));
        const int kind = e->k1_ev_kind[i];
        if (kind >= 0 && kind < 4) ms[kind] += t;
    }
    unsigned long long h[K1S_MAX_ROUNDS * 4];
    CU(cudaMemcpy(h, e->d_k1_dbg, sizeof(h), cudaMemcpyDeviceToHost));
    for (int r = 0; r < K1S_MAX_ROUNDS; r++) {
        counts[0] += h[r * 4 + 1]; counts[1] += h[r * 4 + 2]; counts[2] += h[r * 4 + 3];
        if (h[r * 4 + 0]) counts[3] = (uint64_t)(r + 1);
    }
    return DSAC_OK;
}

int dsac_set_score_hook(dsac_engine* e, dsac_score_hook fn, void* user) {
    if (!e) return DSAC_ERR_ARG;
    if (fn && !e->cfg.write_diffmaps) return fail(e, DSAC_ERR_ARG, "a score hook needs write_diffmaps=1");
    e->hook = fn;
    e->hook_user = user;
    return DSAC_OK;
}

int dsac_set_score_backward_hook(dsac_engine* e, dsac_score_backward_hook fn, void* user) {
    if (!e) return DSAC_ERR_ARG;
    e->bw_hook = fn;
    e->bw_hook_user = user;
    return DSAC_OK;
}

// The rig passes' twin of the score seam: both hooks or neither; a rig pass reads them, every other forward refuses while
// they are registered (pass_begin), and the rig backward needs the pair its pass called.
int dsac_set_rig_score_hooks(dsac_engine* e, dsac_score_hook fn, dsac_score_backward_hook bw_fn, void* user) {
    static const char* who = "dsac_set_rig_score_hooks";
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "%s: a submitted pass has not been awaited (dsac_forward_wait)", who);
    if (!fn != !bw_fn)
        return fail(e, DSAC_ERR_ARG, "%s: the forward and the backward hook are set together (both NULL clears them), %s is NULL", who,
                    fn ? "the backward hook" : "the forward hook");
    e->rig_hook = fn;
    e->rig_bw_hook = bw_fn;
    e->rig_hook_user = fn ? user : nullptr;
    return DSAC_OK;
}

// Score seam in the backward pass: with hooks registered, dScore/dDiffMap comes from the backward hook (fills e->d_ext_g);
// returns the pointer k_dscore shall read (null: closed-form soft-inlier derivative).
static int seam_backward(dsac_engine* e, int n, const double* d_sog, cudaStream_t stream, const double** ext_g) {
    *ext_g = nullptr;
    if (!e->hook && !e->bw_hook) return DSAC_OK;
    if (!e->hook || !e->bw_hook)
        return fail(e, DSAC_ERR_ARG, "the score seam needs both hooks: %s is registered but %s is not (dsac_set_score_hook / dsac_set_score_backward_hook)",
                    e->hook ? "the forward hook" : "the backward hook", e->hook ? "the backward hook" : "the forward hook");
    if (!e->d_diffmaps) return fail(e, DSAC_ERR_ARG, "the score seam needs write_diffmaps=1");
    const size_t H = e->cfg.n_hyps, count = (size_t)n * H * DSAC_N;
    CU(e->d_ext_g.reserve((count + (size_t)n * H) * sizeof(double)));
    double* clamped = e->d_ext_g + count;   // [n][H] behind the gradient block
    k_clamp_copy<<<(unsigned)(((size_t)n * H + 255) / 256), 256, 0, stream>>>(d_sog, clamped, (size_t)n * H, e->cfg.grad_clamp);
    e->launches++;
    CU(cudaGetLastError());
    int rc = e->bw_hook(e->d_diffmaps, clamped, n, (int32_t)H, e->d_ext_g, (void*)stream, e->bw_hook_user);
    if (rc != 0) return fail(e, DSAC_ERR_ARG, "score backward hook returned %d", rc);
    *ext_g = e->d_ext_g;
    return DSAC_OK;
}

static int pick_tile(const dsac_engine* e, int n_frames, int H) {
    int t = e->cfg.hyps_per_cta;
    if (t <= 0) {
        // enough CTAs to fill the chip a few times over, but no smaller than 8 hypotheses
        t = 64;
        while (t > 8 && (long long)n_frames * ((H + t - 1) / t) < 4ll * e->sm_count) t >>= 1;
    }
    t = std::max(8, std::min(t, K2_MAX_TILE));
    t = (t + 7) & ~7;
    return t;
}

// Launches the forward stages `stages` (DSAC_STAGE_*) for `n` frames whose per-frame engine buffers start at frame offset
// `off` (inputs are passed already offset).  Used whole (off = 0) and per chunk by the pipelined host path.
static int forward_range(dsac_engine* e, int32_t off, int32_t n, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                         int32_t pix_shared, const double* d_gt_jp, void* stream_v, uint32_t stages, int lane = 0) {
    cudaStream_t stream = (cudaStream_t)stream_v;
    const dsac_config& c = e->cfg;
    const size_t o = (size_t)off, Hh = (size_t)c.n_hyps, Nn = DSAC_N;
    // the variant flags of the pass, which index the kernel tables
    const int cam = e->pass.set_n[SET_CAMS] > 0, guided = e->pass.set_n[SET_LOGITS] > 0, rgbd = e->pass.rgbd();
    const Cam* cams = cam ? e->d_cams + o : nullptr;          // per-frame cameras: those of this range's frames
    const GuidedGen gg{guided ? e->d_g_cum + o * DSAC_N : nullptr, guided ? e->d_g_bad + o : nullptr};
    const double* eye = rgbd ? e->d_eye + o * Nn * 3 : nullptr;   // RGB-D pass: this range's frames of the eye coordinates
    // pose priors: the streams draw n_hyps - prior_k hypotheses into the first slots of each frame, k_prior_inject fills the rest
    const Pass& ps = e->pass;
    const int prior_k = ps.prior_k;
    const int gate = prior_k > 0 && ps.prior_gate;
    const int draw_h = c.n_hyps - prior_k;

    if (stages & DSAC_STAGE_SAMPLE) {
        CU(cudaMemsetAsync(e->d_status + o, 0, (size_t)n * sizeof(uint32_t), stream));
        if (rgbd) {
            const int ps = pix_shared ? 0 : DSAC_N * 2;
            const Cam cam0{c.focal, c.cx, c.cy};
            const uint32_t* gbad = guided ? gg.bad : nullptr;
            k_rgbd_eye_tab[cam]<<<(unsigned)n, KE_THREADS, 0, stream>>>(e->pass.depth + o * Nn, d_pix, ps, cam0, cams, gbad, e->d_eye + o * Nn * 3, e->d_rgbd_skip + o);
            e->launches++;
        }
        SampleParams sp;
        sp.coords = d_coords; sp.pix = d_pix; sp.pix_stride = pix_shared ? 0 : DSAC_N * 2;
        sp.f = c.focal; sp.cx = c.cx; sp.cy = c.cy; sp.cams = cams;
        sp.H = draw_h; sp.Hs = c.n_hyps; sp.T = c.n_streams; sp.thr = c.thr2d;
        sp.seed = c.seed; sp.skip = c.stream_skip; sp.max_candidates = c.max_candidates;
        sp.frame0 = frame0;
        sp.hyp_pose = e->d_hyp_pose + o * Hh * 6; sp.hyp_P = e->d_hyp_P + o * Hh * 12; sp.img_idx = e->d_img_idx + o * Hh * 4; sp.cand_idx = e->d_cand_idx + o * Hh;
        sp.stream_ncand = e->d_stream_ncand + o * c.n_streams; sp.stream_endpos = e->d_stream_endpos + o * c.n_streams; sp.status = e->d_status + o; sp.n_fragile = e->d_fragile;
        sp.phase_cycles = e->d_phase;
        { const char* g = getenv("DSAC_K1_A2_GENERIC"); sp.a2_generic = (g && g[0] == '1') ? 1 : 0; }
        sp.resume = nullptr;
        sp.eye = eye; sp.skip_frame = rgbd ? e->d_rgbd_skip + o : nullptr;
        sp.prior_tab = gate ? ps.prior_tab + o * prior_k : nullptr; sp.prior_bad = gate ? ps.prior_bad + o : nullptr;
        sp.prior_k = gate ? prior_k : 0; sp.prior_chi2 = gate ? ps.prior_chi2 : 0.0;
        // the monolithic sampler: the whole pass, or the resume tail of the split sampler's rounds
        auto launch_sample = [&](const SampleParams& s) {
            k_sample_tab[cam][rgbd][gate]<<<dim3(c.n_streams, n), K1_THREADS, sizeof(K1Smem), stream>>>(s);
        };
        if (!e->k1_mode) {
            launch_sample(sp);
            e->launches++;
            CU(cudaGetLastError());
        } else {
            // round-based pipeline (sampler_split.cuh).  One pass at a time per engine: the queues are shared.
            const size_t T = (size_t)c.n_streams, cap = (size_t)e->k1_cap;
            // the lane's own streams, events, counters and statistics (lane 0: the engine's; lane 1: e->lane1)
            cudaStream_t k_side = lane ? e->lane1.side : e->k1_side, k_side2 = lane ? e->lane1.side2 : e->k1_side2;
            const Event* k_ev_filt = lane ? e->lane1.ev_filt : e->k1_ev_filt;
            const Event* k_ev_solve = lane ? e->lane1.ev_solve : e->k1_ev_solve;
            const Event* k_ev_gen = lane ? e->lane1.ev_gen : e->k1_ev_gen;
            cudaEvent_t k_ev_round = lane ? e->lane1.ev_round : e->k1_ev_round;
            int* k_counters = lane ? e->lane1.counters : e->d_k1_counters;
            const int sampler = (gate ? 2 : 0) + (guided ? 1 : 0);   // statistics block: uniform, guided, gated uniform, gated guided
            unsigned long long* k_stats = (lane ? e->lane1.stats : e->d_k1_stats) + 4 * sampler;
            unsigned long long& k_calls = (lane ? e->lane1.calls : e->k1_calls)[sampler];
            K1SplitParams q;
            q.sp = sp;
            q.state = e->d_k1_state + o * T; q.celltab = e->d_k1_celltab + o * Nn;
            q.cells = e->d_k1_cells + o * T * cap; q.endw = e->d_k1_endw + o * T * cap;
            q.accbits = e->d_k1_accbits + o * T * (cap / 32); q.pose_out = e->d_k1_pose + o * T * cap * 6;
            q.wq = e->d_k1_wq + o * T * 128; q.fq = e->d_k1_fq + o * T * cap;   // (work items / flagged candidates of this range's slots)
            q.wq_n = k_counters; q.fq_n = k_counters + K1S_MAX_SETS;
            q.wq_stride = e->k1_wq_stride;
            q.first_frac = (double)K1S_FIRST_ROUND_FRAC;
            q.spec = 0;
            const int par = (int)(k_calls & 1ull);
            k_calls++;
            q.stats_cur = k_stats + 2 * par; q.stats_prev = k_stats + 2 * (par ^ 1);
            q.dbg = e->d_k1_dbg;
            q.cap = e->k1_cap;
            const long long n_slots = (long long)n * c.n_streams;
            // a round is generated in up to 4 portions of cap / 4 candidates (round 0: 4, round 1: 2, later rounds: the whole
            // round at once); a filter work item is a chunk of a portion
            int n_port = 4;                       // portions of round 0 (round 1: half as many, twice as large)
            bool port_forced = false;
            if (const char* pp = getenv("DSAC_K1_PORTIONS")) {
                const int v = atoi(pp);
                if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) { n_port = v; port_forced = true; }
            }
            if (!port_forced && n_slots < 256) n_port = 2;   // few streams: fewer, larger portions (DSAC_K1_PORTIONS compares them)
            const int portion4 = e->k1_cap / n_port;
            int want_chunk = n_slots >= 512 ? 2048 : (n_slots >= 64 ? 512 : 256);
            if (const char* ch = getenv("DSAC_K1_CHUNK")) want_chunk = std::max(256, atoi(ch));
            q.chunk = 256;
            for (int cc : {2048, 1024, 512, 256})
                if (cc <= want_chunk && cc <= K1F_MAX_CHUNK && portion4 % cc == 0) { q.chunk = cc; break; }
            q.n_slots = (int)n_slots;
            q.round = 0; q.select_only = 0; q.gen_only = 0;
            CU(cudaMemsetAsync(k_counters, 0, 2 * K1S_MAX_SETS * sizeof(int), stream));
            CU(cudaMemsetAsync(q.stats_cur, 0, 2 * sizeof(unsigned long long), stream));
            if (q.dbg) CU(cudaMemsetAsync(q.dbg, 0, K1S_MAX_ROUNDS * 4 * sizeof(unsigned long long), stream));
            e->k1_ev_n = 0;
            auto mark = [&](int kind) {   // dsac_sampler_profile: an event after every launch
                if (!e->k1_profile) return;
                if ((size_t)e->k1_ev_n >= e->k1_ev.size()) {
                    Event ev;
                    if (cudaEventCreate(ev.put()) != cudaSuccess) return;
                    e->k1_ev.push_back(std::move(ev));
                    e->k1_ev_kind.push_back(0);
                }
                e->k1_ev_kind[e->k1_ev_n] = kind;
                cudaEventRecord(e->k1_ev[e->k1_ev_n++], stream);
            };
            // threads per (frame, stream) of the generator.  A stream's generation is a serial chain of windows; with fewer
            // streams than the SMs hold at 256 threads, larger CTAs shorten the parallel phases of a window (DSAC_K1_SLOT_THREADS
            // compares 256 / 512 / 1024).  The MT19937 regeneration itself (half of a window) does not scale: 227 words are independent.
            int slot_threads = K1S_THREADS;
            if (n_slots <= 32) slot_threads = 1024;
            else if (n_slots <= 2 * e->sm_count) slot_threads = 512;
            if (e->k1_slot_threads > 0) slot_threads = e->k1_slot_threads;
            auto launch_slot = [&](const K1SplitParams& qq) {
                const dim3 g(c.n_streams, n);
                if (rgbd && guided) k1_gslot_rgbd<<<g, K1S_THREADS, 0, stream>>>(qq, gg);
                else if (rgbd) k1_slot_rgbd<<<g, K1S_THREADS, 0, stream>>>(qq);
                else if (guided) k1_gslot<<<g, K1S_THREADS, 0, stream>>>(qq, gg);
                else if (slot_threads == 1024) k1_slot_t<1024><<<g, 1024, 0, stream>>>(qq);
                else if (slot_threads == 512) k1_slot_t<512><<<g, 512, 0, stream>>>(qq);
                else k1_slot<<<g, K1S_THREADS, 0, stream>>>(qq);
            };
            // with the profile on everything runs on one stream so that the event intervals are the kernels' own durations
            const bool fused = e->k1_fused != 0 && !cams && !guided && !rgbd;   // (k1_fused has no per-frame instantiation; the schedule does not change results)
            // streams: generator on `stream`, filter (and solve) on a side stream; with a batch that does not fill the GPU several
            // times over the solve gets a stream of its own, so that the filter of set k+1 need not wait for the solve of set k
            // (DSAC_K1_OVERLAP=1 / 2 compares them; on an H100 SXM at 700 W: 128 frames 0.856 / 0.862 ms, 1024 frames 3.09 / 3.10 ms)
            const int ov_mode = e->k1_overlap_fixed ? e->k1_overlap : (n_slots <= 768 ? 2 : 1);
            const bool overlap = ov_mode && !e->k1_profile && !fused;
            cudaStream_t side = overlap ? k_side : stream;
            cudaStream_t solve_side = (overlap && ov_mode >= 2 && !rgbd) ? k_side2 : side;   // (k1_kabsch: no solve)
            const size_t n_slots_cap = (size_t)e->cfg.max_frames * c.n_streams * (size_t)e->k1_cap;
            mark(-1);
            {
                // (guided passes read no MT19937 stream: nothing to seed)
                const int cell_blocks = (int)(((size_t)n * Nn + 255) / 256), seed_blocks = guided ? 0 : (int)((n_slots + 31) / 32);
                k1_cells_tab[cam]<<<(unsigned)(cell_blocks + seed_blocks), 256, 0, stream>>>(q, n, seed_blocks);
            }
            mark(0);
            e->launches++;
            int set = 0;
            // few streams (single-frame latency): no previous call's shortfall to make up in later rounds -- the first round
            // takes 115 % of the expected need and one top-up round follows (every round is three dependent launches);
            // the rare straggler goes to the monolithic kernel
            const bool few = n_slots < 128;
            const bool fused_req = fused;
            if (few) q.first_frac = 1.15;
            // speculative first round (k1_spec / k1_stitch): one stream generated window by window on many SMs; pays when a
            // stream's first round is several windows long (>= 64 hypotheses per stream) and the GPU is otherwise idle
            const int quota_max = (draw_h + c.n_streams - 1) / c.n_streams;
            const bool use_spec = few && off == 0 && n_slots <= e->k1_spec_slots && quota_max >= 64 && c.max_candidates >= (1 << 16) && !fused_req && !guided && !rgbd;   // (the candidate bound cannot fall inside the speculative round)
            // chained generator (k1_pipe): K CTAs per stream, all of them resident at once
            const int pipe_K = (int)std::min<long long>(8, e->k1_slot_capacity / std::max<long long>(1, n_slots));
            const bool use_pipe = e->k1_pipe && !use_spec && pipe_K >= 3 && n_slots >= 9 && quota_max >= 64 && c.max_candidates >= (1 << 16) &&
                                  !fused_req && !e->k1_profile && !guided && !rgbd;
            const int n_rounds = (few && !e->k1_rounds_fixed) ? std::min(e->k1_rounds, 2) : e->k1_rounds;
            for (int r = 0; r < n_rounds; r++) {
                // portions only pay when the generator has the whole GPU to fill (many streams); a few streams (single-frame
                // latency, BASELINE config 2) take every round in one launch set: fewer dependent launches
                const bool portioned = (n_slots >= 128 || port_forced) && r < 2 && n_port > 1 && !(use_pipe && r == 0);
                const int sets = portioned ? (r == 0 ? n_port : n_port / 2) : 1;
                q.round = r;
                q.portion = portioned ? (r == 0 ? portion4 : 2 * portion4) : e->k1_cap;   // round 1 may use the whole capacity too
                q.round_limit = q.portion * sets;
                const int fgrid = (int)std::min<long long>(e->k1_filter_grid, n_slots * ((q.portion + q.chunk - 1) / q.chunk));
                if (overlap && r > 0) CU(cudaStreamWaitEvent(stream, k_ev_round, 0));   // the selection needs the previous round's solves
                if (fused) {
                    // one stream: slot (select + first portion), then per set { filter(k) | generator(k+1) } fused, solve(k)
                    q.gen_only = 0; q.qidx = set; q.fqidx = set; q.fq = e->d_k1_fq + o * T * cap + (size_t)(set & 1) * n_slots_cap;
                    launch_slot(q);
                    mark(0);
                    e->launches++;
                    for (int k = 0; k < sets && set < K1S_MAX_SETS; k++, set++) {
                        K1SplitParams qf = q;
                        qf.gen_only = 0; qf.qidx = set; qf.fqidx = set; qf.fq = e->d_k1_fq + o * T * cap + (size_t)(set & 1) * n_slots_cap;
                        if (k + 1 < sets && set + 1 < K1S_MAX_SETS) {
                            K1SplitParams qg = q;
                            qg.gen_only = 1; qg.qidx = set + 1; qg.fqidx = set + 1;
                            k1_fused<<<e->sm_count, K1X_THREADS, sizeof(K1XSmem), stream>>>(qf, qg);
                        } else {
                            k1_filter<<<fgrid, K1F_THREADS, sizeof(K1FSmem), stream>>>(qf);
                        }
                        mark(1);
                        k1_solve_tab[0][gate][0]<<<e->k1_solve_grid, K1V_THREADS, 0, stream>>>(qf);
                        mark(2);
                        e->launches += 2;
                    }
                    continue;
                }
                const int first_set = set;
                for (int k = 0; k < sets && set < K1S_MAX_SETS; k++, set++) {
                    // solve_batch: the sets of a round append to ONE flag queue and a single k1_solve runs after the round's
                    // last filter (a solve over one set is a partial wave bound by the latency of one P3P)
                    const bool batch = e->k1_solve_batch != 0;
                    const bool solve_now = !batch || k + 1 == sets || set + 1 == K1S_MAX_SETS;
                    const int fset = batch ? first_set : set;
                    q.gen_only = (k > 0);
                    q.qidx = set;
                    q.fqidx = fset;
                    q.fq = e->d_k1_fq + o * T * cap + (size_t)(fset & 1) * (size_t)n_slots_cap;
                    if (use_spec && r == 0 && k == 0) {
                        K1SpecParams spp;
                        spp.vstate = e->d_k1_vstate; spp.vcells = e->d_k1_vcells; spp.vendw = e->d_k1_vendw; spp.result = e->d_k1_spec_result; spp.table = e->d_k1_spec_table;
                        k1_spec<<<dim3(K1P_VPER, (unsigned)n_slots), K1S_THREADS, 0, stream>>>(q, spp);
                        k1_stitch<<<(unsigned)n_slots, K1T_THREADS, 0, stream>>>(q, spp);
                        k1_gather<<<dim3((unsigned)((e->k1_cap + K1G_PER_CTA - 1) / K1G_PER_CTA), (unsigned)n_slots), K1G_THREADS, 0, stream>>>(q, spp);
                        e->launches += 2;
                    } else if (use_pipe && r == 0 && k == 0) {
                        K1PipeParams ppm;
                        ppm.chain = e->d_k1_chain + o * T * (K1Q_MAX_WIN + 1) * 4;
                        ppm.epoch = (uint32_t)(++e->k1_epoch & 0x7fffffffull) + 1u;
                        ppm.K = pipe_K;
                        k1_pipe<<<dim3((unsigned)pipe_K, (unsigned)n_slots), K1S_THREADS, 0, stream>>>(q, ppm);
                    } else {
                        launch_slot(q);
                    }
                    mark(0);
                    if (overlap) {
                        CU(cudaEventRecord(k_ev_gen[set], stream));
                        CU(cudaStreamWaitEvent(side, k_ev_gen[set], 0));
                        if (!batch && solve_side != side && set >= 2) CU(cudaStreamWaitEvent(side, k_ev_solve[set - 2], 0));   // the flag-queue region is free again
                    }
                    if (rgbd) {   // the acceptance test writes the accept bits itself: no flag queue, no solve
                        k1_kabsch_tab[cam][gate]<<<fgrid, K1F_THREADS, 0, side>>>(q);
                        if (!overlap) mark(1);
                        e->launches += 2;
                        continue;
                    }
                    k1_filter_tab[cam]<<<fgrid, K1F_THREADS, sizeof(K1FSmem), side>>>(q);
                    if (!overlap) mark(1);
                    e->launches += 2;
                    if (!solve_now) continue;
                    if (solve_side != side) {
                        CU(cudaEventRecord(k_ev_filt[set], side));
                        CU(cudaStreamWaitEvent(solve_side, k_ev_filt[set], 0));
                    }
                    const int group4 = few && e->k1_solve_group4;
                    k1_solve_tab[cam][gate][group4]<<<e->k1_solve_grid, K1V_THREADS, 0, solve_side>>>(q);
                    if (solve_side != side) CU(cudaEventRecord(k_ev_solve[set], solve_side));
                    if (!overlap) mark(2);
                    e->launches++;
                }
                if (overlap) CU(cudaEventRecord(k_ev_round, solve_side));
            }
            if (overlap) CU(cudaStreamWaitEvent(stream, k_ev_round, 0));
            q.round = n_rounds; q.select_only = 1; q.gen_only = 0;
            launch_slot(q);
            mark(0);
            sp.resume = q.state;   // streams the rounds left unfinished (normally none) continue in the monolithic kernel
            const dim3 gt(c.n_streams, n);   // ... or in guided steps
            if (guided) k1_gtail_tab[cam][rgbd][gate]<<<gt, KG_THREADS, 0, stream>>>(q, gg);
            else launch_sample(sp);
            mark(3);
            e->launches += 2;
            if (cams) {   // the generator's selection wrote hyp_P with the config's focal length
                k1_focal_rows_cam<<<(unsigned)(((size_t)n * c.n_hyps + 255) / 256), 256, 0, stream>>>(sp, n);
                e->launches++;
            }
            CU(cudaGetLastError());
        }
        if (prior_k) {   // the prior slots behind the sampled ones, or the empty frames of a bad setting
            PriorInjectParams ip;
            ip.poses = ps.prior_pose + o * prior_k * 6; ip.bad = ps.prior_bad + o;
            ip.k = prior_k; ip.H = c.n_hyps; ip.T = c.n_streams; ip.skip = c.stream_skip; ip.f = c.focal; ip.cams = cams;
            ip.hyp_pose = sp.hyp_pose; ip.hyp_P = sp.hyp_P; ip.img_idx = sp.img_idx; ip.cand_idx = sp.cand_idx;
            ip.stream_ncand = sp.stream_ncand; ip.stream_endpos = sp.stream_endpos; ip.status = sp.status;
            k_prior_inject<<<(unsigned)n, 128, 0, stream>>>(ip);
            e->launches++;
            CU(cudaGetLastError());
        }
    }
    if (stages & DSAC_STAGE_SCORE) {
        ScoreParams kp;
        kp.coords = d_coords; kp.pix = d_pix; kp.pix_stride = pix_shared ? 0 : DSAC_N * 2;
        kp.hyp_P = e->d_hyp_P + o * Hh * 12; kp.hyp_pose = e->d_hyp_pose + o * Hh * 6;
        kp.diffmaps = e->d_diffmaps ? e->d_diffmaps + o * Hh * Nn : nullptr; kp.scores = e->d_scores + o * Hh; kp.sf = e->d_sf + o * Hh; kp.entropy = e->d_entropy + o;
        kp.avg_pose = e->d_avg + o * 6; kp.frame_counter = e->d_frame_counter + o;
        kp.H = c.n_hyps;
        kp.tile = pick_tile(e, n, c.n_hyps);
        kp.tiles_per_frame = (c.n_hyps + kp.tile - 1) / kp.tile;
        kp.cxf = (float)c.cx; kp.cyf = (float)c.cy; kp.cams = cams;
        kp.thr = (float)c.thr2d;
        kp.kbeta = (float)(c.beta * 1.4426950408889634);
        kp.alpha = c.alpha;
        kp.external_scores = 0;
        dim3 grid(kp.tiles_per_frame, n);
        k_score_tab[cam][e->d_diffmaps.get() != nullptr]<<<grid, K2_THREADS, 0, stream>>>(kp);
        e->launches++;
        CU(cudaGetLastError());
        if (e->hook) {
            // score seam (lua_calls.h:284-300): external scorer on the materialised diffmaps,
            // then only the softmax / soft-argmax tail
            int rc = e->hook(kp.diffmaps, n, c.n_hyps, kp.scores, stream_v, e->hook_user);
            if (rc != 0) return fail(e, DSAC_ERR_ARG, "score hook returned %d", rc);
            kp.external_scores = 1;
            kp.tiles_per_frame = 1;
            k_score<false><<<dim3(1, n), K2_THREADS, 0, stream>>>(kp);
            e->launches++;
            CU(cudaGetLastError());
        }
    }
    if (stages & DSAC_STAGE_REFINE) {
        RefineParams rp = refine_params(e, d_coords, d_pix, pix_shared, cams);
        rp.n_jobs = n;
        rp.job_init = e->d_avg + o * 6;
        rp.out_pose = e->d_ref + o * 6;
        rp.inlier_map = e->d_inlier_map + o * Nn; rp.steps_done = e->d_steps_done + o; rp.n_perm_steps = e->d_n_perm + o;
        rp.status = e->d_status + o;
        if ((stages & DSAC_STAGE_EVAL) && d_gt_jp) {
            rp.gt_jp = d_gt_jp;
            rp.loss = e->d_loss + o; rp.rot_err = e->d_rot_err + o; rp.t_err = e->d_t_err + o; rp.correct = e->d_correct + o;
        }
        launch_refine(rp, (unsigned)n, stream, eye);
        e->launches++;
        CU(cudaGetLastError());
    }
    return DSAC_OK;
}

// forward_range over the whole batch, with the tail split: the sampler runs one CTA per (frame, stream) and
// e->k1_slots CTAs are resident at a time, so a batch is a number of whole waves plus a partial one during which
// most of every SM idles.  Frames [0, n1) (the whole waves) go to the high-priority side stream, the rest stays on
// `stream`: the block scheduler dispatches the side stream's sampler CTAs first, its scoring / refinement kernels
// then run next to the partial wave.  Fork / join with events, so for the caller everything still happens in
// stream order on `stream`.  Frames are independent (disjoint slices of every engine buffer).
static int forward_split(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                         int32_t pix_shared, const double* d_gt_jp, cudaStream_t stream, bool allow_split, uint32_t stages) {
    int32_t n1 = 0;
    // (the tail split overlaps the later stages of the whole waves with the partial wave's sampler: it needs later stages)
    if (allow_split && e->tail_split && !e->k1_mode && (stages & DSAC_STAGE_SAMPLE) && (stages & ~DSAC_STAGE_SAMPLE) && !e->hook) {
        const int per_wave = e->k1_slots / std::max(1, e->cfg.n_streams);   // frames per sampler wave
        if (per_wave >= 1 && n > per_wave && n % per_wave != 0) n1 = (n / per_wave) * per_wave;
    }
    // Two lanes (split sampler): a large batch as two concurrent half-batches, each a complete pass (sampler, H x N matrix,
    // refinement) over its frames with its own queues, counters and side streams.  The passes de-phase on the GPU -- one half's
    // generator and latency-bound refinement run beside the other half's register-filling filter -- which a single pass,
    // whose kernels depend on each other in sequence, cannot: 3.28 -> 3.09 ms per 1024 frames on an H100 SXM at 700 W, with
    // the 50/50 split (40/60: 3.13 / 3.21 ms); tools/lane_probe.py compares more lanes.  Frames are independent and sampler streams keyed by the global frame index, so
    // results do not depend on the split.
    if (allow_split && e->k1_mode && e->k1_lanes && n >= 768 && e->lane1.main && !e->k1_profile && !e->d_k1_dbg && !e->k1_fused &&
        !e->hook && (stages & DSAC_STAGE_SAMPLE)) {
        int32_t na = n / 2;
        if (const char* lf = getenv("DSAC_K1_LANE_FRAC")) na = std::max(1, std::min(n - 1, (int32_t)(atof(lf) * n)));   // development aid
        const size_t N = DSAC_N, f = (size_t)na;
        CU(cudaEventRecord(e->ev_fork, stream));
        CU(cudaStreamWaitEvent(e->lane1.main, e->ev_fork, 0));
        int rc = forward_range(e, na, n - na, frame0 + na, d_coords + f * N * 3, pix_shared ? d_pix : d_pix + f * N * 2, pix_shared,
                               d_gt_jp ? d_gt_jp + f * 12 : nullptr, e->lane1.main, stages, 1);
        cudaEventRecord(e->ev_join, e->lane1.main);   // the caller's stream joins the lane again whatever happens below
        if (rc == DSAC_OK) rc = forward_range(e, 0, na, frame0, d_coords, d_pix, pix_shared, d_gt_jp, stream, stages, 0);
        CU(cudaStreamWaitEvent(stream, e->ev_join, 0));
        return rc;
    }
    if (n1 <= 0) return forward_range(e, 0, n, frame0, d_coords, d_pix, pix_shared, d_gt_jp, stream, stages);
    const size_t N = DSAC_N, f = (size_t)n1;
    CU(cudaEventRecord(e->ev_fork, stream));
    CU(cudaStreamWaitEvent(e->hi, e->ev_fork, 0));
    int rc = forward_range(e, 0, n1, frame0, d_coords, d_pix, pix_shared, d_gt_jp, e->hi, stages);
    // whatever happens below, the caller's stream joins the side stream again: nothing may still be writing engine
    // buffers on e->hi when the caller sees this call's work as complete (or its error)
    cudaEventRecord(e->ev_join, e->hi);
    if (rc == DSAC_OK)
        rc = forward_range(e, n1, n - n1, frame0 + n1, d_coords + f * N * 3, pix_shared ? d_pix : d_pix + f * N * 2, pix_shared,
                           d_gt_jp ? d_gt_jp + f * 12 : nullptr, stream, stages);
    CU(cudaStreamWaitEvent(stream, e->ev_join, 0));
    return rc;
}

int dsac_forward_device(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                        int32_t pix_shared, const double* d_gt_jp, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_CAPACITY, "n_frames %d exceeds engine capacity %d", n, e->cfg.max_frames);
    if (!d_coords || !d_pix) return fail(e, DSAC_ERR_ARG, "null input");
    CU(cudaSetDevice(e->cfg.device));
    if (int rc = pass_begin(e, DSAC_PASS_SOFTAM, n, frame0, d_coords, d_pix, pix_shared, d_gt_jp, {(cudaStream_t)stream_v})) return rc;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_forward_device: a submitted pass has not been awaited (dsac_forward_wait)");
    int rc = forward_split(e, n, frame0, d_coords, d_pix, pix_shared, d_gt_jp, (cudaStream_t)stream_v, true, e->stages);
    if (rc != DSAC_OK) return rc;
    CU(cudaEventRecord(e->ev_fwd, (cudaStream_t)stream_v));   // dsac_backward (engine stream) waits on this
    return DSAC_OK;
}

// Queues the copies of frames [off, off+n) into the caller's buffers (no synchronisation).  cudaMemcpyDefault: a
// destination may be host or device memory; n_candidates goes through the pinned per-stream counts (summed on the host).
static int fetch_range(dsac_engine* e, int32_t off, int32_t n, dsac_forward_out* o, cudaStream_t stream) {
    const size_t H = e->cfg.n_hyps, N = DSAC_N, T = e->cfg.n_streams, nn = (size_t)n, f = (size_t)off;
#define D2H(dst, src, per)                                                                                          \
    do {                                                                                                            \
        if ((dst) && (src))                                                                                         \
            CU(cudaMemcpyAsync((dst) + f * (per), (src) + f * (per), nn * (per) * sizeof(*(dst)), cudaMemcpyDefault, stream)); \
    } while (0)
    D2H(o->hyp_pose, e->d_hyp_pose, H * 6);
    D2H(o->img_idx, e->d_img_idx, H * 4);
    D2H(o->cand_idx, e->d_cand_idx, H);
    D2H(o->scores, e->d_scores, H);
    D2H(o->sf, e->d_sf, H);
    if (o->diffmaps) {
        if (!e->d_diffmaps) return fail(e, DSAC_ERR_ARG, "diffmaps requested but the engine was created with write_diffmaps=0");
        D2H(o->diffmaps, e->d_diffmaps, H * N);
    }
    D2H(o->entropy, e->d_entropy, 1);
    D2H(o->avg_pose, e->d_avg, 6);
    D2H(o->ref_pose, e->d_ref, 6);
    D2H(o->inlier_map, e->d_inlier_map, N);
    D2H(o->ref_steps_done, e->d_steps_done, 1);
    D2H(o->n_perm_steps, e->d_n_perm, 1);
    D2H(o->loss, e->d_loss, 1);
    D2H(o->rot_err, e->d_rot_err, 1);
    D2H(o->t_err, e->d_t_err, 1);
    D2H(o->correct, e->d_correct, 1);
    D2H(o->status, e->d_status, 1);
    if (o->n_candidates) {
        long long* hdst = e->h_stream_ncand;
        D2H(hdst, e->d_stream_ncand, T);
    }
#undef D2H
    return DSAC_OK;
}

static void sum_candidates(dsac_engine* e, int32_t n, dsac_forward_out* o) {
    const size_t T = e->cfg.n_streams;
    if (!o->n_candidates) return;
    for (size_t f = 0; f < (size_t)n; f++) {
        long long s = 0;
        for (size_t t = 0; t < T; t++) s += e->h_stream_ncand[f * T + t];
        o->n_candidates[f] = s;
    }
}

int dsac_fetch(dsac_engine* e, int32_t n, dsac_forward_out* o, void* stream_v) {
    if (!e || !o) return DSAC_ERR_ARG;
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_CAPACITY, "n_frames %d exceeds engine capacity %d", n, e->cfg.max_frames);
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaSetDevice(e->cfg.device));
    int rc = fetch_range(e, 0, n, o, stream);
    if (rc != DSAC_OK) return rc;
    CU(cudaStreamSynchronize(stream));
    sum_candidates(e, n, o);
    return DSAC_OK;
}

int dsac_device_view_get(dsac_engine* e, dsac_device_view* v) {
    if (!e || !v) return DSAC_ERR_ARG;
    v->diffmaps = e->d_diffmaps;
    v->hyp_pose = e->d_hyp_pose;
    v->scores = e->d_scores;
    v->sf = e->d_sf;
    v->avg_pose = e->d_avg;
    v->ref_pose = e->d_ref;
    v->img_idx = e->d_img_idx;
    return DSAC_OK;
}

static int forward_submit_impl(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* coords, const int32_t* pix,
                               int32_t pix_shared, const double* gt_jp, dsac_forward_out* out, bool blocking) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_forward_submit: the previous submitted pass has not been awaited");
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_CAPACITY, "n_frames %d exceeds engine capacity %d", n, e->cfg.max_frames);
    if (!coords || !pix) return fail(e, DSAC_ERR_ARG, "null input");
    CU(cudaSetDevice(e->cfg.device));
    if (int rc = pass_begin(e, DSAC_PASS_SOFTAM, n, frame0, e->d_coords, e->d_pix, pix_shared, gt_jp ? e->d_gt.get() : nullptr,
                            {e->pipe[0], e->pipe[1], e->pipe[2], e->pipe[3]}))   // (every chunk's stream: DSAC_PIPE_CHUNKS)
        return rc;
    const size_t N = DSAC_N;
    // Frames are independent, so the batch is cut into up to 4 chunks, each on its own stream:
    // H2D(chunk) -> K1 -> K2 -> K4 -> D2H(chunk).  Copies of later chunks overlap the kernels of earlier
    // ones and the tail of one chunk's kernels is filled by the next chunk's CTAs.
    static const bool trace = getenv("DSAC_TRACE") != nullptr;
    Event tev[4];
    const auto t_host0 = std::chrono::steady_clock::now();
    if (trace) for (int k = 0; k < 4; k++) cudaEventCreate(tev[k].put());
    int chunks = 1;   // the sampler kernel wants the whole batch (tools/e2e_probe.py compares chunks)
    if (const char* ev = getenv("DSAC_PIPE_CHUNKS")) chunks = std::max(1, std::min(4, atoi(ev)));
    if (pix_shared) CU(cudaMemcpyAsync(e->d_pix, pix, N * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, e->pipe[0]));
    if (pix_shared && chunks > 1) {   // every chunk reads the shared grid: make it visible to all streams first
        CU(cudaStreamSynchronize(e->pipe[0]));
    }
    // chunk boundaries at whole waves of the sampler (one CTA per frame and stream, e->k1_slots CTAs resident per GPU),
    // so that a later chunk's CTAs fill the slots an earlier chunk frees instead of adding a partial wave
    int bound[5] = {0, n, n, n, n};
    if (chunks > 1) {
        const int per_wave = std::max(1, e->k1_slots / std::max(1, e->cfg.n_streams));
        const int waves = (n + per_wave - 1) / per_wave;
        for (int c = 1; c < chunks; c++) bound[c] = std::min(n, std::max(1, (int)((long long)waves * c / chunks)) * per_wave);
        bound[chunks] = n;
    }
    for (int c = 0; c < chunks; c++) {
        const int lo = bound[c], hi = bound[c + 1], m = hi - lo;
        if (m <= 0) continue;
        cudaStream_t st = e->pipe[c];
        const size_t f = (size_t)lo;
        if (trace) cudaEventRecord(tev[0], st);
        CU(cudaMemcpyAsync(e->d_coords + f * N * 3, coords + f * N * 3, (size_t)m * N * 3 * sizeof(int16_t), cudaMemcpyHostToDevice, st));
        if (!pix_shared)
            CU(cudaMemcpyAsync(e->d_pix + f * N * 2, pix + f * N * 2, (size_t)m * N * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        if (gt_jp) CU(cudaMemcpyAsync(e->d_gt + f * 12, gt_jp + f * 12, (size_t)m * 12 * sizeof(double), cudaMemcpyHostToDevice, st));
        if (trace) cudaEventRecord(tev[1], st);
        // one chunk: the tail split applies (mode 1: blocking calls only -- with several passes in flight the other
        // pass already fills the partial wave and a high-priority stream would only delay it; mode 2: always)
        int rc = (chunks == 1)
                     ? forward_split(e, m, frame0, e->d_coords, e->d_pix, pix_shared, gt_jp ? e->d_gt.get() : nullptr, st,
                                     blocking ? e->tail_split >= 1 : e->tail_split >= 2, e->stages)
                     : forward_range(e, lo, m, frame0 + lo, e->d_coords + f * N * 3, pix_shared ? e->d_pix : e->d_pix + f * N * 2,
                                     pix_shared, gt_jp ? e->d_gt + f * 12 : nullptr, st, e->stages);
        if (rc == DSAC_OK && out) {
            if (trace) cudaEventRecord(tev[2], st);
            rc = fetch_range(e, lo, m, out, st);
        }
        if (rc != DSAC_OK) {   // copies from the caller's host buffers may already be queued: drain before reporting
            for (int k = 0; k <= c; k++) cudaStreamSynchronize(e->pipe[k]);
            return rc;
        }
        if (trace && !out) cudaEventRecord(tev[2], st);
        if (trace) cudaEventRecord(tev[3], st);
    }
    e->pending_out = out;
    e->pending_n = n;
    e->pending_chunks = chunks;
    CU(cudaEventRecord(e->ev_fwd, e->pipe[chunks - 1]));
    if (trace) {   // DSAC_TRACE=1: where one pass spends its time (last chunk's stream); forces the wait
        for (int c = 0; c < chunks; c++) CU(cudaStreamSynchronize(e->pipe[c]));
        float a = 0, b = 0, d = 0;
        cudaEventElapsedTime(&a, tev[0], tev[1]); cudaEventElapsedTime(&b, tev[1], tev[2]); cudaEventElapsedTime(&d, tev[2], tev[3]);
        const double host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count();
        fprintf(stderr, "[dsac trace] H2D %.3f ms  kernels %.3f ms  D2H %.3f ms  | call %.3f ms (host wall)\n", a, b, d, host_ms);
    }
    return DSAC_OK;
}

int dsac_forward_wait(dsac_engine* e) {
    if (!e) return DSAC_ERR_ARG;
    if (!e->pending_chunks) return DSAC_OK;
    CU(cudaSetDevice(e->cfg.device));
    const int chunks = e->pending_chunks;
    e->pending_chunks = 0;
    for (int c = 0; c < chunks; c++) CU(cudaStreamSynchronize(e->pipe[c]));
    if (e->pending_out) sum_candidates(e, e->pending_n, e->pending_out);
    e->pending_out = nullptr;
    return DSAC_OK;
}

int dsac_forward_submit(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* coords, const int32_t* pix,
                        int32_t pix_shared, const double* gt_jp, dsac_forward_out* out) {
    return forward_submit_impl(e, n, frame0, coords, pix, pix_shared, gt_jp, out, false);
}

int dsac_forward(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* coords, const int32_t* pix,
                 int32_t pix_shared, const double* gt_jp, dsac_forward_out* out) {
    int rc = forward_submit_impl(e, n, frame0, coords, pix, pix_shared, gt_jp, out, true);
    if (rc != DSAC_OK) return rc;
    return dsac_forward_wait(e);
}

// The DSAC variant's forward over device-resident inputs into the engine's buffers: sampling and scoring, refinement of
// every hypothesis from its own pose (cnn.h:1155-1218), then the draw and the expected loss (k_dsac_draw).  Nothing is
// copied to the host.  want_imaps: keep the inlier maps of every hypothesis.
static int forward_dsac_run(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                            int32_t pix_shared, const double* d_gt, int32_t random_draw, bool want_imaps, cudaStream_t stream) {
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_forward_dsac: a submitted pass has not been awaited (dsac_forward_wait)");
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_CAPACITY, "n_frames %d exceeds engine capacity %d", n, e->cfg.max_frames);
    if (!d_coords || !d_pix) return fail(e, DSAC_ERR_ARG, "null input");
    const dsac_config& c = e->cfg;
    CU(cudaSetDevice(c.device));
    // the record holds no pass until this one is complete: the soft-argmax backward does not apply to it
    if (int rc = pass_begin(e, 0, n, frame0, d_coords, d_pix, pix_shared, d_gt, {stream})) return rc;
    const size_t N = DSAC_N, nn = (size_t)n, H = c.n_hyps, jobs = nn * H;
    // refine-all buffers: they grow together, and the job -> frame table is written whenever they do
    if (jobs > e->ra_jobs) {
        e->ra_jobs = 0;
        CU(e->d_ra_frame.reserve(jobs * sizeof(int32_t)));
        CU(e->d_ra_pose.reserve(jobs * 6 * sizeof(double)));
        CU(e->d_ra_loss.reserve(jobs * sizeof(double)));
        CU(e->d_ra_rot.reserve(jobs * sizeof(double)));
        CU(e->d_ra_t.reserve(jobs * sizeof(double)));
        CU(e->d_ra_correct.reserve(jobs * sizeof(int32_t)));
        CU(e->d_ra_steps.reserve(jobs * sizeof(int32_t)));
        std::vector<int32_t> jf(jobs);
        for (size_t j = 0; j < jobs; j++) jf[j] = (int32_t)(j / H);
        CU(cudaMemcpy(e->d_ra_frame, jf.data(), jobs * sizeof(int32_t), cudaMemcpyHostToDevice));
        e->ra_jobs = jobs;
    }
    if (want_imaps) CU(e->d_ra_imap.reserve(jobs * N * sizeof(int32_t)));
    int rc = forward_range(e, 0, n, frame0, d_coords, d_pix, pix_shared, d_gt, stream, DSAC_STAGE_SAMPLE | DSAC_STAGE_SCORE);
    if (rc != DSAC_OK) return rc;
    if (!d_gt) {   // no ground truth: losses and errors are zero
        CU(cudaMemsetAsync(e->d_ra_loss, 0, jobs * sizeof(double), stream));
        CU(cudaMemsetAsync(e->d_ra_rot, 0, jobs * sizeof(double), stream));
        CU(cudaMemsetAsync(e->d_ra_t, 0, jobs * sizeof(double), stream));
        CU(cudaMemsetAsync(e->d_ra_correct, 0, jobs * sizeof(int32_t), stream));
    }
    {   // every hypothesis is a refinement job starting from its own pose (cnn.h:1155-1218)
        RefineParams rp = pass_refine_params(e);
        rp.n_jobs = (int)jobs;
        rp.job_frame = e->d_ra_frame;
        rp.job_init = e->d_hyp_pose;
        rp.out_pose = e->d_ra_pose;
        rp.steps_done = e->d_ra_steps;
        rp.inlier_map = want_imaps ? e->d_ra_imap.get() : nullptr;
        if (d_gt) {
            rp.gt_jp = d_gt;
            rp.loss = e->d_ra_loss; rp.rot_err = e->d_ra_rot; rp.t_err = e->d_ra_t; rp.correct = e->d_ra_correct;
        }
        launch_refine(rp, (unsigned)jobs, stream, pass_eye(e));
        e->launches++;
        CU(cudaGetLastError());
    }
    {
        DrawParams dp;
        dp.H = c.n_hyps; dp.T = c.n_streams; dp.random_draw = random_draw ? 1 : 0;
        dp.seed = c.seed; dp.frame0 = frame0;
        dp.sf = e->d_sf; dp.img_idx = e->d_img_idx; dp.stream_endpos = e->d_stream_endpos;
        dp.loss = e->d_ra_loss; dp.rot_err = e->d_ra_rot; dp.t_err = e->d_ra_t; dp.correct = e->d_ra_correct;
        dp.inlier_maps = want_imaps ? e->d_ra_imap.get() : nullptr;
        dp.hyp_idx = e->d_dsac_pick; dp.expected_loss = e->d_dsac_exp;
        dp.out_rot_err = e->d_dsac_rot; dp.out_t_err = e->d_dsac_terr; dp.out_correct = e->d_dsac_correct;
        k_dsac_draw<<<n, DRAW_THREADS, 0, stream>>>(dp);
        e->launches++;
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(e->ev_fwd, stream));   // the backward waits on this
    e->pass.kind = DSAC_PASS_DSAC;
    return DSAC_OK;
}

// Queues the copies of the outputs `out` asks for; destinations may be host or device memory (cudaMemcpyDefault).
static int forward_dsac_copy(dsac_engine* e, int32_t n, const dsac_dsac_out* out, cudaStream_t stream) {
    const size_t N = DSAC_N, nn = (size_t)n, H = e->cfg.n_hyps, jobs = nn * H;
#define CP(dst, src, bytes)                                                                     \
    do {                                                                                        \
        if (dst) CU(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyDefault, stream));        \
    } while (0)
    CP(out->hyp_pose, e->d_hyp_pose, jobs * 6 * sizeof(double));
    CP(out->img_idx, e->d_img_idx, jobs * 4 * sizeof(int32_t));
    CP(out->sf, e->d_sf, jobs * sizeof(double));
    CP(out->entropy, e->d_entropy, nn * sizeof(double));
    CP(out->ref_pose, e->d_ra_pose, jobs * 6 * sizeof(double));
    CP(out->losses, e->d_ra_loss, jobs * sizeof(double));
    CP(out->inlier_maps, e->d_ra_imap, jobs * N * sizeof(int32_t));
    CP(out->steps_done, e->d_ra_steps, jobs * sizeof(int32_t));
    CP(out->expected_loss, e->d_dsac_exp, nn * sizeof(double));
    CP(out->hyp_idx, e->d_dsac_pick, nn * sizeof(int32_t));
    CP(out->rot_err, e->d_dsac_rot, nn * sizeof(double));
    CP(out->t_err, e->d_dsac_terr, nn * sizeof(double));
    CP(out->correct, e->d_dsac_correct, nn * sizeof(int32_t));
    CP(out->status, e->d_status, nn * sizeof(uint32_t));
#undef CP
    return DSAC_OK;
}

int dsac_forward_dsac_device(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                             int32_t pix_shared, const double* d_gt_jp, int32_t random_draw, const dsac_dsac_out* d_out, void* stream_v) {
    if (!e || !d_out) return DSAC_ERR_ARG;
    cudaStream_t stream = (cudaStream_t)stream_v;
    int rc = forward_dsac_run(e, n, frame0, d_coords, d_pix, pix_shared, d_gt_jp, random_draw, d_out->inlier_maps != nullptr, stream);
    if (rc != DSAC_OK) return rc;
    return forward_dsac_copy(e, n, d_out, stream);
}

int dsac_forward_dsac(dsac_engine* e, int32_t n, int64_t frame0, const int16_t* coords, const int32_t* pix,
                      int32_t pix_shared, const double* gt_jp, int32_t random_draw, dsac_dsac_out* out) {
    if (!e || !out) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_forward_dsac: a submitted pass has not been awaited (dsac_forward_wait)");
    if (n < 1 || n > e->cfg.max_frames) return fail(e, DSAC_ERR_CAPACITY, "n_frames %d exceeds engine capacity %d", n, e->cfg.max_frames);
    if (!coords || !pix) return fail(e, DSAC_ERR_ARG, "null input");
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = e->pipe[0];
    const size_t N = DSAC_N, nn = (size_t)n;
    CU(cudaMemcpyAsync(e->d_coords, coords, nn * N * 3 * sizeof(int16_t), cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(e->d_pix, pix, (pix_shared ? 1 : nn) * N * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    if (gt_jp) CU(cudaMemcpyAsync(e->d_gt, gt_jp, nn * 12 * sizeof(double), cudaMemcpyHostToDevice, stream));
    int rc = forward_dsac_run(e, n, frame0, e->d_coords, e->d_pix, pix_shared, gt_jp ? e->d_gt.get() : nullptr, random_draw,
                              out->inlier_maps != nullptr, stream);
    if (rc == DSAC_OK) rc = forward_dsac_copy(e, n, out, stream);
    const cudaError_t st = cudaStreamSynchronize(stream);   // also before an error return: copies from the caller's buffers may be queued
    if (rc != DSAC_OK) return rc;
    if (st != cudaSuccess) return fail(e, DSAC_ERR_CUDA, "dsac_forward_dsac: %s", cudaGetErrorString(st));
    return DSAC_OK;
}

int dsac_backward(dsac_engine* e, int32_t n, const int16_t* coords, const int32_t* pix, int32_t pix_shared,
                  const double* gt_jp, dsac_backward_out* out) {
    if (!e || !out) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward: a submitted pass has not been awaited (dsac_forward_wait)");
    return backward_run(e, n, coords, pix, pix_shared, gt_jp, out);
}

int dsac_backward_device(dsac_engine* e, int32_t n, const double* d_loss_grad, double* d_dloss_dobj, float* d_dloss_dpred,
                         float clamp, void* stream) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward_device: a submitted pass has not been awaited (dsac_forward_wait)");
    return backward_device_run(e, n, d_loss_grad, d_dloss_dobj, d_dloss_dpred, clamp, (cudaStream_t)stream);
}

int dsac_backward_dsac(dsac_engine* e, int32_t n, dsac_backward_dsac_out* out) {
    if (!e || !out) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward_dsac: a submitted pass has not been awaited (dsac_forward_wait)");
    cudaStream_t stream = e->pipe[0];
    int rc = backward_dsac_run(e, n, nullptr, out, true, nullptr, 0.f, stream);
    const cudaError_t st = cudaStreamSynchronize(stream);
    if (rc != DSAC_OK) return rc;
    if (st != cudaSuccess) return fail(e, DSAC_ERR_CUDA, "dsac_backward_dsac: %s", cudaGetErrorString(st));
    return DSAC_OK;
}

int dsac_backward_dsac_device(dsac_engine* e, int32_t n, const double* d_loss_grad, const dsac_backward_dsac_out* d_out,
                              float* d_dloss_dpred, float clamp, void* stream) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward_dsac_device: a submitted pass has not been awaited (dsac_forward_wait)");
    const dsac_backward_dsac_out none = {};
    return backward_dsac_run(e, n, d_loss_grad, d_out ? d_out : &none, false, d_dloss_dpred, clamp, (cudaStream_t)stream);
}

int dsac_refined_jp6_device(dsac_engine* e, int32_t n, double* d_jp6, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_refined_jp6_device: a submitted pass has not been awaited (dsac_forward_wait)");
    if (!d_jp6) return fail(e, DSAC_ERR_ARG, "dsac_refined_jp6_device: null output");
    if (int rc = pass_check(e, "dsac_refined_jp6_device", n, PASS_EITHER, SETTINGS_GEOMETRY)) return rc;
    // a soft-argmax pass refines one pose per frame, the DSAC variant every hypothesis
    const bool dsac = e->pass.kind == DSAC_PASS_DSAC;
    const double* pose = dsac ? e->d_ra_pose.get() : e->d_ref.get();
    const size_t count = (size_t)n * (dsac ? e->cfg.n_hyps : 1);
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = (cudaStream_t)stream_v;
    CU(cudaStreamWaitEvent(stream, e->ev_fwd, 0));
    k_pose_jp6<<<(unsigned)((count + 127) / 128), 128, 0, stream>>>(pose, count, d_jp6);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_backward_pose_device(dsac_engine* e, int32_t n, const double* d_grad_ref, double* d_dloss_dobj, float* d_dloss_dpred,
                              float clamp, void* stream) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward_pose_device: a submitted pass has not been awaited (dsac_forward_wait)");
    if (!d_grad_ref) return fail(e, DSAC_ERR_ARG, "dsac_backward_pose_device: null d_grad_ref");
    return backward_device_run(e, n, nullptr, d_dloss_dobj, d_dloss_dpred, clamp, (cudaStream_t)stream, d_grad_ref);
}

int dsac_backward_dsac_pose_device(dsac_engine* e, int32_t n, const double* d_grad_ref, const double* d_grad_sf,
                                   const dsac_backward_dsac_out* d_out, float* d_dloss_dpred, float clamp, void* stream) {
    if (!e) return DSAC_ERR_ARG;
    if (e->pending_chunks) return fail(e, DSAC_ERR_ARG, "dsac_backward_dsac_pose_device: a submitted pass has not been awaited (dsac_forward_wait)");
    const dsac_backward_dsac_out none = {};
    return backward_dsac_run(e, n, nullptr, d_out ? d_out : &none, false, d_dloss_dpred, clamp, (cudaStream_t)stream, true,
                             d_grad_ref, d_grad_sf);
}

int dsac_gather_patches_device(dsac_engine* e, int32_t n, const uint8_t* d_frames, int32_t width, int32_t height,
                               const int32_t* d_pix, int32_t pix_shared, float mean, float* d_patches, uint32_t* d_status,
                               void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n < 1 || !d_frames || !d_pix || !d_patches) return fail(e, DSAC_ERR_ARG, "dsac_gather_patches_device: bad arguments");
    if (width < UP_PATCH || height < UP_PATCH) return fail(e, DSAC_ERR_ARG, "frame %dx%d smaller than a %d-pixel patch", width, height, UP_PATCH);
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = (cudaStream_t)stream_v;
    GatherParams p;
    p.frames = d_frames; p.width = width; p.height = height;
    p.pix = d_pix; p.pix_stride = pix_shared ? 0 : DSAC_N * 2; p.n_cells = DSAC_N;
    p.mean = mean; p.patches = d_patches; p.status = d_status;
    if (d_status) CU(cudaMemsetAsync(d_status, 0, (size_t)n * sizeof(uint32_t), stream));
    k_gather_patches<<<dim3(DSAC_N, n), UP_THREADS, 0, stream>>>(p);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_coords_from_prediction_device(dsac_engine* e, int32_t n, const float* d_prediction, int16_t* d_coords, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n < 1 || !d_prediction || !d_coords) return fail(e, DSAC_ERR_ARG, "dsac_coords_from_prediction_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    const size_t count = (size_t)n * DSAC_N * 3;
    k_coords_from_prediction<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream_v>>>(d_prediction, d_coords, count);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_kabsch(dsac_engine* e, int32_t n, int32_t m, const double* a, const double* b, double* R, double* t) {
    if (!e) return DSAC_ERR_ARG;
    return kabsch_run(e, n, m, a, b, R, t);
}

// ----------------------------------------------------------------------------- coordinate-CNN pre-training data path

int dsac_default_rgbd_camera(dsac_rgbd_camera* c) {
    if (!c) return DSAC_ERR_ARG;
    memset(c, 0, sizeof(*c));
    c->focal = 525.f;              // properties.cpp defaults, as the shipped 7-Scenes default.config also sets them
    c->secondary_focal = 585.f;
    c->raw_data = 1;
    c->width = 640;
    c->height = 480;
    for (int k = 0; k < 4; k++) c->sensor_trans[5 * k] = 1.0;   // no sensorTrans.dat: identity
    return DSAC_OK;
}

static bool obj_cam(dsac_engine* e, const dsac_rgbd_camera* c, ObjCam* o) {
    if (!c || c->width < 1 || c->height < 1) { fail(e, DSAC_ERR_ARG, "bad camera"); return false; }
    o->focal = c->focal; o->x_shift = c->x_shift; o->y_shift = c->y_shift;
    o->secondary_focal = c->secondary_focal; o->raw_x_shift = c->raw_x_shift; o->raw_y_shift = c->raw_y_shift;
    memcpy(o->sensor_trans, c->sensor_trans, sizeof(o->sensor_trans));
    o->raw_data = c->raw_data ? 1 : 0; o->width = c->width; o->height = c->height;
    return true;
}

int dsac_set_dataset_cameras(dsac_engine* e, int32_t n_frames, const dsac_rgbd_camera* cams, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (!cams) {
        e->ds_cams_n = 0;
        return DSAC_OK;
    }
    if (n_frames < 1) return fail(e, DSAC_ERR_ARG, "dsac_set_dataset_cameras: n_frames %d must be >= 1", n_frames);
    const dsac_rgbd_camera& c0 = cams[0];
    for (int32_t i = 0; i < n_frames; i++) {
        const dsac_rgbd_camera& c = cams[i];
        bool finite = std::isfinite(c.x_shift) && std::isfinite(c.y_shift) && std::isfinite(c.raw_x_shift) &&
                      std::isfinite(c.raw_y_shift);
        for (int k = 0; k < 16; k++) finite = finite && std::isfinite(c.sensor_trans[k]);
        if (!std::isfinite(c.focal) || !(c.focal > 0) || (c.raw_data && (!std::isfinite(c.secondary_focal) || !(c.secondary_focal > 0))) ||
            !finite)
            return fail(e, DSAC_ERR_ARG, "dsac_set_dataset_cameras: camera %d is invalid (focal %g, and secondary focal %g with raw_data, "
                        "must be finite and > 0; shifts and sensor_trans finite)", i, c.focal, c.secondary_focal);
        if (c.width < 1 || c.height < 1 || c.width != c0.width || c.height != c0.height || !c.raw_data != !c0.raw_data)
            return fail(e, DSAC_ERR_ARG, "dsac_set_dataset_cameras: camera %d is %dx%d with raw_data %d; every camera must be %dx%d "
                        "with raw_data %d like camera 0", i, c.width, c.height, c.raw_data, c0.width, c0.height, c0.raw_data);
    }
    cudaStream_t stream = (cudaStream_t)stream_v;
    const size_t bytes = (size_t)n_frames * sizeof(ObjCam);
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaEventSynchronize(e->ev_ds_cams));          // the previous copy has left the staging buffer
    e->ds_cams_n = 0;                                  // (a failed copy leaves no table)
    CU(e->h_ds_cams.reserve(bytes));
    memcpy(e->h_ds_cams.get(), cams, bytes);
    for (int32_t i = 0; i < n_frames; i++) e->h_ds_cams.get()[i].raw_data = cams[i].raw_data ? 1 : 0;
    CU(cudaStreamWaitEvent(stream, e->ev_ds_use, 0));  // the last reader of the old table is done with it
    CU(e->d_ds_cams.reserve(bytes));
    CU(cudaMemcpyAsync(e->d_ds_cams.get(), e->h_ds_cams.get(), bytes, cudaMemcpyHostToDevice, stream));
    CU(cudaEventRecord(e->ev_ds_cams, stream));
    e->ds_cam0 = e->h_ds_cams.get()[0];
    e->ds_cams_n = n_frames;
    return DSAC_OK;
}

// The check of an entry point called with cam == NULL, which means the per-dataset table: a table is set and covers the
// call's n frames.
static int dataset_cameras_check(dsac_engine* e, const char* who, int32_t n) {
    if (!e->ds_cams_n) return fail(e, DSAC_ERR_ARG, "%s: cam is NULL and no dataset cameras are set (dsac_set_dataset_cameras)", who);
    if (n != e->ds_cams_n)
        return fail(e, DSAC_ERR_ARG, "%s: %d frames, but the dataset cameras cover %d", who, n, e->ds_cams_n);
    return DSAC_OK;
}
// Around the launches that read the table: `stream` waits for the table's copy, and the next copy waits for them.
static int dataset_cameras_wait(dsac_engine* e, cudaStream_t stream) {
    CU(cudaStreamWaitEvent(stream, e->ev_ds_cams, 0));
    return DSAC_OK;
}
static int dataset_cameras_done(dsac_engine* e, cudaStream_t stream) {
    CU(cudaEventRecord(e->ev_ds_use, stream));
    return DSAC_OK;
}

static inline unsigned grid_of(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

__global__ void k_dropped_status(int n, const int32_t* dropped, uint32_t* status) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) status[f] = dropped[f] ? DSAC_ST_DEPTH_DROPPED : 0u;
}

int dsac_register_depth_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n, const uint16_t* d_raw,
                               uint16_t* d_depth, int32_t* d_dropped, uint32_t* d_status, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    ObjCam c;
    if (cam ? !obj_cam(e, cam, &c) : false) return DSAC_ERR_ARG;
    if (!cam) {
        if (int rc = dataset_cameras_check(e, "dsac_register_depth_device", n)) return rc;
        c = e->ds_cam0;
    }
    if (n < 1 || !d_raw || !d_depth || d_raw == d_depth || (d_status && !d_dropped))
        return fail(e, DSAC_ERR_ARG, "dsac_register_depth_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = (cudaStream_t)stream_v;
    // cam == NULL: the per-dataset table; only a registration reads it (raw_data 0 passes the depth through)
    const bool table = !cam && c.raw_data;
    if (table)
        if (int rc = dataset_cameras_wait(e, stream)) return rc;
    const size_t count = (size_t)n * c.width * c.height;
    if (d_dropped) CU(cudaMemsetAsync(d_dropped, 0, (size_t)n * sizeof(int32_t), stream));
    if (c.raw_data) {
        CU(e->d_reg_keys.reserve(count * sizeof(uint64_t)));
        CU(cudaMemsetAsync(e->d_reg_keys, 0, count * sizeof(uint64_t), stream));
    }
    if (table) k_register_depth_cam<<<grid_of(count, 256), 256, 0, stream>>>(c, e->d_ds_cams, n, d_raw, e->d_reg_keys, d_depth, d_dropped);
    else k_register_depth<<<grid_of(count, 256), 256, 0, stream>>>(c, n, d_raw, e->d_reg_keys, d_depth, d_dropped);
    e->launches++;
    if (table)
        if (int rc = dataset_cameras_done(e, stream)) return rc;
    if (c.raw_data) {
        k_register_finish<<<grid_of(count, 256), 256, 0, stream>>>(count, e->d_reg_keys, d_depth);
        e->launches++;
    }
    if (d_status) {
        k_dropped_status<<<grid_of(n, 128), 128, 0, stream>>>(n, d_dropped, d_status);
        e->launches++;
    }
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_obj_coords_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n_frames, int32_t n, const int32_t* d_idx,
                           const uint16_t* d_depth, const double* d_poses, int16_t* d_coords, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    ObjCam c;
    if (cam ? !obj_cam(e, cam, &c) : false) return DSAC_ERR_ARG;
    if (!cam) {
        if (int rc = dataset_cameras_check(e, "dsac_obj_coords_device", n_frames)) return rc;
        c = e->ds_cam0;
    }
    if (n < 1 || n_frames < 1 || (!d_idx && n > n_frames) || !d_depth || !d_poses || !d_coords)
        return fail(e, DSAC_ERR_ARG, "dsac_obj_coords_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = (cudaStream_t)stream_v;
    const size_t count = (size_t)n * c.width * c.height;
    if (cam) {
        k_obj_coords<<<grid_of(count, 256), 256, 0, stream>>>(c, n_frames, n, d_idx, d_depth, d_poses, d_coords);
    } else {
        if (int rc = dataset_cameras_wait(e, stream)) return rc;
        k_obj_coords_cam<<<grid_of(count, 256), 256, 0, stream>>>(c, e->d_ds_cams, n_frames, n, d_idx, d_depth, d_poses, d_coords);
        if (int rc = dataset_cameras_done(e, stream)) return rc;
    }
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_obj_rng_init_device(dsac_engine* e, uint32_t seed, int32_t n_streams, uint32_t* d_state, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n_streams < 1 || !d_state) return fail(e, DSAC_ERR_ARG, "dsac_obj_rng_init_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    k_obj_rng_init<<<grid_of(n_streams, 32), 32, 0, (cudaStream_t)stream_v>>>(seed, n_streams, d_state);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_obj_draw_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n_frames, const uint16_t* d_depth,
                         const double* d_poses, int32_t n_images, int32_t n_patches, int32_t n_streams,
                         int32_t max_attempts, uint32_t* d_state, int32_t* d_img, int32_t* d_centre, float* d_label,
                         uint32_t* d_status, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    ObjDrawParams p;
    if (cam ? !obj_cam(e, cam, &p.cam) : false) return DSAC_ERR_ARG;
    if (!cam) {
        if (int rc = dataset_cameras_check(e, "dsac_obj_draw_device", n_frames)) return rc;
        p.cam = e->ds_cam0;   // the frame size of every entry
    }
    if (p.cam.width <= UP_PATCH || p.cam.height <= UP_PATCH)
        return fail(e, DSAC_ERR_ARG, "a %dx%d frame holds no %d-pixel patch centre", p.cam.width, p.cam.height, UP_PATCH);
    if (n_frames < 1 || n_images < 1 || n_patches < 1 || n_streams < 1 || max_attempts < 32 || !d_depth || !d_poses ||
        !d_state || !d_img || !d_centre || !d_label || !d_status)
        return fail(e, DSAC_ERR_ARG, "dsac_obj_draw_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    p.depth = d_depth; p.poses = d_poses;
    p.n_frames = n_frames; p.n_images = n_images; p.n_patches = n_patches; p.n_streams = n_streams;
    p.max_attempts = max_attempts; p.state = d_state;
    p.img = d_img; p.centre = d_centre; p.label = d_label; p.status = d_status;
    p.cams = nullptr;
    cudaStream_t stream = (cudaStream_t)stream_v;
    if (cam) {
        k_obj_draw<<<grid_of(n_streams, OBJ_DRAW_WARPS), 32 * OBJ_DRAW_WARPS, 0, stream>>>(p);
    } else {
        if (int rc = dataset_cameras_wait(e, stream)) return rc;
        p.cams = e->d_ds_cams;
        k_obj_draw_cam<<<grid_of(n_streams, OBJ_DRAW_WARPS), 32 * OBJ_DRAW_WARPS, 0, stream>>>(p);
        if (int rc = dataset_cameras_done(e, stream)) return rc;
    }
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_gather_patches_at_device(dsac_engine* e, int32_t n, const uint8_t* d_frames, int32_t n_frames, int32_t width,
                                  int32_t height, const int32_t* d_frame, const int32_t* d_centre, float mean,
                                  float* d_patches, uint32_t* d_status, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n < 1 || n_frames < 1 || !d_frames || !d_frame || !d_centre || !d_patches)
        return fail(e, DSAC_ERR_ARG, "dsac_gather_patches_at_device: bad arguments");
    if (width < UP_PATCH || height < UP_PATCH) return fail(e, DSAC_ERR_ARG, "frame %dx%d smaller than a %d-pixel patch", width, height, UP_PATCH);
    CU(cudaSetDevice(e->cfg.device));
    cudaStream_t stream = (cudaStream_t)stream_v;
    GatherAtParams p;
    p.frames = d_frames; p.width = width; p.height = height; p.n_frames = n_frames;
    p.frame = d_frame; p.centre = d_centre; p.mean = mean; p.patches = d_patches; p.status = d_status;
    if (d_status) CU(cudaMemsetAsync(d_status, 0, sizeof(uint32_t), stream));
    k_gather_patches_at<<<n, UP_THREADS, 0, stream>>>(p);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

// ----------------------------------------------------------------------------- score-CNN pre-training data path

int dsac_score_draw_device(dsac_engine* e, int32_t n_frames, int32_t width, int32_t height, int32_t n_images,
                           int32_t hyps_per_image, int32_t n_streams, uint32_t* d_state, int32_t* d_img, int32_t* d_pix,
                           int32_t* d_drift, double* d_noise, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n_frames < 1 || n_images < 1 || hyps_per_image < 1 || n_streams < 1 || !d_state || !d_img || !d_pix || !d_drift ||
        !d_noise)
        return fail(e, DSAC_ERR_ARG, "dsac_score_draw_device: bad arguments");
    ScoreDrawParams p;
    if (width <= UP_PATCH || height <= UP_PATCH)
        return fail(e, DSAC_ERR_ARG, "a %dx%d frame holds no %d-pixel patch centre", width, height, UP_PATCH);
    p.nx = score_grid_bounds(width, p.xb, SCORE_GRID_MAX);
    p.ny = score_grid_bounds(height, p.yb, SCORE_GRID_MAX);
    // below 83 px the loop runs more than 40 times and the reference writes past its 40x40 sampling grid
    if (p.nx != DSAC_GRID || p.ny != DSAC_GRID)
        return fail(e, DSAC_ERR_ARG, "a %dx%d frame gives a %dx%d sampling loop (40x40 needed: 83 px or more)", width,
                    height, p.nx, p.ny);
    CU(cudaSetDevice(e->cfg.device));
    p.n_frames = n_frames; p.n_images = n_images; p.hyps = hyps_per_image; p.n_streams = n_streams;
    p.state = d_state; p.img = d_img; p.pix = d_pix; p.drift = d_drift; p.noise = d_noise;
    k_score_draw<<<grid_of(n_streams, OBJ_DRAW_WARPS), 32 * OBJ_DRAW_WARPS, 0, (cudaStream_t)stream_v>>>(p);
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

int dsac_score_maps_device(dsac_engine* e, int32_t n_images, int32_t hyps_per_image, const int32_t* d_img,
                           const double* d_gt_jp, const int16_t* d_coords, const int32_t* d_pix, const double* d_noise,
                           float temperature, float* d_maps, double* d_labels, int32_t* d_correct, void* stream_v) {
    if (!e) return DSAC_ERR_ARG;
    if (n_images < 1 || hyps_per_image < 1 || (int64_t)n_images * hyps_per_image > INT32_MAX || !d_img || !d_gt_jp ||
        !d_coords || !d_pix || !d_noise || !d_maps || !d_labels)
        return fail(e, DSAC_ERR_ARG, "dsac_score_maps_device: bad arguments");
    CU(cudaSetDevice(e->cfg.device));
    ScoreMapsParams p;
    p.img = d_img; p.gt_jp = d_gt_jp; p.coords = d_coords; p.pix = d_pix; p.noise = d_noise;
    p.hyps = hyps_per_image;
    p.f = e->cfg.focal; p.cxf = (float)e->cfg.cx; p.cyf = (float)e->cfg.cy; p.temperature = temperature;
    p.maps = d_maps; p.labels = d_labels; p.correct = d_correct;
    p.cams = nullptr; p.n_cams = 0;
    cudaStream_t stream = (cudaStream_t)stream_v;
    if (!e->ds_cams_n) {
        k_score_maps<<<(unsigned)(n_images * hyps_per_image), SM_THREADS, 0, stream>>>(p);
    } else {   // the camera of frame img[i] (getCamMat of its dataset entry)
        if (int rc = dataset_cameras_wait(e, stream)) return rc;
        p.cams = e->d_ds_cams; p.n_cams = e->ds_cams_n;
        k_score_maps_cam<<<(unsigned)(n_images * hyps_per_image), SM_THREADS, 0, stream>>>(p);
        if (int rc = dataset_cameras_done(e, stream)) return rc;
    }
    e->launches++;
    CU(cudaGetLastError());
    return DSAC_OK;
}

}  // extern "C"

// One grow-only scratch block of views, each at 256-byte alignment, in the order given: the block grows to hold them,
// then every view points at its slice.  ev (nullable): the block's last user, on any stream -- the host waits for it
// before the block is re-allocated, `stream` otherwise.
struct ScratchView {
    size_t bytes;
    void* view;
    void (*set)(void* view, char* at);
};
template <class T> static ScratchView view(T*& v, size_t count) {
    return {count * sizeof(T), &v, [](void* w, char* at) { *static_cast<T**>(w) = reinterpret_cast<T*>(at); }};
}
static int carve_scratch(dsac_engine* e, DevMem<char>& buf, std::initializer_list<ScratchView> views, cudaEvent_t ev = nullptr,
                         cudaStream_t stream = nullptr) {
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    size_t total = 0;
    for (const ScratchView& v : views) total += al(v.bytes);
    if (ev && total > buf.bytes()) CU(cudaEventSynchronize(ev));
    else if (ev) CU(cudaStreamWaitEvent(stream, ev, 0));
    CU(buf.reserve(total));
    char* p = buf;
    for (const ScratchView& v : views) {
        v.set(v.view, p);
        p += al(v.bytes);
    }
    return DSAC_OK;
}

#include "backward_host.inc"
#include "backward_dsac_host.inc"
#include "uncertainty_host.inc"
#include "modes_host.inc"
#include "rig_host.inc"
#include "rig_backward_host.inc"
#include "rig_tracking_host.inc"
#include "rig_modes_host.inc"
