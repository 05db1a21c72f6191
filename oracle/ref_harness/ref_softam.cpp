// ref_softam.cpp -- oracle/_ref/libref_softam.so: the reference's OWN soft-argmax pipeline (core/cnn_softam.h,
// core/maxloss.h, core/Hypothesis.cpp, core/types.h, core/thread_rand.cpp, core/properties.cpp, core/read_data.cpp,
// core/dataset.h and the whole of core/test_ransac_softam.cpp), compiled UNMODIFIED from /root/reference against the
// API shims of oracle/shim, behind a C interface for tests/test_oracle_vs_ref.py.  TEST INFRASTRUCTURE ONLY.
//
// The reference's main() is kept (renamed by the preprocessor) and run as is on a synthetic dataset directory; the
// free functions of cnn_softam.h are additionally called directly so that every intermediate result can be compared
// at full precision.
#include <unistd.h>

#include <iostream>
#include <sstream>

#include "ref_env.h"

#define main ref_test_ransac_softam_main
#include "test_ransac_softam.cpp"   // -> properties.h, thread_rand.h, util.h, stop_watch.h, dataset.h, lua_calls.h, cnn_softam.h
#undef main

namespace {
struct CoutSilencer {   // the reference narrates every stage on std::cout
    std::streambuf* old;
    std::ostringstream sink;
    CoutSilencer() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~CoutSilencer() { std::cout.rdbuf(old); }
};

// outputs of the last processImage call, kept for the gradient-factor calls
struct LastForward {
    std::vector<jp::cv_trans_t> hyps;
    jp::cv_trans_t refAvgHyp, avgHyp;
    std::vector<std::vector<cv::Point2f>> imgPts;
    std::vector<std::vector<cv::Point3f>> objPts;
    std::vector<std::vector<int>> imgIdx;
    std::vector<cv::Mat_<cv::Vec3f>> patches;
    std::vector<double> sfScores;
    jp::img_coord_t estObj;
    cv::Mat_<cv::Point2i> sampling;
    std::vector<std::vector<cv::Point2i>> sampledPoints;
    cv::Mat_<int> inlierMap;
    std::vector<std::vector<int>> pixelIdxs;
    Hypothesis poseGT;
    lua_State *stateRGB = nullptr, *stateObj = nullptr;
} g_last;

void vec3(const cv::Mat& m, double* out) {
    for (int i = 0; i < 3; i++) out[i] = m.rows == 1 ? m.at<double>(0, i) : m.at<double>(i, 0);
}
}  // namespace

extern "C" {

// The camera GlobalProperties::getCamMat() builds the calibration matrix from (properties.cpp:55-57 defaults, the drivers'
// -fl / -xs / -ys flags): principal point = image centre (320, 240) + shift.  Persists across calls; the default is 525, 0, 0.
int ref_set_camera(float focal, float x_shift, float y_shift) {
    GlobalProperties* gp = GlobalProperties::getInstance();
    gp->dP.focalLength = focal;
    gp->dP.xShift = x_shift;
    gp->dP.yShift = y_shift;
    return 0;
}

struct ref_config {
    double alpha, beta, grad_clamp;
    int32_t n_hyps, thr2d, inlier_count, ref_steps;
    float sub_sample;
    uint32_t seed;
    int32_t n_threads;
    int64_t frame;   // global frame index (stream key)
};

struct ref_forward_out {
    int32_t* pix;          // [1600*2] sampling (x, y), row-major cells
    int16_t* est_obj;      // [1600*3] estObj as the pipeline saw it
    double* hyp_rvec;      // [H*3]
    double* hyp_tvec;      // [H*3]
    int32_t* img_idx;      // [H*4]
    float* diffmaps;       // [H*1600] as handed to the score call
    double* scores;        // [H]
    double* sf;            // [H]
    double entropy;
    double avg[6], ref[6];
    int32_t* inlier_map;   // [1600]
    int32_t* pixel_idxs;   // [ref_steps*1600], -1 beyond the permutations generated
    int32_t n_perm_steps;
    double loss, rot_err, t_err;
    int32_t correct;
};

static void ref_setup(const ref_config* c, const int16_t* coords) {
    g_env.coords = coords;
    g_env.n_frames = 1;
    g_env.frame0 = c->frame;
    g_env.cur = 0;
    g_env.alpha = c->alpha; g_env.beta = c->beta; g_env.grad_clamp = c->grad_clamp;
    g_env.thr = c->thr2d;
    g_env.seed = c->seed;
    g_env.T = c->n_threads;
}

// processImage (cnn_softam.h:960-1180) on one synthetic frame; the sampler streams are those of global frame c->frame.
int ref_softam_forward(const ref_config* c, const int16_t* coords, const double gt_R[9], const double gt_t[3], ref_forward_out* o) {
    CoutSilencer quiet;
    ref_setup(c, coords);
    ref_reseed_for_frame(0);
    if (!g_last.stateRGB) {
        g_last.stateRGB = luaL_newstate(); g_last.stateRGB->script = "coord.lua";
        g_last.stateObj = luaL_newstate(); g_last.stateObj->script = "score.lua";
    }
    GlobalProperties* gp = GlobalProperties::getInstance();
    cv::Mat camMat = gp->getCamMat();
    jp::img_bgr_t img = jp::img_bgr_t::zeros(gp->dP.imageHeight, gp->dP.imageWidth);
    cv::Mat_<double> R(3, 3);
    for (int i = 0; i < 9; i++) R(i / 3, i % 3) = gt_R[i];
    g_last.poseGT = Hypothesis(R, cv::Point3d(gt_t[0], gt_t[1], gt_t[2]));
    double loss = 0, sfEntropy = 0, tErr = 0, rotErr = 0;
    bool correct = false;
    g_last.pixelIdxs.clear();
    processImage(img, g_last.poseGT, g_last.stateRGB, g_last.stateObj, c->n_hyps, 4, camMat, c->thr2d, c->inlier_count, c->ref_steps,
                 loss, sfEntropy, correct, g_last.hyps, g_last.refAvgHyp, g_last.avgHyp, g_last.imgPts, g_last.objPts, g_last.imgIdx,
                 g_last.patches, g_last.sfScores, g_last.estObj, g_last.sampling, g_last.sampledPoints, g_last.inlierMap,
                 g_last.pixelIdxs, tErr, rotErr);
    const int H = c->n_hyps, N = ORC_N;
    for (int y = 0; y < ORC_GRID; y++)
        for (int x = 0; x < ORC_GRID; x++) {
            const int p = y * ORC_GRID + x;
            if (o->pix) { o->pix[p * 2] = g_last.sampling(y, x).x; o->pix[p * 2 + 1] = g_last.sampling(y, x).y; }
            if (o->est_obj) for (int k = 0; k < 3; k++) o->est_obj[p * 3 + k] = g_last.estObj(y, x)[k];
            if (o->inlier_map) o->inlier_map[p] = g_last.inlierMap(y, x);
        }
    for (int h = 0; h < H; h++) {
        if (o->hyp_rvec) vec3(g_last.hyps[h].first, o->hyp_rvec + h * 3);
        if (o->hyp_tvec) vec3(g_last.hyps[h].second, o->hyp_tvec + h * 3);
        if (o->img_idx) for (int j = 0; j < 4; j++) o->img_idx[h * 4 + j] = g_last.imgIdx[h][j];
        if (o->sf) o->sf[h] = g_last.sfScores[h];
        if (o->scores) o->scores[h] = g_env.scores[h];
    }
    if (o->diffmaps) memcpy(o->diffmaps, g_env.diffmaps.data(), (size_t)H * N * sizeof(float));
    o->entropy = sfEntropy;
    vec3(g_last.avgHyp.first, o->avg); vec3(g_last.avgHyp.second, o->avg + 3);
    vec3(g_last.refAvgHyp.first, o->ref); vec3(g_last.refAvgHyp.second, o->ref + 3);
    o->n_perm_steps = 0;
    if (o->pixel_idxs) {
        for (int s = 0; s < c->ref_steps; s++)
            for (int i = 0; i < N; i++) o->pixel_idxs[s * N + i] = -1;
        for (int s = 0; s < (int)g_last.pixelIdxs.size(); s++) {
            if (g_last.pixelIdxs[s].empty()) continue;
            o->n_perm_steps = s + 1;
            for (int i = 0; i < (int)g_last.pixelIdxs[s].size() && i < N; i++) o->pixel_idxs[s * N + i] = g_last.pixelIdxs[s][i];
        }
    } else {
        for (int s = 0; s < (int)g_last.pixelIdxs.size(); s++)
            if (!g_last.pixelIdxs[s].empty()) o->n_perm_steps = s + 1;
    }
    o->loss = loss; o->rot_err = rotErr; o->t_err = tErr; o->correct = correct ? 1 : 0;
    return 0;
}

// The factors of the backward pass, by the reference's own functions on the outputs of the last ref_softam_forward:
// dLossMax (maxloss.h:87), dRefineObj (cnn_softam.h:853), dRefineHyp (:738), dPNP (:101) per hypothesis and dScore (:564)
// summed over the hypotheses for the given score output-gradients.  Any output may be null.
int ref_softam_factors(const ref_config* c, double* dloss_dref /*6*/, double* dref_dobj /*6*4800*/, double* dref_dhyp /*36*/,
                       double* dpnp /*H*72*/, const double* score_out_grads /*H, nullable*/, double* dscore_sum /*4800*/) {
    CoutSilencer quiet;
    GlobalProperties* gp = GlobalProperties::getInstance();
    cv::Mat camMat = gp->getCamMat();
    const int H = c->n_hyps;
    if (dloss_dref) {
        jp::jp_trans_t j = jp::cv2our(g_last.refAvgHyp);
        cv::Mat_<double> d = dLossMax(Hypothesis(j.first, j.second).getRodVecAndTrans(), g_last.poseGT.getRodVecAndTrans());
        for (int k = 0; k < 6; k++) dloss_dref[k] = d(0, k);
    }
    if (dref_dobj) {
        cv::Mat_<double> d = dRefineObj(c->inlier_count, c->ref_steps, c->sub_sample, c->thr2d, g_last.pixelIdxs, g_last.estObj,
                                        g_last.sampling, camMat, g_last.avgHyp, g_last.inlierMap);
        for (int k = 0; k < 6; k++)
            for (int i = 0; i < ORC_N * 3; i++) dref_dobj[k * ORC_N * 3 + i] = d(k, i);
    }
    if (dref_dhyp) {
        cv::Mat_<double> d = dRefineHyp(c->inlier_count, c->ref_steps, c->thr2d, g_last.pixelIdxs, g_last.estObj, g_last.sampling, camMat,
                                        g_last.avgHyp);
        for (int k = 0; k < 36; k++) dref_dhyp[k] = d(k / 6, k % 6);
    }
    if (dpnp)
        for (int h = 0; h < H; h++) {
            cv::Mat_<double> d = dPNP(g_last.imgPts[h], g_last.objPts[h]);
            for (int k = 0; k < 72; k++) dpnp[h * 72 + k] = d(k / 12, k % 12);
        }
    if (score_out_grads && dscore_sum) {
        std::vector<double> sog(score_out_grads, score_out_grads + H);
        std::vector<cv::Mat_<double>> jac;
        dScore(g_last.estObj, g_last.sampling, g_last.sampledPoints, g_last.stateObj, jac, sog);
        for (int i = 0; i < ORC_N * 3; i++) dscore_sum[i] = 0;
        for (int h = 0; h < H; h++)
            for (int i = 0; i < ORC_N * 3; i++) dscore_sum[i] += jac[h](0, i);
    }
    return 0;
}

// stochasticSubSample (cnn_softam.h:283-309) by the reference's own ThreadRand, after `skip_draws` thread-0 draws.
int ref_stochastic_subsample(uint32_t seed, int skip_draws, int32_t* pix) {
    omp_set_num_threads(1);
    ThreadRand::forceInit(seed);
    for (int i = 0; i < skip_draws; i++) irand(0, 1);
    jp::img_bgr_t img = jp::img_bgr_t::zeros(480, 640);
    cv::Mat_<cv::Point2i> s = stochasticSubSample(img, CNN_OBJ_PATCHSIZE, CNN_RGB_PATCHSIZE);
    for (int y = 0; y < ORC_GRID; y++)
        for (int x = 0; x < ORC_GRID; x++) { pix[(y * ORC_GRID + x) * 2] = s(y, x).x; pix[(y * ORC_GRID + x) * 2 + 1] = s(y, x).y; }
    return 0;
}

// The ground-truth pose the reference derives from a 7-Scenes pose file (read_data.cpp:69-133 + Hypothesis(info)),
// read relative to the current directory (translation.txt is looked up there).
int ref_read_pose(const char* dir, const char* pose_file, double R[9], double t[3]) {
    CoutSilencer quiet;
    char old[4096];
    if (!getcwd(old, sizeof(old))) return -1;
    if (chdir(dir) != 0) return -2;
    jp::info_t info;
    const bool ok = jp::readData(std::string(pose_file), info);
    if (chdir(old) != 0) return -3;
    if (!ok) return -4;
    Hypothesis h(info);
    cv::Mat rot = h.getRotation();
    for (int i = 0; i < 9; i++) R[i] = rot.at<double>(i / 3, i % 3);
    t[0] = h.getTranslation().x; t[1] = h.getTranslation().y; t[2] = h.getTranslation().z;
    return 0;
}

// The reference's test driver, main() of test_ransac_softam.cpp, run in `dir` (which holds ./test/<scene>/{rgb_noseg,
// depth_noseg,poses}/frame-%06d.*, optional translation.txt / default.config); writes its two log files there.
int ref_run_test_main(const ref_config* c, const char* dir, const int16_t* coords, int n_frames, int n_args, const char** args) {
    CoutSilencer quiet;
    ref_setup(c, coords);
    g_env.n_frames = n_frames;
    char old[4096];
    if (!getcwd(old, sizeof(old))) return -1;
    if (chdir(dir) != 0) return -2;
    std::vector<const char*> argv;
    argv.push_back("test_ransac_softam");
    for (int i = 0; i < n_args; i++) argv.push_back(args[i]);
    argv.push_back(REF_ARGV_SENTINEL);
    int rc = ref_test_ransac_softam_main((int)argv.size(), argv.data());
    if (chdir(old) != 0) return -3;
    return rc;
}

}  // extern "C"
