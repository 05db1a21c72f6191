// ref_dsac.cpp -- oracle/_ref/libref_dsac.so: the reference's OWN DSAC / RANSAC variant (core/cnn.h and the whole of
// core/test_ransac.cpp), compiled UNMODIFIED from /root/reference against the API shims of oracle/shim, behind a C
// interface for tests/test_oracle_vs_ref.py (SURVEY.md section 8f row N1).  TEST INFRASTRUCTURE ONLY.
#include <unistd.h>

#include <iostream>
#include <sstream>

#include "ref_env.h"

#define main ref_test_ransac_main
#include "test_ransac.cpp"   // -> properties.h, thread_rand.h, util.h, stop_watch.h, dataset.h, lua_calls.h, cnn.h
#undef main

namespace {
struct CoutSilencer {
    std::streambuf* old;
    std::ostringstream sink;
    CoutSilencer() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~CoutSilencer() { std::cout.rdbuf(old); }
};
void vec3(const cv::Mat& m, double* out) {
    for (int i = 0; i < 3; i++) out[i] = m.rows == 1 ? m.at<double>(0, i) : m.at<double>(i, 0);
}
lua_State *g_stateRGB = nullptr, *g_stateObj = nullptr;
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
    int64_t frame;
};

struct ref_dsac_out {
    double* hyp_rvec;      // [H*3]
    double* hyp_tvec;      // [H*3]
    int32_t* img_idx;      // [H*4]
    double* sf;            // [H]
    double* ref_pose;      // [H*6] refined hypotheses, cv convention
    double* losses;        // [H]
    int32_t* inlier_maps;  // [H*1600]
    double entropy, expected_loss, rot_err, t_err;
    int32_t hyp_idx, correct;
};

// processImage of the DSAC / RANSAC variant (cnn.h:1028-1257) on one synthetic frame; random_draw = pP.randomDraw.
int ref_dsac_forward(const ref_config* c, int random_draw, const int16_t* coords, const double gt_R[9], const double gt_t[3], ref_dsac_out* o) {
    CoutSilencer quiet;
    g_env.coords = coords; g_env.n_frames = 1; g_env.frame0 = c->frame; g_env.cur = 0;
    g_env.alpha = c->alpha; g_env.beta = c->beta; g_env.grad_clamp = c->grad_clamp; g_env.thr = c->thr2d;
    g_env.seed = c->seed; g_env.T = c->n_threads;
    ref_reseed_for_frame(0);
    if (!g_stateRGB) {
        g_stateRGB = luaL_newstate(); g_stateRGB->script = "coord.lua";
        g_stateObj = luaL_newstate(); g_stateObj->script = "score.lua";
    }
    GlobalProperties* gp = GlobalProperties::getInstance();
    gp->pP.randomDraw = random_draw != 0;
    cv::Mat camMat = gp->getCamMat();
    jp::img_bgr_t img = jp::img_bgr_t::zeros(gp->dP.imageHeight, gp->dP.imageWidth);
    cv::Mat_<double> R(3, 3);
    for (int i = 0; i < 9; i++) R(i / 3, i % 3) = gt_R[i];
    Hypothesis poseGT(R, cv::Point3d(gt_t[0], gt_t[1], gt_t[2]));
    double expectedLoss = 0, sfEntropy = 0, tErr = 0, rotErr = 0;
    bool correct = false;
    int hypIdx = 0;
    std::vector<jp::cv_trans_t> hyps, refHyps;
    std::vector<std::vector<cv::Point2f>> imgPts;
    std::vector<std::vector<cv::Point3f>> objPts;
    std::vector<std::vector<int>> imgIdx;
    std::vector<cv::Mat_<cv::Vec3f>> patches;
    std::vector<double> sfScores, losses;
    jp::img_coord_t estObj;
    cv::Mat_<cv::Point2i> sampling;
    std::vector<std::vector<cv::Point2i>> sampledPoints;
    std::vector<cv::Mat_<int>> inlierMaps;
    std::vector<std::vector<std::vector<int>>> pixelIdxs;
    processImage(img, poseGT, g_stateRGB, g_stateObj, c->n_hyps, 4, camMat, c->thr2d, c->inlier_count, c->ref_steps, expectedLoss, sfEntropy,
                 correct, hyps, refHyps, imgPts, objPts, imgIdx, patches, sfScores, estObj, sampling, sampledPoints, losses, inlierMaps,
                 pixelIdxs, tErr, rotErr, hypIdx);
    const int H = c->n_hyps;
    for (int h = 0; h < H; h++) {
        if (o->hyp_rvec) vec3(hyps[h].first, o->hyp_rvec + h * 3);
        if (o->hyp_tvec) vec3(hyps[h].second, o->hyp_tvec + h * 3);
        if (o->img_idx) for (int j = 0; j < 4; j++) o->img_idx[h * 4 + j] = imgIdx[h][j];
        if (o->sf) o->sf[h] = sfScores[h];
        if (o->ref_pose) { vec3(refHyps[h].first, o->ref_pose + h * 6); vec3(refHyps[h].second, o->ref_pose + h * 6 + 3); }
        if (o->losses) o->losses[h] = losses[h];
        if (o->inlier_maps)
            for (int y = 0; y < ORC_GRID; y++)
                for (int x = 0; x < ORC_GRID; x++) o->inlier_maps[(size_t)h * ORC_N + y * ORC_GRID + x] = inlierMaps[h](y, x);
    }
    o->entropy = sfEntropy; o->expected_loss = expectedLoss; o->rot_err = rotErr; o->t_err = tErr;
    o->hyp_idx = hypIdx; o->correct = correct ? 1 : 0;
    return 0;
}

}  // extern "C"
