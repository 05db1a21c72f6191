// ref_train_score.cpp -- the reference's own train_score.cpp (main renamed) with its jp::Dataset, compiled unmodified by
// tests/golden/make_ref_score.py against the API shims of oracle/shim and the png++ stand-in of tests/golden/ref_obj.  It
// exposes getRandHyp and assembleData, so that the fixture ref_score.npz holds what the reference itself computes.
// TEST INFRASTRUCTURE ONLY (fixture generation; never part of a test run).
//
// The coordinate CNN is a stub behind the Lua API stand-in (oracle/shim/lua.hpp), dispatched here (oracle/ref_harness/
// ref_env.h is not used: its png hook re-seeds ThreadRand on every load).  forward(count, patches) reads each patch's
// centre pixel, which on the coded frames of tests/obj_oracle.coded_bgr gives (frame, x, y) back, records it (the
// frame and the sampling grid of the image being assembled) and returns score_stub_coord(frame, x, y) / 1000, a
// deterministic scene coordinate that tests/test_score_ref_fixture.py recomputes.
#include <omp.h>

#include <cmath>
#include <iostream>
#include <map>
#include <sstream>
#include <vector>

#include <opencv2/opencv.hpp>
#include <lua.hpp>

// One OpenCV operation train_score.cpp uses (getRandHyp) that the API shim does not provide, restated from OpenCV's
// definition (core/include/opencv2/core/types.hpp): Point3_ * double scales each component, saturate_cast back to T
// (the identity for double).
namespace cv {
template <typename T> inline Point3_<T> operator*(const Point3_<T>& a, double b) {
    return Point3_<T>((T)(a.x * b), (T)(a.y * b), (T)(a.z * b));
}
}  // namespace cv

#define main ref_train_score_main
#include "train_score.cpp"
#undef main

namespace {
struct RegImage {
    int w = 0, h = 0;
    std::vector<uint8_t> bgr;
};
std::map<std::string, RegImage> g_images;
jp::Dataset* g_dataset = nullptr;
std::vector<double> g_gt;            // [F][12] jp poses (info.rotation, info.center * 1000) of the dataset
std::vector<int32_t> g_grid;         // per getCoordImg call: frame, then 1600 (x, y)
float g_focal = 525.f, g_cx = 320.f, g_cy = 240.f;

struct Quiet {   // the reference prints; the fixture generator does not want it
    std::streambuf* old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf()) { std::cout.rdbuf(sink.rdbuf()); }
    ~Quiet() { std::cout.rdbuf(old); }
};

// The stub's scene coordinate (mm) of pixel (x, y) of frame f: a depth d = 1500 + (7x + 13y + 29f) mod 1000, the pixel
// back-projected with the reference's camera into the jp camera frame (y and z flipped), moved into the scene by the
// frame's ground truth (R^T (cam - t)) and rounded to integers (floor(v + 0.5)).
void score_stub_coord(int f, int x, int y, double out[3]) {
    const double d = 1500.0 + (double)((7 * x + 13 * y + 29 * f) % 1000);
    const double cam[3] = {((double)x - g_cx) * d / g_focal, -(((double)y - g_cy) * d / g_focal), -d};
    const double* P = &g_gt[(size_t)f * 12];
    const double q[3] = {cam[0] - P[9], cam[1] - P[10], cam[2] - P[11]};
    for (int r = 0; r < 3; r++) out[r] = std::floor(P[r] * q[0] + P[3 + r] * q[1] + P[6 + r] * q[2] + 0.5);
}
}  // namespace

void shim_lua_dispatch(lua_State* L, const std::string& fn, std::vector<shim_lua_value>& args, int /*nresults*/,
                       std::vector<shim_lua_value>& results) {
    if (fn != "forward" || L->script.find("score") != std::string::npos) return;
    // lua_calls.h:252-273: (count, patches pushed n -> c -> y -> x, BGR bytes as numbers) -> count * 3 metres
    const int count = (int)args[0].num;
    const std::vector<double>& px = *args[1].tab;
    shim_lua_value t;
    t.kind = shim_lua_value::TABLE;
    t.tab = std::make_shared<std::vector<double>>((size_t)count * 3, 0.0);
    const size_t plane = 42 * 42, centre = 21 * 42 + 21;
    for (int i = 0; i < count; i++) {
        const int b = (int)px[(size_t)i * 3 * plane + centre], g = (int)px[((size_t)i * 3 + 1) * plane + centre],
                  r = (int)px[((size_t)i * 3 + 2) * plane + centre];
        const int f = r / 16, x = b + 256 * ((r % 16) % 4), y = g + 256 * ((r % 16) / 4);
        if (i == 0) g_grid.push_back(f);
        g_grid.push_back(x);
        g_grid.push_back(y);
        double c[3];
        score_stub_coord(f, x, y, c);
        // +-0.25 mm keeps float(v / 1000) * 1000 on the same side of the integer, whichever rounding the conversion uses
        for (int k = 0; k < 3; k++) (*t.tab)[(size_t)i * 3 + k] = (c[k] + (c[k] < 0 ? -0.25 : 0.25)) / 1000.0;
    }
    results.push_back(t);
}

extern "C" {
int ref_obj_png_lookup(const char* path, int* width, int* height, const uint8_t** bgr, const uint16_t** depth) {
    auto it = g_images.find(path);
    if (it == g_images.end()) return 0;
    *width = it->second.w;
    *height = it->second.h;
    *bgr = it->second.bgr.data();
    *depth = nullptr;
    return 1;
}

void ref_score_register_bgr(const char* path, int w, int h, const uint8_t* bgr) {
    RegImage& r = g_images[path];
    r.w = w; r.h = h;
    r.bgr.assign(bgr, bgr + (size_t)w * h * 3);
}

// dP of GlobalProperties: the RGB camera getCamMat builds (centre = width / 2 + xShift) and the frame size
void ref_score_camera(float focal, int w, int h) {
    Quiet q;
    GlobalProperties* gp = GlobalProperties::getInstance();
    gp->dP.focalLength = focal; gp->dP.xShift = 0; gp->dP.yShift = 0;
    gp->dP.imageWidth = w; gp->dP.imageHeight = h;
    gp->dP.rawData = false;
    cv::Mat_<float> K = gp->getCamMat();
    g_focal = K(0, 0); g_cx = K(0, 2); g_cy = K(1, 2);
}

// jp::Dataset(basePath); gt [F][12] receives the poses as jp::info_t holds them (rotation, centre * 1000, from float)
int ref_score_dataset(const char* base, double* gt) {
    Quiet q;
    delete g_dataset;
    g_dataset = new jp::Dataset(base, 1);
    const int F = (int)g_dataset->size();
    g_gt.assign((size_t)F * 12, 0.0);
    for (int f = 0; f < F; f++) {
        jp::info_t info;
        if (!g_dataset->getInfo(f, info)) return -1;
        for (int y = 0; y < 3; y++)
            for (int x = 0; x < 3; x++) g_gt[(size_t)f * 12 + 3 * y + x] = info.rotation(y, x);
        for (int k = 0; k < 3; k++) g_gt[(size_t)f * 12 + 9 + k] = (double)info.center[k] * 1000.0;
    }
    for (size_t i = 0; i < g_gt.size(); i++) gt[i] = g_gt[i];
    return F;
}

// ThreadRand::forceInit(seed) for T OpenMP threads
void ref_score_threads(uint32_t seed, int T) {
    omp_set_dynamic(0);
    omp_set_num_threads(T);
    ThreadRand::forceInit(seed);
}

// n calls of getRandHyp(gaussRot, gaussTrans) on thread 0 of the current generators: translation [n][3] and rotation
// matrix [n][9] of each returned Hypothesis
void ref_score_rand_hyp(float gauss_rot, float gauss_trans, int n, double* trans, double* rot) {
    for (int i = 0; i < n; i++) {
        Hypothesis h = getRandHyp(gauss_rot, gauss_trans);
        const cv::Point3d t = h.getTranslation();
        trans[3 * i] = t.x; trans[3 * i + 1] = t.y; trans[3 * i + 2] = t.z;
        const cv::Mat R = h.getRotation();
        for (int k = 0; k < 9; k++) rot[i * 9 + k] = R.at<double>(k / 3, k % 3);
    }
}

// one assembleData round (objTemperature 10): maps [n][40][40], labels [n], and per image the frame and the sampling
// grid [1600][2] (cell y * 40 + x) the coordinate stub saw
int ref_score_assemble(int n_images, int hyps, float* maps, double* labels, int32_t* frames, int32_t* grid) {
    Quiet q;
    lua_State* state = luaL_newstate();
    state->script = "train_obj.lua";
    std::vector<cv::Mat_<float>> data;
    std::vector<double> lab;
    g_grid.clear();
    assembleData(n_images, hyps, CNN_OBJ_PATCHSIZE, CNN_RGB_PATCHSIZE, *g_dataset, state, data, lab, 10.f);
    lua_close(state);
    for (size_t k = 0; k < data.size(); k++) {
        labels[k] = lab[k];
        for (int y = 0; y < 40; y++)
            for (int x = 0; x < 40; x++) maps[k * 1600 + y * 40 + x] = data[k](y, x);
    }
    // the stub saw the patches in getCoordImg's order: px = y * 40 + x (all 1600: no cell lies on the border)
    if (g_grid.size() != (size_t)n_images * 3201) return -1;
    for (int i = 0; i < n_images; i++) {
        const int32_t* g = &g_grid[(size_t)i * 3201];
        frames[i] = g[0];
        for (int k = 0; k < 3200; k++) grid[(size_t)i * 3200 + k] = g[1 + k];
    }
    return (int)data.size();
}
}
