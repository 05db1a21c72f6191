// ref_train_obj.cpp -- the reference's own train_obj.cpp (main renamed) with its jp::Dataset, compiled unmodified by
// tests/golden/make_ref_obj.py against the API shims of oracle/shim and the png++ stand-in next to this file.  It
// exposes getDepth, getObj, the pose reader's jp::info_t and assembleData, so that the fixture ref_obj.npz holds what
// the reference itself computes.  TEST INFRASTRUCTURE ONLY (fixture generation; never part of a test run).
//
// This harness keeps its own environment: oracle/ref_harness/ref_env.h is included for the Lua glue only, and its
// png hook (which re-seeds ThreadRand on every load) is never reached, since the png++ stand-in here does not call it.
// assembleData must run on the generators as ThreadRand::forceInit left them, across consecutive rounds.
#include <omp.h>

#include <iostream>
#include <map>
#include <sstream>
#include <vector>

#include "ref_env.h"
#include <opencv2/opencv.hpp>

// Two OpenCV operations train_obj.cpp uses that the API shim does not provide, restated from OpenCV's definitions
// (core/include/opencv2/core/matx.hpp): Vec /= int multiplies by the double 1./alpha and saturate_casts back;
// norm of a Vec is the L2 norm accumulated in double.
namespace cv {
template <typename T, int n> inline Vec<T, n>& operator/=(Vec<T, n>& a, int alpha) {
    const double ialpha = 1. / alpha;
    for (int i = 0; i < n; i++) a.val[i] = saturate_cast<T>(a.val[i] * ialpha);
    return a;
}
template <typename T, int n> inline double norm(const Vec<T, n>& v) {
    double s = 0;
    for (int i = 0; i < n; i++) s += (double)v.val[i] * v.val[i];
    return std::sqrt(s);
}
}  // namespace cv

#define main ref_train_obj_main
#include "train_obj.cpp"
#undef main

namespace {
struct RegImage {
    int w = 0, h = 0;
    std::vector<uint8_t> bgr;
    std::vector<uint16_t> depth;
};
std::map<std::string, RegImage> g_images;
jp::Dataset* g_dataset = nullptr;

struct Quiet {   // the reference prints; the fixture generator does not want it
    std::streambuf* old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf()) { std::cout.rdbuf(sink.rdbuf()); }
    ~Quiet() { std::cout.rdbuf(old); }
};
}  // namespace

extern "C" {
int ref_obj_png_lookup(const char* path, int* width, int* height, const uint8_t** bgr, const uint16_t** depth) {
    auto it = g_images.find(path);
    if (it == g_images.end()) return 0;
    *width = it->second.w;
    *height = it->second.h;
    *bgr = it->second.bgr.empty() ? nullptr : it->second.bgr.data();
    *depth = it->second.depth.empty() ? nullptr : it->second.depth.data();
    return 1;
}

void ref_obj_register_bgr(const char* path, int w, int h, const uint8_t* bgr) {
    RegImage& r = g_images[path];
    r.w = w; r.h = h;
    r.bgr.assign(bgr, bgr + (size_t)w * h * 3);
    r.depth.clear();
}

void ref_obj_register_depth(const char* path, int w, int h, const uint16_t* d) {
    RegImage& r = g_images[path];
    r.w = w; r.h = h;
    r.depth.assign(d, d + (size_t)w * h);
    r.bgr.clear();
}

// dP of GlobalProperties (properties.h): the camera the dataset reader uses
void ref_obj_camera(float focal, float xs, float ys, float sfl, float rxs, float rys, const double* trans, int raw_data, int w,
                    int h) {
    Quiet q;
    GlobalProperties* gp = GlobalProperties::getInstance();
    gp->dP.focalLength = focal; gp->dP.xShift = xs; gp->dP.yShift = ys;
    gp->dP.secondaryFocalLength = sfl; gp->dP.rawXShift = rxs; gp->dP.rawYShift = rys;
    gp->dP.sensorTrans = cv::Mat_<double>(4, 4);
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) gp->dP.sensorTrans(i, j) = trans[4 * i + j];
    gp->dP.rawData = raw_data != 0;
    gp->dP.imageWidth = w; gp->dP.imageHeight = h;
}

// jp::Dataset(basePath): rgb_noseg/, depth_noseg/, poses/ (file names only; pixels come from the registry)
int ref_obj_dataset(const char* base) {
    Quiet q;
    delete g_dataset;
    g_dataset = new jp::Dataset(base, 1);
    return (int)g_dataset->size();
}

void ref_obj_depth(int i, uint16_t* out) {
    jp::img_depth_t img;
    g_dataset->getDepth(i, img);
    for (int y = 0; y < img.rows; y++)
        for (int x = 0; x < img.cols; x++) out[(size_t)y * img.cols + x] = img(y, x);
}

void ref_obj_coords(int i, int16_t* out) {
    jp::img_coord_t img;
    g_dataset->getObj(i, img);
    for (int y = 0; y < img.rows; y++)
        for (int x = 0; x < img.cols; x++)
            for (int c = 0; c < 3; c++) out[((size_t)y * img.cols + x) * 3 + c] = img(y, x)[c];
}

int ref_obj_info(int i, float* rot9, float* center3) {
    Quiet q;
    jp::info_t info;
    if (!g_dataset->getInfo(i, info)) return 0;
    for (int y = 0; y < 3; y++)
        for (int x = 0; x < 3; x++) rot9[3 * y + x] = info.rotation(y, x);
    for (int k = 0; k < 3; k++) center3[k] = info.center[k];
    return 1;
}

// ThreadRand::forceInit(seed) for T OpenMP threads
void ref_obj_threads(uint32_t seed, int T) {
    omp_set_dynamic(0);
    omp_set_num_threads(T);
    ThreadRand::forceInit(seed);
}

// one assembleData round: per patch its top-left and centre pixels (BGR as float) and its label
void ref_obj_assemble(int n_images, int n_patches, float* corner, float* centre, float* labels) {
    Quiet q;
    std::vector<cv::Mat_<cv::Vec3f>> data;
    std::vector<cv::Vec3f> lab;
    assembleData(n_images, n_patches, 42, *g_dataset, data, lab);
    for (size_t k = 0; k < data.size(); k++)
        for (int c = 0; c < 3; c++) {
            corner[3 * k + c] = data[k](0, 0)[c];
            centre[3 * k + c] = data[k](21, 21)[c];
            labels[3 * k + c] = lab[k][c];
        }
}

// std::shuffle of iota(n) by the reference's default-seeded std::mt19937 (train_obj.cpp:266-270)
void ref_obj_permutation(int n, int32_t* out) {
    std::mt19937 randG;
    std::vector<int> p((size_t)n);
    for (int i = 0; i < n; i++) p[(size_t)i] = i;
    std::shuffle(p.begin(), p.end(), randG);
    for (int i = 0; i < n; i++) out[i] = p[(size_t)i];
}
}
