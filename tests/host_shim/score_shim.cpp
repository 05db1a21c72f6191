// Host build of the score-CNN pre-training data path's arithmetic (dsac_b200/csrc/scoretrain.cuh, DSAC_HOST_ONLY) for
// CPU-side checks against tests/score_oracle.py and against libstdc++ / gcc themselves.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include <random>
#include <sstream>
#include "../../dsac_b200/csrc/scoretrain.cuh"

namespace {
// a std::mt19937 holding [625] words + position (libstdc++'s stream format: the 624 words, then the position)
std::mt19937 engine_from(const uint32_t* st) {
    std::ostringstream os;
    for (int k = 0; k < 625; k++) os << st[k] << ' ';
    std::istringstream is(os.str());
    std::mt19937 g;
    is >> g;
    return g;
}
void engine_to(const std::mt19937& g, uint32_t* st) {
    std::stringstream ss;
    ss << g;
    for (int k = 0; k < 625; k++) ss >> st[k];
}

// what the reference spells: a three-argument constructor whose arguments are the draws (train_score.cpp:51-57)
struct P3 {
    double x, y, z;
    P3(double a, double b, double c) : x(a), y(b), z(c) {}
};
double ref_dgauss(std::mt19937& g, double stddev) { std::normal_distribution<double> d(0, stddev); return d(g); }
double ref_drand(std::mt19937& g) { std::uniform_real_distribution<double> d(0, 1); return d(g); }
}  // namespace

extern "C" {
// the draw of k_score_draw, sequentially: the streams of T threads from states [T][625], advanced in place
void shim_score_draw(uint32_t* state, int T, int n_frames, int width, int height, int n_images, int hyps, int32_t* img,
                     int32_t* pix, int32_t* drift, double* noise) {
    float xb[dsac::SCORE_GRID_MAX], yb[dsac::SCORE_GRID_MAX];
    const int nx = dsac::score_grid_bounds(width, xb, dsac::SCORE_GRID_MAX);
    const int ny = dsac::score_grid_bounds(height, yb, dsac::SCORE_GRID_MAX);
    std::vector<std::mt19937> g;
    for (int t = 0; t < T; t++) g.push_back(engine_from(state + (size_t)t * 625));
    for (int i = 0; i < n_images; i++) {
        auto next0 = [&]() { return (uint32_t)g[0](); };
        img[i] = (int32_t)dsac::lemire_draw((uint32_t)n_frames, next0);
        for (int sx = 0; sx < nx; sx++)
            for (int sy = 0; sy < ny; sy++) {
                const double x0 = sx ? xb[sx - 1] : 21.f, x1 = xb[sx], y0 = sy ? yb[sy - 1] : 21.f, y1 = yb[sy];
                const int cx = (int)dsac::uniform_real(dsac::canonical_draw(next0), x0, x1);
                const int cy = (int)dsac::uniform_real(dsac::canonical_draw(next0), y0, y1);
                if (sx < 40 && sy < 40) {
                    pix[((size_t)i * 1600 + sy * 40 + sx) * 2] = cx;
                    pix[((size_t)i * 1600 + sy * 40 + sx) * 2 + 1] = cy;
                }
            }
        for (int t = 0; t < T; t++) {
            auto next = [&]() { return (uint32_t)g[t](); };
            int h0, hc;
            dsac::stream_chunk(hyps, T, t, &h0, &hc);
            for (int h = h0; h < h0 + hc; h++) {
                const size_t k = (size_t)i * hyps + h;
                drift[k] = (int32_t)dsac::lemire_draw(2u, next);
                if (drift[k] == 0) dsac::score_rand_hyp(2.f, 2.f, next, noise + k * 6);
                else dsac::score_rand_hyp(10.f, 100.f, next, noise + k * 6);
            }
        }
    }
    for (int t = 0; t < T; t++) engine_to(g[t], state + (size_t)t * 625);
}

// normal_draw / uniform_real next to a fresh std::normal_distribution / std::uniform_real_distribution per call, each on
// its own std::mt19937(seed); returns 1 if both engines end in the same state
int shim_normal_vs_std(uint32_t seed, double stddev, int n, double* mine, double* theirs) {
    std::mt19937 a(seed), b(seed);
    auto next = [&]() { return (uint32_t)a(); };
    for (int i = 0; i < n; i++) {
        mine[i] = dsac::normal_draw(0.0, stddev, next);
        theirs[i] = ref_dgauss(b, stddev);
    }
    return a == b ? 1 : 0;
}
int shim_uniform_vs_std(uint32_t seed, double lo, double hi, int n, double* mine, double* theirs) {
    std::mt19937 a(seed), b(seed);
    auto next = [&]() { return (uint32_t)a(); };
    for (int i = 0; i < n; i++) {
        mine[i] = dsac::uniform_real(dsac::canonical_draw(next), lo, hi);
        std::uniform_real_distribution<double> d(lo, hi);
        theirs[i] = d(b);
    }
    return a == b ? 1 : 0;
}
// score_rand_hyp next to getRandHyp as the reference writes it (the draws as constructor arguments, evaluated in
// whatever order gcc chooses; the normalisation and the angle as Point3d arithmetic)
int shim_rand_hyp_vs_ref(uint32_t seed, float gauss_rot, float gauss_trans, int n, double* mine, double* theirs) {
    std::mt19937 a(seed), b(seed);
    auto next = [&]() { return (uint32_t)a(); };
    for (int i = 0; i < n; i++) {
        dsac::score_rand_hyp(gauss_rot, gauss_trans, next, mine + 6 * i);
        P3 trans(ref_dgauss(b, gauss_trans), ref_dgauss(b, gauss_trans), ref_dgauss(b, gauss_trans));
        P3 ax(ref_drand(b), ref_drand(b), ref_drand(b));
        const double s = 1.0 / std::sqrt((double)ax.x * ax.x + (double)ax.y * ax.y + (double)ax.z * ax.z);
        ax = P3(ax.x * s, ax.y * s, ax.z * s);
        const double g = ref_dgauss(b, gauss_rot);
        ax = P3(ax.x * g, ax.y * g, ax.z * g);
        const double k = 3.1415926 / 180.0;
        ax = P3(ax.x * k, ax.y * k, ax.z * k);
        double* o = theirs + 6 * i;
        o[0] = ax.x; o[1] = ax.y; o[2] = ax.z; o[3] = trans.x; o[4] = trans.y; o[5] = trans.z;
    }
    return a == b ? 1 : 0;
}
void shim_score_sample(const double* gt_jp, const double* v, double f, float temperature, float* P, double* label,
                       int32_t* correct) {
    dsac::ScoreSample s;
    dsac::score_sample(gt_jp, v, f, temperature, &s);
    for (int k = 0; k < 12; k++) P[k] = s.P[k];
    *label = s.label;
    *correct = s.correct;
}
int shim_grid_bounds(int size, float* bounds) { return dsac::score_grid_bounds(size, bounds, 1 << 20); }
}
