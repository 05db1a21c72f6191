// Host build of k_dsac_draw's arithmetic (dsac_b200/csrc/train.cuh with DSAC_HOST_ONLY) next to the libstdc++ calls it
// reproduces, for tests/test_train_draw.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include <cstring>
#include <random>
#include <vector>

#include "../../dsac_b200/csrc/train.cuh"

namespace {
// Words endpos and endpos + 1 of mt19937(seed) the way k_dsac_draw gets them: the state regenerated block by block with
// mt_regenerate_words into the other half of a double buffer, the words taken from the blocks draw_word_blocks names.
void product_words(uint32_t seed, unsigned long long endpos, uint32_t w[2]) {
    static uint32_t st[2][dsac::MT_N];
    dsac::mt_seed(st[0], seed);
    unsigned long long b0, b1;
    int i0, i1;
    dsac::draw_word_blocks(endpos, &b0, &i0, &b1, &i1);
    int cur = 0;
    for (unsigned long long b = 0; b <= b1; b++) {
        for (int t = 0; t < dsac::MT_N - dsac::MT_M; t++) {
            uint32_t x[3];
            const int m = dsac::mt_regenerate_words(st[cur], t, x);
            for (int k = 0; k < m; k++) st[cur ^ 1][t + k * (dsac::MT_N - dsac::MT_M)] = x[k];
        }
        cur ^= 1;
        if (b == b0) w[0] = dsac::mt_temper(st[cur][i0]);
        if (b == b1) w[1] = dsac::mt_temper(st[cur][i1]);
    }
}

// A generator that returns two given words: feeds chosen words to std::uniform_real_distribution.
struct TwoWords {
    using result_type = uint32_t;
    uint32_t w[2];
    int i = 0;
    static constexpr result_type min() { return 0; }
    static constexpr result_type max() { return 0xffffffffu; }
    result_type operator()() { return w[i++]; }
};

// The draw as the engine's host code computed it: libstdc++ draws u, the first cumulative sum above u wins.
template <class G> int std_pick(const double* p, int H, int random_draw, G& gen, double* u_out) {
    double probSum = 0, maxProb = -1;
    int maxIdx = 0, pick = 0;
    for (int i = 0; i < H; i++) {
        if (p[i] < 1e-8) continue;
        probSum += p[i];
        if (maxProb < 0 || p[i] > maxProb) { maxProb = p[i]; maxIdx = i; }
    }
    if (!random_draw) { *u_out = 0; return maxIdx; }
    std::uniform_real_distribution<double> dist(0, probSum);
    const double u = dist(gen);
    *u_out = u;
    double cum = 0;
    for (int i = 0; i < H; i++) {
        if (p[i] < 1e-8) continue;
        cum += p[i];
        pick = i;
        if (cum > u) break;
    }
    return pick;
}
}  // namespace

extern "C" {
// Per case c: the product's pick from mt19937(seeds[c]) after endpos[c] words, and std::mt19937 + discard + the engine's
// former host draw.
void shim_draw_cases(int n, int H, const double* sf, const uint32_t* seeds, const unsigned long long* endpos, int random_draw,
                     int32_t* pick_product, int32_t* pick_std, uint32_t* words_product, uint32_t* words_std) {
    for (int c = 0; c < n; c++) {
        const double* p = sf + (size_t)c * H;
        uint32_t w[2] = {0, 0};
        if (random_draw) product_words(seeds[c], endpos[c], w);
        pick_product[c] = dsac::draw_pick(p, H, random_draw, random_draw ? dsac::canonical53(w[0], w[1]) : 0.0);
        std::mt19937 gen(seeds[c]);
        gen.discard(endpos[c]);
        std::mt19937 peek = gen;
        words_product[2 * c] = w[0]; words_product[2 * c + 1] = w[1];
        words_std[2 * c] = peek(); words_std[2 * c + 1] = peek();
        double u;
        pick_std[c] = std_pick(p, H, random_draw, gen, &u);
    }
}

// One draw from given words: the product's u and pick against libstdc++'s (u next to probSum when the words are large).
void shim_draw_words(int H, const double* sf, uint32_t w0, uint32_t w1, double* u_product, double* u_std, int32_t* pick_product,
                     int32_t* pick_std) {
    double probSum = 0;
    for (int i = 0; i < H; i++)
        if (sf[i] >= 1e-8) probSum += sf[i];
    const double canon = dsac::canonical53(w0, w1);
    *u_product = canon * probSum + 0.0;
    *pick_product = dsac::draw_pick(sf, H, 1, canon);
    TwoWords g{{w0, w1}};
    *pick_std = std_pick(sf, H, 1, g, u_std);
}
}
