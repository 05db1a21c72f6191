// guided_rng.cuh -- the random numbers and the draw rule of guided sampling (dsac_set_sampling_logits_device).
//
// Every candidate of every (frame, stream) slot has its own counter-based stream: Philox4x32-10 with key (seed, 0) and,
// for block b of candidate i of slot z = g * T + s (g: global frame index), counter (b, i, lo32(z), hi32(z)).  Each block
// gives four 32-bit words, used in order.  A candidate therefore does not depend on any other candidate: the generator
// draws one candidate per thread, and the log-probability kernel regenerates a candidate from its index alone.
#pragma once
#include <stdint.h>

#include "pose_math.cuh"

namespace dsac {

constexpr uint32_t GUIDED_ONE = 1u << 31;   // q_j = floor(w_j * 2^31)

DSAC_HD uint32_t philox_mulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }

// Philox4x32-10 (Salmon et al., SC 2011; the Random123 reference): ten rounds, the key bumped between rounds.
DSAC_HD void philox4x32_10(const uint32_t ctr_in[4], uint32_t k0, uint32_t k1, uint32_t out[4]) {
    uint32_t c0 = ctr_in[0], c1 = ctr_in[1], c2 = ctr_in[2], c3 = ctr_in[3];
    for (int r = 0; r < 10; r++) {
        if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = philox_mulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = philox_mulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// The word sequence of one candidate.
struct GuidedWords {
    uint32_t ctr[4], key, buf[4];
    int k;
    DSAC_HD GuidedWords(uint32_t seed, unsigned long long z, uint32_t i) : key(seed), k(4) {
        ctr[0] = 0u; ctr[1] = i; ctr[2] = (uint32_t)z; ctr[3] = (uint32_t)(z >> 32);
    }
    DSAC_HD uint32_t next() {
        if (k == 4) {
            philox4x32_10(ctr, key, 0u, buf);
            ctr[0]++;
            k = 0;
        }
        return buf[k++];
    }
};

// Four distinct cells of one candidate, in draw order.  cum: the frame's inclusive prefix sums C_j of the integer weights,
// Q = cum[N - 1].  Each point: r uniform in [0, Q) by Lemire's multiply-shift (a low half below 2^32 mod Q is re-drawn),
// the cell is the smallest j with C_j > r, and a cell the candidate already holds is drawn again (the reference's
// alreadyChosen rule), so cell j comes with probability q_j / (Q - sum of the q of the cells drawn before).
template <typename CumPtr>
DSAC_HD void guided_draw(CumPtr cum, uint32_t seed, unsigned long long z, uint32_t i, int cells[4]) {
    const uint32_t Q = cum[DSAC_N_CONST - 1];
    const uint32_t thr = (0u - Q) % Q;
    GuidedWords g(seed, z, i);
    int n = 0;
    while (n < 4) {
        uint64_t m = (uint64_t)g.next() * Q;
        while ((uint32_t)m < thr) m = (uint64_t)g.next() * Q;
        const uint32_t r = (uint32_t)(m >> 32);
        int lo = 0, hi = DSAC_N_CONST - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cum[mid] > r) hi = mid;
            else lo = mid + 1;
        }
        bool dup = false;
        for (int j = 0; j < n; j++) dup |= cells[j] == lo;
        if (!dup) cells[n++] = lo;
    }
}

}  // namespace dsac
