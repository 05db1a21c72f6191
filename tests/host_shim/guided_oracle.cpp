// guided_oracle.cpp -- test helper (tests/guided_oracle.py builds it): guided sampling restated on the CPU in fp64, the
// reference the engine's guided passes (dsac_set_sampling_logits_device) are checked against.  It compiles the unmodified
// oracle sources into the same library (the flags of oracle/Makefile's parity build) and restates orc_forward with the
// candidate source swapped for the guided draw -- the same operations in the same order, on the oracle's own Frame /
// gather_set / solve_p3p / minimal_set_ok / refine helpers -- and likewise orc_forward_dsac; plus the weight table,
// Philox4x32-10, the draw rule, the log-probability of a pass's draw and its gradient.
#include "dsac_oracle.cpp"

namespace {

void philox(const uint32_t ctr[4], uint32_t k0, uint32_t k1, uint32_t out[4]) {
    uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
    for (int r = 0; r < 10; r++) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1;
        c[0] = n0; c[1] = (uint32_t)p1; c[2] = n2; c[3] = (uint32_t)p0;
    }
    for (int i = 0; i < 4; i++) out[i] = c[i];
}

// the four cells of candidate i of slot z, in draw order
void draw(const uint32_t* cum, uint32_t seed, uint64_t z, uint32_t i, int cells[4]) {
    const uint32_t Q = cum[ORC_N - 1];
    uint32_t buf[4], ctr[4] = {0u, i, (uint32_t)z, (uint32_t)(z >> 32)};
    int used = 4;
    auto word = [&]() {
        if (used == 4) { philox(ctr, seed, 0u, buf); ctr[0]++; used = 0; }
        return buf[used++];
    };
    int n = 0;
    while (n < 4) {
        uint64_t m = (uint64_t)word() * Q;
        if ((uint32_t)m < Q) {
            const uint32_t t = (0u - Q) % Q;
            while ((uint32_t)m < t) m = (uint64_t)word() * Q;
        }
        const uint32_t r = (uint32_t)(m >> 32);
        const int j = (int)(std::upper_bound(cum, cum + ORC_N, r) - cum);   // smallest j with C_j > r
        bool dup = false;
        for (int k = 0; k < n; k++) dup |= cells[k] == j;
        if (!dup) cells[n++] = j;
    }
}

}  // namespace

extern "C" {

void gor_philox(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) { philox(ctr, key[0], key[1], out); }

void gor_draw(const uint32_t* cum, uint32_t seed, uint64_t z, uint32_t i, int32_t cells[4]) {
    int c[4];
    draw(cum, seed, z, i, c);
    for (int k = 0; k < 4; k++) cells[k] = c[k];
}

// w = softmax(logits) in fp64, q = floor(w 2^31), cum = inclusive prefix sums; returns 1 for DSAC_ST_BAD_WEIGHTS
int gor_table(const float* logits, double* w, uint32_t* q, uint32_t* cum) {
    double mx = -INFINITY;
    bool nonfinite = false;
    for (int k = 0; k < ORC_N; k++) {
        if (std::isnan(logits[k]) || logits[k] == INFINITY) nonfinite = true;
        else mx = std::max(mx, (double)logits[k]);
    }
    const bool usable = !nonfinite && mx > -INFINITY;
    double s = 0;
    if (usable)
        for (int k = 0; k < ORC_N; k++) s += std::exp((double)logits[k] - mx);
    uint32_t c = 0;
    int pos = 0;
    for (int k = 0; k < ORC_N; k++) {
        w[k] = usable ? std::exp((double)logits[k] - mx) / s : 0.0;
        q[k] = (uint32_t)std::floor(w[k] * 2147483648.0);
        c += q[k];
        pos += q[k] > 0;
        cum[k] = c;
    }
    return (!usable || pos < 4) ? 1 : 0;
}

// orc_forward with the guided draw (frame g of the pass; the candidate index is the slot's counter).  stream_ncand [T]:
// the used candidates of every stream.  Returns -1 if a stream ran out (DSAC_ST_SAMPLER_EXHAUSTED).
int gor_forward(const orc_config* cfgp, const uint32_t* cum, int64_t g, const int16_t* coords, const int32_t* pix, const double gt_R[9],
                const double gt_t[3], orc_forward_out* out, int64_t* stream_ncand) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, T = std::max(1, cfg.n_streams);
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> rv(H * 3), tv(H * 3);
    out->n_candidates = 0;
    out->n_fragile = 0;
    int status = 0;
    for (int s = 0; s < T; s++) {
        int h0, cnt;
        stream_chunk(H, T, s, &h0, &cnt);
        const uint64_t z = (uint64_t)g * T + s;
        int64_t k = 0;
        stream_ncand[s] = 0;
        for (int h = h0; h < h0 + cnt; h++) {
            for (;;) {
                if (cfg.max_candidates > 0 && k >= cfg.max_candidates) {
                    status = -1;
                    for (int i = 0; i < 3; i++) rv[h * 3 + i] = tv[h * 3 + i] = 0;
                    if (out->img_idx)
                        for (int j = 0; j < 4; j++) out->img_idx[h * 4 + j] = -1;
                    if (out->cand_idx) out->cand_idx[h] = -1;
                    stream_ncand[s] = k;
                    break;
                }
                int c4[4];
                draw(cum, cfg.seed, z, (uint32_t)k, c4);
                int32_t cells[8];
                for (int j = 0; j < 4; j++) { cells[j * 2] = c4[j] % ORC_GRID; cells[j * 2 + 1] = c4[j] / ORC_GRID; }
                int64_t this_k = k++;
                out->n_candidates++;
                float obj[12], img[8];
                gather_set(fr, cells, obj, img);
                double r[3], t[3];
                if (!solve_p3p(obj, img, fr.f, fr.cx, fr.cy, r, t)) continue;
                if (!minimal_set_ok(obj, img, r, t, fr, cfg.thr2d, &out->n_fragile)) continue;
                for (int i = 0; i < 3; i++) {
                    rv[h * 3 + i] = r[i];
                    tv[h * 3 + i] = t[i];
                }
                if (out->img_idx)
                    for (int j = 0; j < 4; j++) out->img_idx[h * 4 + j] = c4[j];
                if (out->cand_idx) out->cand_idx[h] = (int32_t)this_k;
                stream_ncand[s] = this_k + 1;
                break;
            }
        }
    }
    if (out->hyp_rvec) std::memcpy(out->hyp_rvec, rv.data(), H * 3 * sizeof(double));
    if (out->hyp_tvec) std::memcpy(out->hyp_tvec, tv.data(), H * 3 * sizeof(double));

    // ---- from here on orc_forward unchanged: scores, softmax, soft-argmax, refinement, evaluation
    std::vector<double> scores(H), sf(H);
    std::vector<float> dm(ORC_N);
    for (int h = 0; h < H; h++) {
        float* d = out->diffmaps ? out->diffmaps + (size_t)h * ORC_N : dm.data();
        orc_diff_map(coords, pix, &rv[h * 3], &tv[h * 3], fr.f, fr.cx, fr.cy, d);
        scores[h] = orc_soft_inlier_score(d, ORC_N, (double)cfg.thr2d, cfg.alpha, cfg.beta);
    }
    orc_softmax(scores.data(), H, sf.data());
    out->entropy = orc_entropy(sf.data(), H);
    double avg[6] = {0, 0, 0, 0, 0, 0};
    for (int h = 0; h < H; h++)
        for (int i = 0; i < 3; i++) {
            if (h == 0) {
                avg[i] = sf[h] * rv[h * 3 + i];
                avg[3 + i] = sf[h] * tv[h * 3 + i];
            } else {
                avg[i] += sf[h] * rv[h * 3 + i];
                avg[3 + i] += sf[h] * tv[h * 3 + i];
            }
        }
    if (out->scores) std::memcpy(out->scores, scores.data(), H * sizeof(double));
    if (out->sf) std::memcpy(out->sf, sf.data(), H * sizeof(double));
    std::memcpy(out->avg, avg, sizeof(avg));
    double ref[6];
    std::memcpy(ref, avg, sizeof(ref));
    std::vector<int32_t> imap(ORC_N, 0);
    if (out->pixel_idxs)
        for (int i = 0; i < cfg.ref_steps * ORC_N; i++) out->pixel_idxs[i] = -1;
    std::mt19937 randG;
    int n_perm = 0;
    out->ref_steps_done = refine_loop(cfg, fr, nullptr, 0, true, &randG, out->pixel_idxs, &n_perm, imap.data(), ref);
    out->n_perm_steps = n_perm;
    std::memcpy(out->ref, ref, sizeof(ref));
    if (out->inlier_map) std::memcpy(out->inlier_map, imap.data(), ORC_N * sizeof(int32_t));
    out->loss = out->rot_err = out->t_err = 0;
    out->correct = 0;
    if (gt_R && gt_t) {
        double eR[9], et[3];
        cv2our(ref, ref + 3, eR, et);
        out->loss = max_loss(gt_R, gt_t, eR, et, &out->rot_err, &out->t_err);
        out->correct = (out->rot_err < 5 && out->t_err < 50) ? 1 : 0;
    }
    return status;
}

// orc_forward_dsac with the guided draw (frame g of the pass).  The random draw reads MT19937 stream 0 of frame g
// (seed + g*T) right after stream_skip: the guided sampling consumes none of it.
int gor_forward_dsac(const orc_config* cfgp, int random_draw, const uint32_t* cum, int64_t g, const int16_t* coords, const int32_t* pix,
                     const double gt_R[9], const double gt_t[3], orc_dsac_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, T = std::max(1, cfg.n_streams);
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> rv(H * 3), tv(H * 3);
    std::vector<int32_t> idx(H * 4);
    std::mt19937 gen0;
    gen0.seed(cfg.seed + (uint32_t)(g * T));
    gen0.discard(cfg.stream_skip);
    int status = 0;
    out->stream0_endpos = cfg.stream_skip;
    for (int s = 0; s < T; s++) {
        int h0, cnt;
        stream_chunk(H, T, s, &h0, &cnt);
        const uint64_t z = (uint64_t)g * T + s;
        int64_t k = 0;
        for (int h = h0; h < h0 + cnt; h++) {
            for (;;) {
                if (cfg.max_candidates > 0 && k >= cfg.max_candidates) {
                    status = -1;
                    for (int i = 0; i < 3; i++) rv[h * 3 + i] = tv[h * 3 + i] = 0;
                    for (int j = 0; j < 4; j++) idx[h * 4 + j] = -1;
                    break;
                }
                int c4[4];
                draw(cum, cfg.seed, z, (uint32_t)k, c4);
                int32_t cells[8];
                for (int j = 0; j < 4; j++) { cells[j * 2] = c4[j] % ORC_GRID; cells[j * 2 + 1] = c4[j] / ORC_GRID; }
                k++;
                float obj[12], img[8];
                gather_set(fr, cells, obj, img);
                double r[3], t[3];
                if (!solve_p3p(obj, img, fr.f, fr.cx, fr.cy, r, t)) continue;
                if (!minimal_set_ok(obj, img, r, t, fr, cfg.thr2d, nullptr)) continue;
                for (int i = 0; i < 3; i++) { rv[h * 3 + i] = r[i]; tv[h * 3 + i] = t[i]; }
                for (int j = 0; j < 4; j++) idx[h * 4 + j] = c4[j];
                break;
            }
        }
    }
    // ---- from here on orc_forward_dsac unchanged: scores, softmax, entropy, draw, refinement of every hypothesis, losses
    std::vector<double> scores(H), sf(H);
    std::vector<std::vector<float>> dms(H, std::vector<float>(ORC_N));
    for (int h = 0; h < H; h++) {
        orc_diff_map(coords, pix, &rv[h * 3], &tv[h * 3], fr.f, fr.cx, fr.cy, dms[h].data());
        scores[h] = orc_soft_inlier_score(dms[h].data(), ORC_N, (double)cfg.thr2d, cfg.alpha, cfg.beta);
    }
    orc_softmax(scores.data(), H, sf.data());
    out->entropy = orc_entropy(sf.data(), H);
    {
        std::vector<std::pair<double, int>> cum_sf;
        double probSum = 0, maxProb = -1;
        int maxIdx = 0;
        for (int i = 0; i < H; i++) {
            if (sf[i] < kEps) continue;
            probSum += sf[i];
            cum_sf.push_back({probSum, i});
            if (maxProb < 0 || sf[i] > maxProb) { maxProb = sf[i]; maxIdx = i; }
        }
        if (random_draw) {
            std::uniform_real_distribution<double> d(0, probSum);
            double u = d(gen0);
            int pick = cum_sf.empty() ? 0 : cum_sf.back().second;
            for (auto& c : cum_sf)
                if (c.first > u) { pick = c.second; break; }
            out->hyp_idx = pick;
        } else {
            out->hyp_idx = maxIdx;
        }
    }
    double expected = 0;
    for (int h = 0; h < H; h++) {
        double pose[6] = {rv[h * 3], rv[h * 3 + 1], rv[h * 3 + 2], tv[h * 3], tv[h * 3 + 1], tv[h * 3 + 2]};
        std::vector<int32_t> imap(ORC_N, 0);
        std::mt19937 randG;
        int nperm = 0;
        int done = refine_loop(cfg, fr, nullptr, 0, true, &randG, nullptr, &nperm, imap.data(), pose);
        for (int j = 0; j < 4; j++)
            if (idx[h * 4 + j] >= 0) imap[idx[h * 4 + j]] = 0;
        if (out->inlier_maps) std::memcpy(out->inlier_maps + (size_t)h * ORC_N, imap.data(), ORC_N * sizeof(int32_t));
        if (out->steps_done) out->steps_done[h] = done;
        if (out->ref_pose) std::memcpy(out->ref_pose + h * 6, pose, sizeof(pose));
        double eR[9], et[3], re, te;
        cv2our(pose, pose + 3, eR, et);
        double l = (gt_R && gt_t) ? max_loss(gt_R, gt_t, eR, et, &re, &te) : 0.0;
        if (out->losses) out->losses[h] = l;
        expected += sf[h] * l;
        if (h == out->hyp_idx) {
            out->rot_err = (gt_R && gt_t) ? re : 0;
            out->t_err = (gt_R && gt_t) ? te : 0;
            out->correct = (gt_R && gt_t && re < 5 && te < 50) ? 1 : 0;
        }
    }
    out->expected_loss = expected;
    if (out->hyp_rvec) std::memcpy(out->hyp_rvec, rv.data(), H * 3 * sizeof(double));
    if (out->hyp_tvec) std::memcpy(out->hyp_tvec, tv.data(), H * 3 * sizeof(double));
    if (out->img_idx) std::memcpy(out->img_idx, idx.data(), H * 4 * sizeof(int32_t));
    if (out->sf) std::memcpy(out->sf, sf.data(), H * sizeof(double));
    return status;
}

// Log-probability of the used candidates of one frame (stream s: candidates 0 .. stream_ncand[s] - 1) and, if grad is
// not null, its gradient with respect to the logits, both in fp64 from the continuous w.
double gor_log_prob(const double* w, const uint32_t* cum, int T, uint32_t seed, int64_t g, const int64_t* stream_ncand, double* grad) {
    double lp = 0, A = 0;
    int64_t M = 0;
    std::vector<double> B(ORC_N, 0.0), cnt(ORC_N, 0.0);
    for (int s = 0; s < T; s++) {
        const uint64_t z = (uint64_t)g * T + s;
        M += stream_ncand[s];
        for (int64_t i = 0; i < stream_ncand[s]; i++) {
            int c[4];
            draw(cum, seed, z, (uint32_t)i, c);
            double S = 0;
            for (int k = 0; k < 4; k++) {
                const double R = 1.0 - S;
                lp += std::log(w[c[k]]) - std::log(R);
                A += S / R;
                for (int j = 0; j < k; j++) B[c[j]] += 1.0 / R;
                cnt[c[k]] += 1;
                S += w[c[k]];
            }
        }
    }
    if (grad)
        for (int j = 0; j < ORC_N; j++) grad[j] = cnt[j] - w[j] * (4.0 * (double)M + A) + w[j] * B[j];
    return lp;
}

}  // extern "C"
