// rgbd_oracle.cpp -- test helper (tests/rgbd_oracle.py builds it): RGB-D localisation restated on the CPU in fp64, the
// reference the engine's RGB-D passes (dsac_set_cell_depth_device) are checked against.  It compiles the unmodified oracle
// sources into the same library (the flags of oracle/Makefile's parity build) and restates orc_forward with the P3P
// acceptance swapped for the Kabsch one and the LM refinement for the Kabsch refinement -- the same operations in the same
// order, on the oracle's own Frame / gather_set / orc_kabsch / minimal_set_ok helpers.  The candidate stream is the
// uniform MT19937 one of orc_forward (stream s of global frame g seeded with seed + g*T + s) or, with `cum`, the guided
// draw (the same Philox rule as guided_oracle.cpp).  No engine header is used.
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

void guided_draw(const uint32_t* cum, uint32_t seed, uint64_t z, uint32_t i, int cells[4]) {
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
        const int j = (int)(std::upper_bound(cum, cum + ORC_N, r) - cum);
        bool dup = false;
        for (int k = 0; k < n; k++) dup |= cells[k] == j;
        if (!dup) cells[n++] = j;
    }
}

bool has_depth(const double* eye, int c) { return eye[c * 3 + 2] > 0.0; }   // (NaN: no depth)

bool triangle_ok(const double P[9]) {
    const double a[3] = {P[3] - P[0], P[4] - P[1], P[5] - P[2]}, b[3] = {P[6] - P[0], P[7] - P[1], P[8] - P[2]};
    const double c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    return std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) >= 1.0;
}

// The RGB-D acceptance test of cells c4 (draw order); the hypothesis is (rodrigues(R), t) of the Kabsch fit of c0..c2.
bool accept(const Frame& fr, const double* eye, const int c4[4], int thr, double r[3], double t[3], int64_t* fragile) {
    for (int j = 0; j < 4; j++)
        if (!has_depth(eye, c4[j])) return false;
    double S[12], E[12];
    for (int j = 0; j < 4; j++)
        for (int k = 0; k < 3; k++) { S[j * 3 + k] = fr.coords[c4[j] * 3 + k]; E[j * 3 + k] = eye[c4[j] * 3 + k]; }
    if (!triangle_ok(S) || !triangle_ok(E)) return false;
    double R[9];
    orc_kabsch(3, S, E, R, t);
    for (int j = 0; j < 4; j++)
        if (!(R[6] * S[j * 3] + R[7] * S[j * 3 + 1] + R[8] * S[j * 3 + 2] + t[2] > 0.0)) return false;
    rodrigues_m2v(R, r);
    int32_t cells[8];
    for (int j = 0; j < 4; j++) { cells[j * 2] = c4[j] % ORC_GRID; cells[j * 2 + 1] = c4[j] / ORC_GRID; }
    float obj[12], img[8];
    gather_set(fr, cells, obj, img);
    return minimal_set_ok(obj, img, r, t, fr, thr, fragile);
}

// refine_loop with the selection restricted to cells with depth and the Kabsch fit (scene -> eye) as the pose update;
// the same two modes: generate the permutations (processImage) or replay n_perm_avail given ones (refine()).
int refine_rgbd(const orc_config& cfg, const Frame& fr, const double* eye, const int32_t* perm, int n_perm_avail, bool generate_perm,
                std::mt19937* randG, int32_t* perm_out, int* n_perm_steps, int32_t* inlier_map, double pose[6]) {
    std::vector<float> diff(ORC_N);
    orc_diff_map(fr.coords, fr.pix, pose, pose + 3, fr.f, fr.cx, fr.cy, diff.data());
    int done = 0;
    if (n_perm_steps) *n_perm_steps = 0;
    std::vector<int> idxs(ORC_N);
    std::vector<double> a, b;
    for (int rStep = 0; rStep < cfg.ref_steps; rStep++) {
        const int32_t* pp = nullptr;
        if (generate_perm) {
            for (int i = 0; i < ORC_N; i++) idxs[i] = i;
            std::shuffle(idxs.begin(), idxs.end(), *randG);
            if (perm_out)
                for (int i = 0; i < ORC_N; i++) perm_out[rStep * ORC_N + i] = idxs[i];
            if (n_perm_steps) (*n_perm_steps)++;
        } else {
            if (rStep >= n_perm_avail) break;
            pp = perm + rStep * ORC_N;
        }
        a.clear();
        b.clear();
        for (int k = 0; k < ORC_N; k++) {
            const int c = generate_perm ? idxs[k] : pp[k];
            if (diff[c] < (float)cfg.thr2d && has_depth(eye, c)) {
                for (int q = 0; q < 3; q++) { a.push_back(fr.coords[c * 3 + q]); b.push_back(eye[c * 3 + q]); }
                if (inlier_map) inlier_map[c] += 1;
            }
            if ((int)(a.size() / 3) >= cfg.inlier_count) break;
        }
        const int n = (int)(a.size() / 3);
        if (n < 50) break;
        double R[9], upd[6];
        orc_kabsch(n, a.data(), b.data(), R, upd + 3);
        rodrigues_m2v(R, upd);
        bool nan = false;
        for (int i = 0; i < 6; i++)
            if (upd[i] != upd[i]) nan = true;
        if (nan) break;
        std::memcpy(pose, upd, sizeof(upd));
        done++;
        orc_diff_map(fr.coords, fr.pix, pose, pose + 3, fr.f, fr.cx, fr.cy, diff.data());
    }
    return done;
}

// The uniform or guided draw of stream s of global frame g with the Kabsch acceptance: hypotheses rv / tv, img_idx, cand_idx
// (nullable), stream_ncand (nullable).  Returns -1 if a stream ran out, -2 for a frame with fewer than 4 cells with depth.
int sample_rgbd(const orc_config& cfg, const Frame& fr, const double* eye, const uint32_t* cum, int64_t g, double* rv, double* tv,
                int32_t* img_idx, int32_t* cand_idx, int64_t* stream_ncand, int64_t* n_candidates, int64_t* n_fragile,
                std::mt19937* gen0 = nullptr) {
    const int H = cfg.n_hyps, T = std::max(1, cfg.n_streams);
    int status = 0, have = 0;
    for (int c = 0; c < ORC_N; c++) have += has_depth(eye, c);
    for (int s = 0; s < T; s++) {
        int h0, cnt;
        stream_chunk(H, T, s, &h0, &cnt);
        std::mt19937 gen;
        gen.seed(cfg.seed + (uint32_t)(g * T + s));
        if (s == 0) gen.discard(cfg.stream_skip);
        std::vector<unsigned char> chosen(ORC_N, 0);
        const uint64_t z = (uint64_t)g * T + s;
        int64_t k = 0;
        if (stream_ncand) stream_ncand[s] = 0;
        for (int h = h0; h < h0 + cnt; h++) {
            for (;;) {
                if (have < 4 || (cfg.max_candidates > 0 && k >= cfg.max_candidates)) {
                    status = have < 4 ? -2 : -1;
                    for (int i = 0; i < 3; i++) rv[h * 3 + i] = tv[h * 3 + i] = 0;
                    for (int j = 0; j < 4; j++) img_idx[h * 4 + j] = -1;
                    if (cand_idx) cand_idx[h] = -1;
                    if (stream_ncand) stream_ncand[s] = k;
                    break;
                }
                int c4[4];
                if (cum) {
                    guided_draw(cum, cfg.seed, z, (uint32_t)k, c4);
                } else {
                    int32_t cells[8];
                    draw_candidate(gen, cells, chosen.data());
                    for (int j = 0; j < 4; j++) c4[j] = cells[j * 2 + 1] * ORC_GRID + cells[j * 2];
                }
                const int64_t this_k = k++;
                if (n_candidates) (*n_candidates)++;
                double r[3], t[3];
                if (!accept(fr, eye, c4, cfg.thr2d, r, t, n_fragile)) continue;
                for (int i = 0; i < 3; i++) { rv[h * 3 + i] = r[i]; tv[h * 3 + i] = t[i]; }
                for (int j = 0; j < 4; j++) img_idx[h * 4 + j] = c4[j];
                if (cand_idx) cand_idx[h] = (int32_t)this_k;
                if (stream_ncand) stream_ncand[s] = this_k + 1;
                break;
            }
        }
        if (s == 0 && gen0) *gen0 = gen;   // stream 0 as the sampling left it (guided: right after stream_skip)
    }
    return status;
}

// The 3-point Kabsch hypothesis of the (float) scene points obj[0..8] to eye points b, as a cv pose
void kabsch_pose(const float obj[9], const double b[9], double pose[6]) {
    double a[9], R[9];
    for (int k = 0; k < 9; k++) a[k] = obj[k];
    orc_kabsch(3, a, b, R, pose + 3);
    rodrigues_m2v(R, pose);
}

// dPNP with the Kabsch hypothesis: orc_dpnp's central differences (eps 0.1f, serial perturb / restore); the 4th point's
// columns are zero
void dkabsch(const float obj_in[12], const double b[9], double jac[72]) {
    float obj[12];
    std::memcpy(obj, obj_in, sizeof(obj));
    for (int k = 0; k < 72; k++) jac[k] = 0;
    const float eps = 0.1f;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double pose[6], fS[6], bS[6];
            obj[i * 3 + j] += eps;
            kabsch_pose(obj, b, pose);
            jp6_from_cv(pose, pose + 3, fS);
            obj[i * 3 + j] -= 2 * eps;
            kabsch_pose(obj, b, pose);
            jp6_from_cv(pose, pose + 3, bS);
            obj[i * 3 + j] += eps;
            bool nan = false;
            for (int k = 0; k < 6; k++) {
                double v = (fS[k] - bS[k]) / (2 * eps);
                jac[k * 12 + i * 3 + j] = v;
                if (v != v) nan = true;
            }
            if (nan) {
                for (int k = 0; k < 72; k++) jac[k] = 0;
                return;
            }
        }
}

void set_eye(const double* eye, const int32_t* idx, double b[9]) {
    for (int j = 0; j < 3; j++)
        for (int k = 0; k < 3; k++) b[j * 3 + k] = eye[idx[j] * 3 + k];
}

// dscore_accumulate with the hypothesis pose taken as sampled (the Kabsch fit) instead of re-solved by P3P
void dscore_rgbd(const orc_config& cfg, const Frame& fr, int H, const int32_t* img_idx, const double* hrv, const double* htv,
                 const std::vector<double>& sog, const std::vector<double>& dpnp_all, int fix_q4, std::vector<double>& row) {
    std::vector<float> diff(ORC_N);
    for (int h = 0; h < H; h++) {
        double R[9], tj[3];
        cv2our(hrv + h * 3, htv + h * 3, R, tj);
        orc_diff_map(fr.coords, fr.pix, hrv + h * 3, htv + h * 3, fr.f, fr.cx, fr.cy, diff.data());
        double go = sog[h];
        if (cfg.grad_clamp > 0) go = std::max(-cfg.grad_clamp, std::min(cfg.grad_clamp, go));
        const double* dHdO = &dpnp_all[(size_t)h * 72];
        double sp[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int x = 0; x < ORC_GRID; x++)
            for (int y = 0; y < ORC_GRID; y++) {
                int c = y * ORC_GRID + x;
                double sg = 1.0 / (1.0 + std::exp(-cfg.beta * ((double)cfg.thr2d - (double)diff[c])));
                double g = go * (-cfg.alpha * cfg.beta * sg * (1.0 - sg));
                float pt[2] = {(float)fr.pix[c * 2], (float)fr.pix[c * 2 + 1]};
                float ob[3] = {(float)fr.coords[c * 3], (float)fr.coords[c * 3 + 1], (float)fr.coords[c * 3 + 2]};
                double d3[3], d6[6];
                orc_dproject_dobj(pt, ob, R, tj, fr.f, fr.cx, fr.cy, d3);
                int col = fix_q4 ? (y * ORC_GRID + x) * 3 : (x * ORC_GRID + y) * 3;
                for (int k = 0; k < 3; k++) row[col + k] += g * d3[k];
                orc_dproject_dhyp(pt, ob, R, tj, fr.f, fr.cx, fr.cy, d6);
                for (int m = 0; m < 12; m++) {
                    double s = 0;
                    for (int k = 0; k < 6; k++) s += d6[k] * dHdO[k * 12 + m];
                    sp[m] += g * s;
                }
            }
        for (int i = 0; i < 4; i++) {
            const int cell = img_idx[h * 4 + i];
            if (cell < 0) continue;
            int x = cell % ORC_GRID, y = cell / ORC_GRID;
            int col = fix_q4 ? (y * ORC_GRID + x) * 3 : (x * ORC_GRID + y) * 3;
            for (int k = 0; k < 3; k++) row[col + k] += sp[i * 3 + k];
        }
    }
}

// the gathered float scene points of hypothesis h and their eye points (the dPNP inputs); false for an empty hypothesis
bool hyp_points(const Frame& fr, const double* eye, const int32_t* idx, float obj[12], double b[9]) {
    for (int j = 0; j < 4; j++)
        if (idx[j] < 0) return false;
    for (int j = 0; j < 4; j++)
        for (int k = 0; k < 3; k++) obj[j * 3 + k] = (float)fr.coords[idx[j] * 3 + k];
    set_eye(eye, idx, b);
    return true;
}

}  // namespace

extern "C" {

// eye [N][3]: ((u - cx) d / f, (v - cy) d / f, d) for finite d > 0, NaN otherwise; returns the cells with depth
int ror_eye(const int32_t* pix, const float* depth, double f, double cx, double cy, double* eye) {
    int have = 0;
    for (int c = 0; c < ORC_N; c++) {
        const float z = depth[c];
        if (std::isfinite(z) && z > 0.f) {
            const double Z = z;
            eye[c * 3] = ((double)pix[c * 2] - cx) * Z / f;
            eye[c * 3 + 1] = ((double)pix[c * 2 + 1] - cy) * Z / f;
            eye[c * 3 + 2] = Z;
            have++;
        } else {
            eye[c * 3] = eye[c * 3 + 1] = eye[c * 3 + 2] = NAN;
        }
    }
    return have;
}

int ror_accept(const orc_config* cfg, const int16_t* coords, const int32_t* pix, const double* eye, const int32_t cells[4],
               double r[3], double t[3], int64_t* fragile) {
    Frame fr{coords, pix, cfg->f, cfg->cx, cfg->cy};
    const int c4[4] = {cells[0], cells[1], cells[2], cells[3]};
    return accept(fr, eye, c4, cfg->thr2d, r, t, fragile) ? 1 : 0;
}

// orc_forward of global frame g as an RGB-D pass (cum: guided prefix sums, or null for the uniform MT19937 streams).
// stream_ncand [T].  Returns -1 if a stream ran out, -2 for a frame with fewer than 4 cells with depth (nothing sampled).
int ror_forward(const orc_config* cfgp, const uint32_t* cum, int64_t g, const int16_t* coords, const int32_t* pix, const double* eye,
                const double gt_R[9], const double gt_t[3], orc_forward_out* out, int64_t* stream_ncand) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> rv(H * 3, 0.0), tv(H * 3, 0.0);
    std::vector<int32_t> idx(H * 4);
    out->n_candidates = 0;
    out->n_fragile = 0;
    const int status = sample_rgbd(cfg, fr, eye, cum, g, rv.data(), tv.data(), idx.data(), out->cand_idx, stream_ncand,
                                   &out->n_candidates, &out->n_fragile);
    if (out->img_idx) std::memcpy(out->img_idx, idx.data(), H * 4 * sizeof(int32_t));
    if (out->hyp_rvec) std::memcpy(out->hyp_rvec, rv.data(), H * 3 * sizeof(double));
    if (out->hyp_tvec) std::memcpy(out->hyp_tvec, tv.data(), H * 3 * sizeof(double));

    // ---- scores, softmax and soft-argmax as orc_forward
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
    // ---- the Kabsch refinement of the average
    double ref[6];
    std::memcpy(ref, avg, sizeof(ref));
    std::vector<int32_t> imap(ORC_N, 0);
    if (out->pixel_idxs)
        for (int i = 0; i < cfg.ref_steps * ORC_N; i++) out->pixel_idxs[i] = -1;
    std::mt19937 randG;
    int n_perm = 0;
    out->ref_steps_done = refine_rgbd(cfg, fr, eye, nullptr, 0, true, &randG, out->pixel_idxs, &n_perm, imap.data(), ref);
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

// orc_forward_dsac of global frame g as an RGB-D pass (uniform streams): Kabsch hypotheses, the draw from MT19937 stream 0
// where the sampling left it, and every hypothesis refined by refine_rgbd.
int ror_forward_dsac(const orc_config* cfgp, int random_draw, int64_t g, const int16_t* coords, const int32_t* pix, const double* eye,
                     const double gt_R[9], const double gt_t[3], orc_dsac_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> rv(H * 3, 0.0), tv(H * 3, 0.0);
    std::vector<int32_t> idx(H * 4);
    std::mt19937 gen0;   // stream 0's generator survives the sampling loop and serves draw(), as in orc_forward_dsac
    const int status = sample_rgbd(cfg, fr, eye, nullptr, g, rv.data(), tv.data(), idx.data(), nullptr, nullptr, nullptr, nullptr, &gen0);
    std::vector<double> scores(H), sf(H);
    std::vector<float> dm(ORC_N);
    for (int h = 0; h < H; h++) {
        orc_diff_map(coords, pix, &rv[h * 3], &tv[h * 3], fr.f, fr.cx, fr.cy, dm.data());
        scores[h] = orc_soft_inlier_score(dm.data(), ORC_N, (double)cfg.thr2d, cfg.alpha, cfg.beta);
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
        int done = refine_rgbd(cfg, fr, eye, nullptr, 0, true, &randG, nullptr, &nperm, imap.data(), pose);
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

// orc_backward of an RGB-D pass: the refine() replays through refine_rgbd, dPNP through dkabsch, dScore on the sampled poses.
int ror_backward(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double* eye, const double gt_R[9],
                 const double gt_t[3], const orc_forward_out* fwd, orc_backward_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, N3 = ORC_N * 3;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> row(N3, 0.0);
    auto refine6 = [&](const int16_t* local, const double init[6], double out6[6]) {
        Frame lf{local, pix, cfg.f, cfg.cx, cfg.cy};
        double pose[6];
        std::memcpy(pose, init, sizeof(pose));
        refine_rgbd(cfg, lf, eye, fwd->pixel_idxs, fwd->n_perm_steps, false, nullptr, nullptr, nullptr, nullptr, pose);
        jp6_from_cv(pose, pose + 3, out6);
    };
    double ref6[6], gt6[6], dL[6];
    jp6_from_cv(fwd->ref, fwd->ref + 3, ref6);
    rodrigues_m2v(gt_R, gt6);
    gt6[3] = gt_t[0]; gt6[4] = gt_t[1]; gt6[5] = gt_t[2];
    orc_dloss_max(ref6, gt6, dL);
    std::memcpy(out->dloss_dref, dL, sizeof(dL));
    std::vector<double> dRefObj(6 * N3, 0.0);
    {
        std::vector<int16_t> local(coords, coords + N3);
        const float eps = 2.f;
        int inCount = 0;
        int skip = 1 / (float)cfg.sub_sample;
        for (int x = 0; x < ORC_GRID; x++)
            for (int y = 0; y < ORC_GRID; y++) {
                if (fwd->inlier_map[y * ORC_GRID + x] == 0) continue;
                inCount++;
                if (inCount % skip != 0) continue;
                for (int c = 0; c < 3; c++) {
                    int16_t& v = local[(y * ORC_GRID + x) * 3 + c];
                    double fS[6], bS[6];
                    v += eps;
                    refine6(local.data(), fwd->avg, fS);
                    v -= 2 * eps;
                    refine6(local.data(), fwd->avg, bS);
                    v += eps;
                    for (int k = 0; k < 6; k++) dRefObj[k * N3 + y * ORC_GRID * 3 + x * 3 + c] = (fS[k] - bS[k]) / (2 * eps) * skip;
                }
            }
    }
    if (out->dref_dobj) std::memcpy(out->dref_dobj, dRefObj.data(), 6 * N3 * sizeof(double));
    for (int c = 0; c < N3; c++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += dL[k] * dRefObj[k * N3 + c];
        row[c] += s;
    }
    double dRefHyp[36];
    {
        const float eps = 0.001f;
        double init[6];
        std::memcpy(init, fwd->avg, sizeof(init));
        for (int i = 0; i < 6; i++) {
            double fS[6], bS[6];
            const double e = i < 3 ? eps : eps * 1000;
            init[i] += e;
            refine6(coords, init, fS);
            init[i] -= 2 * e;
            refine6(coords, init, bS);
            init[i] += e;
            for (int k = 0; k < 3; k++) dRefHyp[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps);
            for (int k = 3; k < 6; k++) dRefHyp[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps * 1000);
        }
    }
    std::memcpy(out->dref_dhyp, dRefHyp, sizeof(dRefHyp));
    std::vector<double> dHyp(6 * N3, 0.0), dpnp_all((size_t)H * 72, 0.0);
    for (int h = 0; h < H; h++) {
        float obj[12];
        double b[9];
        double* J = &dpnp_all[(size_t)h * 72];
        if (!hyp_points(fr, eye, fwd->img_idx + h * 4, obj, b)) continue;
        dkabsch(obj, b, J);
        for (int i = 0; i < 4; i++)
            for (int k = 0; k < 6; k++)
                for (int c = 0; c < 3; c++) dHyp[k * N3 + fwd->img_idx[h * 4 + i] * 3 + c] += fwd->sf[h] * J[k * 12 + i * 3 + c];
    }
    if (out->dpnp) std::memcpy(out->dpnp, dpnp_all.data(), dpnp_all.size() * sizeof(double));
    double dLdAvg[6];
    for (int i = 0; i < 6; i++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += dL[k] * dRefHyp[k * 6 + i];
        dLdAvg[i] = s;
    }
    for (int c = 0; c < N3; c++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += dLdAvg[k] * dHyp[k * N3 + c];
        row[c] += s;
    }
    std::vector<double> sog(H, 0.0);
    for (int h = 0; h < H; h++) {
        double hf = 0;
        for (int i = 0; i < 3; i++) hf += dLdAvg[i] * fwd->hyp_rvec[h * 3 + i] + dLdAvg[3 + i] * (fwd->hyp_tvec[h * 3 + i] / 1000);
        sog[h] += fwd->sf[h] * hf;
        for (int j = 0; j < H; j++) sog[j] -= fwd->sf[h] * fwd->sf[j] * hf;
    }
    if (out->score_grads) std::memcpy(out->score_grads, sog.data(), H * sizeof(double));
    dscore_rgbd(cfg, fr, H, fwd->img_idx, fwd->hyp_rvec, fwd->hyp_tvec, sog, dpnp_all, cfg.fix_q4, row);
    std::memcpy(out->dloss_dobj, row.data(), N3 * sizeof(double));
    return 0;
}

// orc_backward_dsac of an RGB-D pass: path I's refine() starts from the Kabsch fit of the (perturbed) minimal set and
// replays refine_rgbd; path II through dkabsch and dScore on the sampled poses.
int ror_backward_dsac(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double* eye, const double gt_R[9],
                      const double gt_t[3], const orc_dsac_out* fwd, orc_backward_dsac_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, N3 = ORC_N * 3;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> p1(N3, 0.0), p2(N3, 0.0);
    double gt6[6];
    rodrigues_m2v(gt_R, gt6);
    gt6[3] = gt_t[0]; gt6[4] = gt_t[1]; gt6[5] = gt_t[2];
    std::vector<int32_t> perms((size_t)cfg.ref_steps * ORC_N);
    orc_refine_permutations(cfg.ref_steps, perms.data());
    int n_sel = 0, n_jobs = 0;
    const float eps = 2.f;
    const int skip = 1 / (float)cfg.sub_sample;
    auto refine_from_set = [&](const float obj[12], const double b[9], const int16_t* local, int n_perm, double out6[6]) {
        double pose[6];
        kabsch_pose(obj, b, pose);
        Frame lf{local, pix, cfg.f, cfg.cx, cfg.cy};
        refine_rgbd(cfg, lf, eye, perms.data(), n_perm, false, nullptr, nullptr, nullptr, nullptr, pose);
        jp6_from_cv(pose, pose + 3, out6);
        n_jobs++;
    };
    for (int h = 0; h < H; h++) {
        if (!(fwd->sf[h] > 0.0001)) continue;
        float obj[12];
        double b[9];
        if (!hyp_points(fr, eye, fwd->img_idx + h * 4, obj, b)) continue;
        n_sel++;
        std::vector<int32_t> imap(ORC_N, 0);
        int n_perm = 0;
        {
            double pose[6] = {fwd->hyp_rvec[h * 3], fwd->hyp_rvec[h * 3 + 1], fwd->hyp_rvec[h * 3 + 2],
                              fwd->hyp_tvec[h * 3], fwd->hyp_tvec[h * 3 + 1], fwd->hyp_tvec[h * 3 + 2]};
            std::mt19937 randG;
            refine_rgbd(cfg, fr, eye, nullptr, 0, true, &randG, nullptr, &n_perm, imap.data(), pose);
            for (int j = 0; j < 4; j++) imap[fwd->img_idx[h * 4 + j]] = 0;
        }
        std::vector<double> J((size_t)6 * N3, 0.0);
        std::vector<int16_t> local(coords, coords + N3);
        for (int pt = 0; pt < 3; pt++)
            for (int c = 0; c < 3; c++) {
                const int cell = fwd->img_idx[h * 4 + pt];
                int16_t& v = local[cell * 3 + c];
                double fS[6], bS[6];
                v += eps; obj[pt * 3 + c] += eps;
                refine_from_set(obj, b, local.data(), n_perm, fS);
                v -= 2 * eps; obj[pt * 3 + c] -= 2 * eps;
                refine_from_set(obj, b, local.data(), n_perm, bS);
                v += eps; obj[pt * 3 + c] += eps;
                for (int k = 0; k < 6; k++) J[(size_t)k * N3 + cell * 3 + c] = (fS[k] - bS[k]) / (2 * eps);
            }
        int inCount = 0;
        for (int x = 0; x < ORC_GRID; x++)
            for (int y = 0; y < ORC_GRID; y++) {
                if (imap[y * ORC_GRID + x] == 0) continue;
                inCount++;
                if (inCount % skip != 0) continue;
                for (int c = 0; c < 3; c++) {
                    int16_t& v = local[(y * ORC_GRID + x) * 3 + c];
                    double fS[6], bS[6];
                    v += eps;
                    refine_from_set(obj, b, local.data(), n_perm, fS);
                    v -= 2 * eps;
                    refine_from_set(obj, b, local.data(), n_perm, bS);
                    v += eps;
                    for (int k = 0; k < 6; k++) J[(size_t)k * N3 + (y * ORC_GRID + x) * 3 + c] = (fS[k] - bS[k]) / (2 * eps) * skip;
                }
            }
        double ref6[6], dL[6];
        jp6_from_cv(fwd->ref_pose + h * 6, fwd->ref_pose + h * 6 + 3, ref6);
        orc_dloss_max(ref6, gt6, dL);
        for (int col = 0; col < N3; col++) {
            double gg = 0;
            for (int k = 0; k < 6; k++) gg += dL[k] * J[(size_t)k * N3 + col];
            p1[col] += fwd->sf[h] * gg;
        }
    }
    std::vector<double> sog(H, 0.0), dpnp_all((size_t)H * 72, 0.0);
    for (int i = 0; i < H; i++) {
        sog[i] = fwd->sf[i] * fwd->losses[i];
        for (int j = 0; j < H; j++) sog[i] -= fwd->sf[i] * fwd->sf[j] * fwd->losses[j];
    }
    if (out->score_grads) std::memcpy(out->score_grads, sog.data(), H * sizeof(double));
    for (int h = 0; h < H; h++) {
        float obj[12];
        double b[9];
        if (hyp_points(fr, eye, fwd->img_idx + h * 4, obj, b)) dkabsch(obj, b, &dpnp_all[(size_t)h * 72]);
    }
    dscore_rgbd(cfg, fr, H, fwd->img_idx, fwd->hyp_rvec, fwd->hyp_tvec, sog, dpnp_all, 1, p2);
    for (int c = 0; c < N3; c++) out->dloss_dobj[c] = p1[c] + p2[c];
    if (out->path1) std::memcpy(out->path1, p1.data(), N3 * sizeof(double));
    if (out->path2) std::memcpy(out->path2, p2.data(), N3 * sizeof(double));
    out->n_selected = n_sel;
    out->n_refine_jobs = n_jobs;
    return 0;
}

}  // extern "C"
