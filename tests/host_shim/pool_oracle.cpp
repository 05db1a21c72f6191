// pool_oracle.cpp -- test helper (tests/pool_oracle.py builds it): the oracle's soft-argmax and DSAC-variant pipelines and
// both backward passes from a GIVEN hypothesis pool instead of the sampler's, for the pose priors of
// dsac_set_pose_priors_device.  It compiles the unmodified oracle sources into the same library (with the flags of the
// oracle's parity build) and restates the stages after sampling in orc_forward / orc_forward_dsac / orc_backward /
// orc_backward_dsac's order, so that on the sampler's own pool it gives their results bit for bit
// (tests/test_pool_oracle_host.py).  A hypothesis without a minimal set (img_idx -1: a pose prior, or an exhausted slot)
// is a constant of the backward passes:
//   - its dPNP is zero and it scatters nothing to support cells;
//   - its score is differentiated through the coordinates at its own pose (a sampled hypothesis' pose is re-solved by P3P
//     from its set, as the oracle does);
//   - in the DSAC variant a selected prior (slot >= H - n_prior) refines from its own pose, has no minimal-set jobs and no
//     excluded support cells; an exhausted slot is not selected.
#include "dsac_oracle.cpp"

namespace {

void pool_dscore_accumulate(const orc_config& cfg, const Frame& fr, const int16_t* coords, const int32_t* pix, int H,
                            const int32_t* img_idx, const double* hyp_rvec, const double* hyp_tvec, const std::vector<double>& sog,
                            const std::vector<double>& dpnp_all, int fix_q4, std::vector<double>& row) {
    std::vector<float> diff(ORC_N);
    for (int h = 0; h < H; h++) {
        const bool has_set = img_idx[h * 4] >= 0;
        float obj[12], img[8];
        int32_t cells[8];
        double r[3], t[3], R[9], tj[3];
        if (has_set) {
            for (int j = 0; j < 4; j++) {
                cells[j * 2] = img_idx[h * 4 + j] % ORC_GRID;
                cells[j * 2 + 1] = img_idx[h * 4 + j] / ORC_GRID;
            }
            gather_set(fr, cells, obj, img);
            orc_solve_p3p(obj, img, fr.f, fr.cx, fr.cy, r, t);
        } else {
            for (int i = 0; i < 3; i++) { r[i] = hyp_rvec[h * 3 + i]; t[i] = hyp_tvec[h * 3 + i]; }
        }
        cv2our(r, t, R, tj);
        orc_diff_map(coords, pix, r, t, fr.f, fr.cx, fr.cy, diff.data());
        double go = sog[h];
        if (cfg.grad_clamp > 0) go = std::max(-cfg.grad_clamp, std::min(cfg.grad_clamp, go));
        const double* dHdO = &dpnp_all[(size_t)h * 72];
        double sp[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int x = 0; x < ORC_GRID; x++)
            for (int y = 0; y < ORC_GRID; y++) {
                int c = y * ORC_GRID + x;
                double sg = 1.0 / (1.0 + std::exp(-cfg.beta * ((double)cfg.thr2d - (double)diff[c])));
                double g = go * (-cfg.alpha * cfg.beta * sg * (1.0 - sg));
                float pt[2] = {(float)pix[c * 2], (float)pix[c * 2 + 1]};
                float ob[3] = {(float)coords[c * 3], (float)coords[c * 3 + 1], (float)coords[c * 3 + 2]};
                double d3[3], d6[6];
                orc_dproject_dobj(pt, ob, R, tj, fr.f, fr.cx, fr.cy, d3);
                int col = fix_q4 ? (y * ORC_GRID + x) * 3 : (x * ORC_GRID + y) * 3;
                for (int k = 0; k < 3; k++) row[col + k] += g * d3[k];
                if (!has_set) continue;
                orc_dproject_dhyp(pt, ob, R, tj, fr.f, fr.cx, fr.cy, d6);
                for (int m = 0; m < 12; m++) {
                    double s = 0;
                    for (int k = 0; k < 6; k++) s += d6[k] * dHdO[k * 12 + m];
                    sp[m] += g * s;
                }
            }
        if (!has_set) continue;
        for (int i = 0; i < 4; i++) {
            int x = cells[i * 2], y = cells[i * 2 + 1];
            int col = fix_q4 ? (y * ORC_GRID + x) * 3 : (x * ORC_GRID + y) * 3;
            for (int k = 0; k < 3; k++) row[col + k] += sp[i * 3 + k];
        }
    }
}

// dPNP of every hypothesis, zero without a minimal set
void pool_dpnp(const Frame& fr, int H, const int32_t* img_idx, std::vector<double>& dpnp_all) {
    for (int h = 0; h < H; h++) {
        double* J = &dpnp_all[(size_t)h * 72];
        if (img_idx[h * 4] < 0) {
            for (int k = 0; k < 72; k++) J[k] = 0;
            continue;
        }
        float obj[12], img[8];
        int32_t cells[8];
        for (int j = 0; j < 4; j++) {
            cells[j * 2] = img_idx[h * 4 + j] % ORC_GRID;
            cells[j * 2 + 1] = img_idx[h * 4 + j] / ORC_GRID;
        }
        gather_set(fr, cells, obj, img);
        orc_dpnp(obj, img, fr.f, fr.cx, fr.cy, J);
    }
}

}  // namespace

extern "C" {

// Soft-argmax forward (cnn_softam.h:1065-1179) of the pool out->hyp_rvec / hyp_tvec [H][3] (inputs): scores, sf, entropy,
// avg, the refinement of the average and its evaluation, as orc_forward computes them after its sampling loop.
int por_forward(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double gt_R[9], const double gt_t[3],
                orc_forward_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> rv(out->hyp_rvec, out->hyp_rvec + H * 3), tv(out->hyp_tvec, out->hyp_tvec + H * 3);
    out->n_candidates = 0;
    out->n_fragile = 0;
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
    return 0;
}

// DSAC-variant forward (cnn.h:1133-1228) of the pool out->hyp_rvec / hyp_tvec / img_idx (inputs), with the arg-max draw.
int por_forward_dsac(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double gt_R[9],
                     const double gt_t[3], orc_dsac_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    const double* rv = out->hyp_rvec;
    const double* tv = out->hyp_tvec;
    const int32_t* idx = out->img_idx;
    out->stream0_endpos = 0;
    std::vector<double> scores(H), sf(H);
    std::vector<float> dmap(ORC_N);
    for (int h = 0; h < H; h++) {
        orc_diff_map(coords, pix, &rv[h * 3], &tv[h * 3], fr.f, fr.cx, fr.cy, dmap.data());
        scores[h] = orc_soft_inlier_score(dmap.data(), ORC_N, (double)cfg.thr2d, cfg.alpha, cfg.beta);
    }
    orc_softmax(scores.data(), H, sf.data());
    out->entropy = orc_entropy(sf.data(), H);
    {
        double maxProb = -1;
        int maxIdx = 0;
        for (int i = 0; i < H; i++) {
            if (sf[i] < kEps) continue;
            if (maxProb < 0 || sf[i] > maxProb) { maxProb = sf[i]; maxIdx = i; }
        }
        out->hyp_idx = maxIdx;
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
    if (out->sf) std::memcpy(out->sf, sf.data(), H * sizeof(double));
    return 0;
}

// Soft-argmax backward (train_ransac_softam.cpp:288-394) of a por_forward / orc_forward result.
int por_backward(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double gt_R[9], const double gt_t[3],
                 const orc_forward_out* fwd, orc_backward_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, N3 = ORC_N * 3;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> row(N3, 0.0);
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
                    orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, local.data(), pix, fwd->avg, fS);
                    v -= 2 * eps;
                    orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, local.data(), pix, fwd->avg, bS);
                    v += eps;
                    for (int k = 0; k < 6; k++)
                        dRefObj[k * N3 + y * ORC_GRID * 3 + x * 3 + c] = (fS[k] - bS[k]) / (2 * eps) * skip;
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
            if (i < 3) {
                init[i] += eps;
                orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, coords, pix, init, fS);
                init[i] -= 2 * eps;
                orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, coords, pix, init, bS);
                init[i] += eps;
            } else {
                init[i] += eps * 1000;
                orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, coords, pix, init, fS);
                init[i] -= 2 * eps * 1000;
                orc_refine(cfgp, fwd->pixel_idxs, fwd->n_perm_steps, coords, pix, init, bS);
                init[i] += eps * 1000;
            }
            for (int k = 0; k < 3; k++) dRefHyp[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps);
            for (int k = 3; k < 6; k++) dRefHyp[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps * 1000);
        }
    }
    std::memcpy(out->dref_dhyp, dRefHyp, sizeof(dRefHyp));
    std::vector<double> dHyp(6 * N3, 0.0), dpnp_all((size_t)H * 72);
    pool_dpnp(fr, H, fwd->img_idx, dpnp_all);
    for (int h = 0; h < H; h++) {
        if (fwd->img_idx[h * 4] < 0) continue;
        const double* J = &dpnp_all[(size_t)h * 72];
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
    pool_dscore_accumulate(cfg, fr, coords, pix, H, fwd->img_idx, fwd->hyp_rvec, fwd->hyp_tvec, sog, dpnp_all, cfg.fix_q4, row);
    std::memcpy(out->dloss_dobj, row.data(), N3 * sizeof(double));
    return 0;
}

// DSAC-variant backward (train_ransac.cpp:304-381) of a por_forward_dsac / orc_forward_dsac result whose last n_prior slots
// are pose priors.
int por_backward_dsac(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double gt_R[9],
                      const double gt_t[3], int n_prior, const orc_dsac_out* fwd, orc_backward_dsac_out* out) {
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
    // refine(), cnn.h:787-852: from the P3P pose of the (possibly perturbed) minimal set, or from a prior's own pose
    auto refine_from = [&](bool has_set, const float obj[12], const float img[8], const double* prior, const int16_t* local,
                           int n_perm, double out6[6]) {
        double pose[6];
        if (has_set) orc_solve_p3p(obj, img, fr.f, fr.cx, fr.cy, pose, pose + 3);
        else std::memcpy(pose, prior, sizeof(pose));
        Frame lf{local, pix, cfg.f, cfg.cx, cfg.cy};
        refine_loop(cfg, lf, perms.data(), n_perm, false, nullptr, nullptr, nullptr, nullptr, pose);
        jp6_from_cv(pose, pose + 3, out6);
        n_jobs++;
    };
    for (int h = 0; h < H; h++) {
        if (!(fwd->sf[h] > 0.0001)) continue;
        const bool has_set = fwd->img_idx[h * 4] >= 0;
        if (!has_set && h < H - n_prior) continue;   // an exhausted slot: no minimal set and no prior
        n_sel++;
        float obj[12], img[8];
        if (has_set) {
            int32_t cells[8];
            for (int j = 0; j < 4; j++) {
                cells[j * 2] = fwd->img_idx[h * 4 + j] % ORC_GRID;
                cells[j * 2 + 1] = fwd->img_idx[h * 4 + j] / ORC_GRID;
            }
            gather_set(fr, cells, obj, img);
        }
        const double prior[6] = {fwd->hyp_rvec[h * 3], fwd->hyp_rvec[h * 3 + 1], fwd->hyp_rvec[h * 3 + 2],
                                 fwd->hyp_tvec[h * 3], fwd->hyp_tvec[h * 3 + 1], fwd->hyp_tvec[h * 3 + 2]};
        std::vector<int32_t> imap(ORC_N, 0);
        int n_perm = 0;
        {
            double pose[6];
            std::memcpy(pose, prior, sizeof(pose));
            std::mt19937 randG;
            refine_loop(cfg, fr, nullptr, 0, true, &randG, nullptr, &n_perm, imap.data(), pose);
            if (has_set)
                for (int j = 0; j < 4; j++) imap[fwd->img_idx[h * 4 + j]] = 0;
        }
        std::vector<double> J((size_t)6 * N3, 0.0);
        std::vector<int16_t> local(coords, coords + N3);
        if (has_set)
            for (int pt = 0; pt < 3; pt++)
                for (int c = 0; c < 3; c++) {
                    const int cell = fwd->img_idx[h * 4 + pt];
                    int16_t& v = local[cell * 3 + c];
                    double fS[6], bS[6];
                    v += eps; obj[pt * 3 + c] += eps;
                    refine_from(true, obj, img, prior, local.data(), n_perm, fS);
                    v -= 2 * eps; obj[pt * 3 + c] -= 2 * eps;
                    refine_from(true, obj, img, prior, local.data(), n_perm, bS);
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
                    refine_from(has_set, obj, img, prior, local.data(), n_perm, fS);
                    v -= 2 * eps;
                    refine_from(has_set, obj, img, prior, local.data(), n_perm, bS);
                    v += eps;
                    for (int k = 0; k < 6; k++)
                        J[(size_t)k * N3 + (y * ORC_GRID + x) * 3 + c] = (fS[k] - bS[k]) / (2 * eps) * skip;
                }
            }
        double ref6[6], dL[6];
        jp6_from_cv(fwd->ref_pose + h * 6, fwd->ref_pose + h * 6 + 3, ref6);
        orc_dloss_max(ref6, gt6, dL);
        for (int col = 0; col < N3; col++) {
            double g = 0;
            for (int k = 0; k < 6; k++) g += dL[k] * J[(size_t)k * N3 + col];
            p1[col] += fwd->sf[h] * g;
        }
    }
    std::vector<double> sog(H, 0.0), dpnp_all((size_t)H * 72);
    for (int i = 0; i < H; i++) {
        sog[i] = fwd->sf[i] * fwd->losses[i];
        for (int j = 0; j < H; j++) sog[i] -= fwd->sf[i] * fwd->sf[j] * fwd->losses[j];
    }
    if (out->score_grads) std::memcpy(out->score_grads, sog.data(), H * sizeof(double));
    pool_dpnp(fr, H, fwd->img_idx, dpnp_all);
    pool_dscore_accumulate(cfg, fr, coords, pix, H, fwd->img_idx, fwd->hyp_rvec, fwd->hyp_tvec, sog, dpnp_all, 1, p2);
    for (int c = 0; c < N3; c++) out->dloss_dobj[c] = p1[c] + p2[c];
    if (out->path1) std::memcpy(out->path1, p1.data(), N3 * sizeof(double));
    if (out->path2) std::memcpy(out->path2, p2.data(), N3 * sizeof(double));
    out->n_selected = n_sel;
    out->n_refine_jobs = n_jobs;
    return 0;
}
}
