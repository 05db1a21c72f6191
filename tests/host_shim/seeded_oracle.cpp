// seeded_oracle.cpp -- test helper (tests/seeded_oracle.py builds it): the oracle's two backward chains seeded by the
// caller, for the engine's pose-valued outputs (dsac_backward_pose_device, dsac_backward_dsac_pose_device).  It compiles
// the unmodified oracle sources into the same library (with the flags of oracle/Makefile's parity build) and restates
// orc_backward / orc_backward_dsac with the seed in place of dLossMax -- the same operations in the same order -- on top
// of the oracle's internal helpers (Frame, gather_set, refine_loop, dscore_accumulate).
//   orc_backward_seeded      : dLossMax replaced by seed6 = dOuter/d(refined jp6); out->dloss_dref receives seed6.
//   orc_backward_dsac_seeded : sf_h * dLossMax_h replaced by seed[h] (H*6) over the hypotheses with sf_h > 1e-4 and a seed
//                              that is not all zero; path II from grad_sf (H) = dOuter/dsf in place of the losses.  Either
//                              seed may be NULL: its path is zero.  No ground truth is read.
#include "dsac_oracle.cpp"

extern "C" {
int orc_backward_seeded(const orc_config* cfg, const int16_t* coords, const int32_t* pix, const orc_forward_out* fwd,
                        const double seed6[6], orc_backward_out* out);
int orc_backward_dsac_seeded(const orc_config* cfg, const int16_t* coords, const int32_t* pix, const orc_dsac_out* fwd,
                             const double* seed, const double* grad_sf, orc_backward_dsac_out* out);
}

// orc_backward with the caller's seed in place of dLossMax (see the head of this file): the same operations in the same order.
int orc_backward_seeded(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const orc_forward_out* fwd,
                        const double seed6[6], orc_backward_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, N3 = ORC_N * 3;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> row(N3, 0.0);
    double dL[6];
    std::memcpy(dL, seed6, sizeof(dL));
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
    for (int h = 0; h < H; h++) {
        float obj[12], img[8];
        int32_t cells[8];
        for (int j = 0; j < 4; j++) {
            cells[j * 2] = fwd->img_idx[h * 4 + j] % ORC_GRID;
            cells[j * 2 + 1] = fwd->img_idx[h * 4 + j] / ORC_GRID;
        }
        gather_set(fr, cells, obj, img);
        double* J = &dpnp_all[(size_t)h * 72];
        orc_dpnp(obj, img, fr.f, fr.cx, fr.cy, J);
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

    dscore_accumulate(cfg, fr, coords, pix, H, fwd->img_idx, sog, dpnp_all, cfg.fix_q4, row);
    std::memcpy(out->dloss_dobj, row.data(), N3 * sizeof(double));
    return 0;
}

// orc_backward_dsac with the caller's seeds in place of sf_h dLossMax_h and the losses (see the head of this file).
int orc_backward_dsac_seeded(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const orc_dsac_out* fwd,
                             const double* seed, const double* grad_sf, orc_backward_dsac_out* out) {
    const orc_config& cfg = *cfgp;
    const int H = cfg.n_hyps, N3 = ORC_N * 3;
    Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    std::vector<double> p1(N3, 0.0), p2(N3, 0.0);
    std::vector<int32_t> perms((size_t)cfg.ref_steps * ORC_N);
    orc_refine_permutations(cfg.ref_steps, perms.data());
    int n_sel = 0, n_jobs = 0;
    const float eps = 2.f;
    const int skip = 1 / (float)cfg.sub_sample;

    auto refine_from_set = [&](const float obj[12], const float img[8], const int16_t* local, int n_perm, double out6[6]) {
        double pose[6];
        orc_solve_p3p(obj, img, fr.f, fr.cx, fr.cy, pose, pose + 3);
        Frame lf{local, pix, cfg.f, cfg.cx, cfg.cy};
        refine_loop(cfg, lf, perms.data(), n_perm, false, nullptr, nullptr, nullptr, nullptr, pose);
        jp6_from_cv(pose, pose + 3, out6);
        n_jobs++;
    };

    // ---- path I: the hypotheses with sf > 1e-4 whose seed is not all zero
    for (int h = 0; h < H && seed; h++) {
        if (!(fwd->sf[h] > 0.0001)) continue;
        bool nz = false;
        for (int k = 0; k < 6; k++) nz |= seed[h * 6 + k] != 0.0;
        if (!nz) continue;
        n_sel++;
        int32_t cells[8];
        for (int j = 0; j < 4; j++) {
            cells[j * 2] = fwd->img_idx[h * 4 + j] % ORC_GRID;
            cells[j * 2 + 1] = fwd->img_idx[h * 4 + j] / ORC_GRID;
        }
        float obj[12], img[8];
        gather_set(fr, cells, obj, img);
        std::vector<int32_t> imap(ORC_N, 0);
        int n_perm = 0;
        {
            double pose[6] = {fwd->hyp_rvec[h * 3], fwd->hyp_rvec[h * 3 + 1], fwd->hyp_rvec[h * 3 + 2],
                              fwd->hyp_tvec[h * 3], fwd->hyp_tvec[h * 3 + 1], fwd->hyp_tvec[h * 3 + 2]};
            std::mt19937 randG;
            refine_loop(cfg, fr, nullptr, 0, true, &randG, nullptr, &n_perm, imap.data(), pose);
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
                refine_from_set(obj, img, local.data(), n_perm, fS);
                v -= 2 * eps; obj[pt * 3 + c] -= 2 * eps;
                refine_from_set(obj, img, local.data(), n_perm, bS);
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
                    refine_from_set(obj, img, local.data(), n_perm, fS);
                    v -= 2 * eps;
                    refine_from_set(obj, img, local.data(), n_perm, bS);
                    v += eps;
                    for (int k = 0; k < 6; k++)
                        J[(size_t)k * N3 + (y * ORC_GRID + x) * 3 + c] = (fS[k] - bS[k]) / (2 * eps) * skip;
                }
            }
        const double* dL = seed + h * 6;
        for (int col = 0; col < N3; col++) {
            double g = 0;
            for (int k = 0; k < 6; k++) g += dL[k] * J[(size_t)k * N3 + col];
            p1[col] += g;
        }
    }

    // ---- path II: the softmax Jacobian applied to grad_sf
    std::vector<double> sog(H, 0.0), dpnp_all((size_t)H * 72);
    if (grad_sf) {
        for (int i = 0; i < H; i++) {
            sog[i] = fwd->sf[i] * grad_sf[i];
            for (int j = 0; j < H; j++) sog[i] -= fwd->sf[i] * fwd->sf[j] * grad_sf[j];
        }
        for (int h = 0; h < H; h++) {
            float obj[12], img[8];
            int32_t cells[8];
            for (int j = 0; j < 4; j++) {
                cells[j * 2] = fwd->img_idx[h * 4 + j] % ORC_GRID;
                cells[j * 2 + 1] = fwd->img_idx[h * 4 + j] / ORC_GRID;
            }
            gather_set(fr, cells, obj, img);
            orc_dpnp(obj, img, fr.f, fr.cx, fr.cy, &dpnp_all[(size_t)h * 72]);
        }
        dscore_accumulate(cfg, fr, coords, pix, H, fwd->img_idx, sog, dpnp_all, 1, p2);
    }
    if (out->score_grads) std::memcpy(out->score_grads, sog.data(), H * sizeof(double));

    for (int c = 0; c < N3; c++) out->dloss_dobj[c] = p1[c] + p2[c];
    if (out->path1) std::memcpy(out->path1, p1.data(), N3 * sizeof(double));
    if (out->path2) std::memcpy(out->path2, p2.data(), N3 * sizeof(double));
    out->n_selected = n_sel;
    out->n_refine_jobs = n_jobs;
    return 0;
}

