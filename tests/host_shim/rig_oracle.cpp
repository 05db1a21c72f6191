// rig_oracle.cpp -- test helper (tests/rig_oracle.py builds it): a CPU restatement in fp64 of one rig of
// dsac_forward_rig_device (include/dsac_b200.h, INTEGRATION.md "Multi-camera rigs") from the frames' given hypotheses.
// It compiles the unmodified oracle sources into the same library, with the flags of the oracle's parity build, and uses
// their Rodrigues, soft-inlier score, softmax, entropy, LM step, cv2our and max_loss.  What the oracle has for one camera
// only is restated here for a camera behind a fixed extrinsic (Rc, tc), X_cam = Rc X_rig + tc:
//   - rig_diff_map: orc_diff_map from a rotation matrix in place of an rvec;
//   - rig_project: project_points' projection and Jacobian, the camera Jacobian chained through Rc;
//   - rig_solve_pnp: solve_pnp_iterative's CvLevMarq schedule over points of several cameras;
//   - the refinement: refine_loop with each camera's selection in turn.
// With C = 1 and a zero extrinsic every product with Rc = I and every sum with tc = 0 is exact, so the result is
// orc_forward's for the same pool bit for bit (tests/test_rig_oracle_host.py).
#include "dsac_oracle.cpp"

namespace {

constexpr int RIG_MAX_C = 8;

// orc_diff_map for the camera pose (R, t)
void rig_diff_map(const int16_t* coords, const int32_t* pix, const double R[9], const double t[3], double f, double cx, double cy,
                  float* diff) {
    for (int i = 0; i < ORC_N; i++) {
        double Xw = (float)coords[i * 3], Yw = (float)coords[i * 3 + 1], Zw = (float)coords[i * 3 + 2];
        double x = R[0] * Xw + R[1] * Yw + R[2] * Zw + t[0];
        double y = R[3] * Xw + R[4] * Yw + R[5] * Zw + t[1];
        double z = R[6] * Xw + R[7] * Yw + R[8] * Zw + t[2];
        z = z ? 1. / z : 1;
        x *= z;
        y *= z;
        float pu = (float)(x * f + cx), pv = (float)(y * f + cy);
        float du = (float)pix[i * 2] - pu, dv = (float)pix[i * 2 + 1] - pv;
        double nrm = std::sqrt((double)du * du + (double)dv * dv);
        diff[i] = (float)std::min(nrm, ORC_MAXINPUT);
    }
}

// Rc R, Rc t + tc
void compose(const double Rc[9], const double tc[3], const double R[9], const double t[3], double Ro[9], double to[3]) {
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) Ro[i * 3 + j] = Rc[i * 3] * R[j] + Rc[i * 3 + 1] * R[3 + j] + Rc[i * 3 + 2] * R[6 + j];
        to[i] = Rc[i * 3] * t[0] + Rc[i * 3 + 1] * t[1] + Rc[i * 3 + 2] * t[2] + tc[i];
    }
}

struct Cam {
    double f, cx, cy, R[9], t[3];   // intrinsics and the extrinsic cam_from_rig
};

// project_points for the rig pose `param` of points X [n][3], point i seen by camera cam[i]: uv [n][2] and, if asked,
// dp/dr, dp/dt [2n][3] with d(camera point) = Rc d(rig point).
void rig_project(int n, const double* X, const int* cam, const Cam* cams, const double param[6], double* uv, double* dpdr,
                 double* dpdt) {
    double R[9], dRdr[27];
    rodrigues_v2m(param, R, dpdr ? dRdr : nullptr);
    for (int i = 0; i < n; i++) {
        const Cam& k = cams[cam[i]];
        const double* Rc = k.R;
        double Xw = X[i * 3], Yw = X[i * 3 + 1], Zw = X[i * 3 + 2];
        double xr = R[0] * Xw + R[1] * Yw + R[2] * Zw + param[3];
        double yr = R[3] * Xw + R[4] * Yw + R[5] * Zw + param[4];
        double zr = R[6] * Xw + R[7] * Yw + R[8] * Zw + param[5];
        double x = Rc[0] * xr + Rc[1] * yr + Rc[2] * zr + k.t[0];
        double y = Rc[3] * xr + Rc[4] * yr + Rc[5] * zr + k.t[1];
        double z = Rc[6] * xr + Rc[7] * yr + Rc[8] * zr + k.t[2];
        z = z ? 1. / z : 1;
        x *= z;
        y *= z;
        uv[i * 2] = x * k.f + k.cx;
        uv[i * 2 + 1] = y * k.f + k.cy;
        if (dpdt) {
            double* a = dpdt + (2 * i) * 3;
            for (int j = 0; j < 3; j++) {
                a[j] = k.f * (z * (Rc[j] - x * Rc[6 + j]));
                a[3 + j] = k.f * (z * (Rc[3 + j] - y * Rc[6 + j]));
            }
        }
        if (dpdr) {
            double* a = dpdr + (2 * i) * 3;
            for (int j = 0; j < 3; j++) {
                double ax = Xw * dRdr[j * 9 + 0] + Yw * dRdr[j * 9 + 1] + Zw * dRdr[j * 9 + 2];
                double ay = Xw * dRdr[j * 9 + 3] + Yw * dRdr[j * 9 + 4] + Zw * dRdr[j * 9 + 5];
                double az = Xw * dRdr[j * 9 + 6] + Yw * dRdr[j * 9 + 7] + Zw * dRdr[j * 9 + 8];
                double dx0 = Rc[0] * ax + Rc[1] * ay + Rc[2] * az;
                double dy0 = Rc[3] * ax + Rc[4] * ay + Rc[5] * az;
                double dz0 = Rc[6] * ax + Rc[7] * ay + Rc[8] * az;
                double dxdr = z * (dx0 - x * dz0), dydr = z * (dy0 - y * dz0);
                a[j] = k.f * dxdr;
                a[3 + j] = k.f * dydr;
            }
        }
    }
}

// solve_pnp_iterative (CvLevMarq, 6 parameters, max_iter 20, eps FLT_EPSILON) with rig_project's residuals
void rig_solve_pnp(int n, const float* obj, const float* img, const int* cam, const Cam* cams, double param[6]) {
    std::vector<double> M(n * 3), m(n * 2), proj(n * 2), dpdr(n * 6), dpdt(n * 6), err(n * 2);
    for (int i = 0; i < n * 3; i++) M[i] = obj[i];
    for (int i = 0; i < n * 2; i++) m[i] = img[i];
    double prev[6];
    double JtJ[36], JtErr[6];
    int lambdaLg10 = -3, iters = 0;
    double prevErrNorm = std::numeric_limits<double>::max(), errNorm = 0;
    const int max_iter = 20;
    const double eps = std::numeric_limits<float>::epsilon();
    auto residual = [&](bool jac) {
        rig_project(n, M.data(), cam, cams, param, proj.data(), jac ? dpdr.data() : nullptr, jac ? dpdt.data() : nullptr);
        for (int i = 0; i < n * 2; i++) err[i] = proj[i] - m[i];
    };
    auto norm_err = [&]() {
        double s = 0;
        for (int i = 0; i < n * 2; i++) s += err[i] * err[i];
        return std::sqrt(s);
    };
    residual(true);
    for (;;) {
        for (int a = 0; a < 6; a++) {
            for (int b = a; b < 6; b++) {
                double s = 0;
                for (int i = 0; i < n * 2; i++) {
                    double ja = a < 3 ? dpdr[i * 3 + a] : dpdt[i * 3 + a - 3];
                    double jb = b < 3 ? dpdr[i * 3 + b] : dpdt[i * 3 + b - 3];
                    s += ja * jb;
                }
                JtJ[a * 6 + b] = JtJ[b * 6 + a] = s;
            }
            double s = 0;
            for (int i = 0; i < n * 2; i++) s += (a < 3 ? dpdr[i * 3 + a] : dpdt[i * 3 + a - 3]) * err[i];
            JtErr[a] = s;
        }
        std::memcpy(prev, param, sizeof(prev));
        lm_step(JtJ, JtErr, prev, lambdaLg10, param);
        if (iters == 0) prevErrNorm = norm_err();
        bool done = false;
        for (;;) {
            residual(false);
            errNorm = norm_err();
            if (errNorm > prevErrNorm) {
                if (++lambdaLg10 <= 16) {
                    lm_step(JtJ, JtErr, prev, lambdaLg10, param);
                    continue;
                }
            }
            lambdaLg10 = std::max(lambdaLg10 - 1, -16);
            double dn = 0, pn = 0;
            for (int i = 0; i < 6; i++) {
                dn += (param[i] - prev[i]) * (param[i] - prev[i]);
                pn += prev[i] * prev[i];
            }
            double change = std::sqrt(dn) / std::sqrt(pn);
            if (++iters >= max_iter || change < eps) done = true;
            break;
        }
        if (done) break;
        prevErrNorm = errNorm;
        residual(true);
    }
}

}  // namespace

extern "C" {

// One rig of C cameras: coords [C][N][3], pix [C][N][2], intr [C][3] (f, cx, cy), ext [C][6] (cam_from_rig, cv),
// hyp_pose [C][H][6] the frames' hypotheses (H = cfg->n_hyps), gt [12] (jp of the rig frame) nullable.  Outputs: rig_hyp
// [C H][6], scores and sf [C H], entropy, avg [6], ref [6], inlier_map [C][N], steps, loss, rot_err, t_err, correct, and
// min_margin: the smallest |error - thr2d| over the cells the refinement's selections tested (threshold ties).  start [6]
// (nullable): refine from this pose in place of the soft-argmax pose, to check the refinement on its own.
int rig_forward(const orc_config* cfgp, int C, const int16_t* coords, const int32_t* pix, const double* intr, const double* ext,
                const double* hyp_pose, const double* gt, const double* start, double* rig_hyp, double* scores, double* sf, double* entropy, double* avg,
                double* ref, int32_t* inlier_map, int32_t* steps, double* loss, double* rot_err, double* t_err, int32_t* correct,
                double* min_margin) {
    const orc_config& cfg = *cfgp;
    if (C < 1 || C > RIG_MAX_C) return -1;
    const int H = cfg.n_hyps, P = C * H;
    Cam cams[RIG_MAX_C];
    bool ident[RIG_MAX_C];
    for (int c = 0; c < C; c++) {
        cams[c].f = intr[c * 3]; cams[c].cx = intr[c * 3 + 1]; cams[c].cy = intr[c * 3 + 2];
        rodrigues_v2m(ext + c * 6, cams[c].R, nullptr);
        for (int k = 0; k < 3; k++) cams[c].t[k] = ext[c * 6 + 3 + k];
        ident[c] = ext[c * 6] == 0 && ext[c * 6 + 1] == 0 && ext[c * 6 + 2] == 0;
    }
    // ---- lift: R_r = Rc^T R_h, t_r = Rc^T (t_h - tc), slot c H + h; a zero extrinsic rvec keeps the hypothesis' rvec
    std::vector<double> Rr((size_t)P * 9), tr((size_t)P * 3);
    for (int c = 0; c < C; c++) {
        const double* Rc = cams[c].R;
        for (int h = 0; h < H; h++) {
            const int j = c * H + h;
            const double* hp = hyp_pose + ((size_t)c * H + h) * 6;
            double Rh[9], d[3];
            rodrigues_v2m(hp, Rh, nullptr);
            for (int k = 0; k < 3; k++) d[k] = hp[3 + k] - cams[c].t[k];
            double* R = &Rr[(size_t)j * 9];
            double* t = &tr[(size_t)j * 3];
            for (int a = 0; a < 3; a++) {
                for (int b = 0; b < 3; b++) R[a * 3 + b] = Rc[a] * Rh[b] + Rc[3 + a] * Rh[3 + b] + Rc[6 + a] * Rh[6 + b];
                t[a] = Rc[a] * d[0] + Rc[3 + a] * d[1] + Rc[6 + a] * d[2];
            }
            double* o = rig_hyp + (size_t)j * 6;
            if (ident[c]) {
                o[0] = hp[0]; o[1] = hp[1]; o[2] = hp[2];
            } else {
                rodrigues_m2v(R, o);
            }
            o[3] = t[0]; o[4] = t[1]; o[5] = t[2];
        }
    }
    // ---- score: the cameras' soft-inlier scores of the composed pose, summed in camera order
    std::vector<float> diff(ORC_N);
    for (int j = 0; j < P; j++) {
        double s = 0;
        for (int c = 0; c < C; c++) {
            double Rk[9], tk[3];
            compose(cams[c].R, cams[c].t, &Rr[(size_t)j * 9], &tr[(size_t)j * 3], Rk, tk);
            rig_diff_map(coords + (size_t)c * ORC_N * 3, pix + (size_t)c * ORC_N * 2, Rk, tk, cams[c].f, cams[c].cx, cams[c].cy, diff.data());
            const double sc = orc_soft_inlier_score(diff.data(), ORC_N, (double)cfg.thr2d, cfg.alpha, cfg.beta);
            s = c == 0 ? sc : s + sc;
        }
        scores[j] = s;
    }
    orc_softmax(scores, P, sf);
    *entropy = orc_entropy(sf, P);
    for (int i = 0; i < 6; i++) avg[i] = 0;
    for (int j = 0; j < P; j++)
        for (int i = 0; i < 6; i++) avg[i] = j == 0 ? sf[j] * rig_hyp[i] : avg[i] + sf[j] * rig_hyp[(size_t)j * 6 + i];
    // ---- refinement of the average (refine_loop, every camera's selection in turn)
    double pose[6];
    std::memcpy(pose, start ? start : avg, sizeof(pose));
    std::memset(inlier_map, 0, (size_t)C * ORC_N * sizeof(int32_t));
    std::vector<float> diffs((size_t)C * ORC_N);
    auto diff_all = [&]() {
        double R[9];
        rodrigues_v2m(pose, R, nullptr);
        for (int c = 0; c < C; c++) {
            double Rk[9], tk[3];
            compose(cams[c].R, cams[c].t, R, pose + 3, Rk, tk);
            rig_diff_map(coords + (size_t)c * ORC_N * 3, pix + (size_t)c * ORC_N * 2, Rk, tk, cams[c].f, cams[c].cx, cams[c].cy,
                         &diffs[(size_t)c * ORC_N]);
        }
    };
    diff_all();
    std::mt19937 randG;
    std::vector<int> idxs(ORC_N);
    std::vector<float> lobj, limg;
    std::vector<int> lcam;
    double margin = std::numeric_limits<double>::infinity();
    int done = 0;
    for (int rStep = 0; rStep < cfg.ref_steps; rStep++) {
        for (int i = 0; i < ORC_N; i++) idxs[i] = i;
        std::shuffle(idxs.begin(), idxs.end(), randG);
        lobj.clear(); limg.clear(); lcam.clear();
        for (int c = 0; c < C; c++) {
            const int16_t* co = coords + (size_t)c * ORC_N * 3;
            const int32_t* px = pix + (size_t)c * ORC_N * 2;
            int count = 0;
            for (int k = 0; k < ORC_N && count < cfg.inlier_count; k++) {
                const int cell = idxs[k];
                const float e = diffs[(size_t)c * ORC_N + cell];
                margin = std::min(margin, std::fabs((double)e - (double)cfg.thr2d));
                if (e < (float)cfg.thr2d) {
                    limg.push_back((float)px[cell * 2]);
                    limg.push_back((float)px[cell * 2 + 1]);
                    for (int q = 0; q < 3; q++) lobj.push_back((float)co[cell * 3 + q]);
                    lcam.push_back(c);
                    inlier_map[(size_t)c * ORC_N + cell] += 1;
                    count++;
                }
            }
        }
        const int n = (int)lcam.size();
        if (n < 50) break;
        double upd[6];
        std::memcpy(upd, pose, sizeof(upd));
        rig_solve_pnp(n, lobj.data(), limg.data(), lcam.data(), cams, upd);
        bool nan = false;
        for (int i = 0; i < 6; i++)
            if (upd[i] != upd[i]) nan = true;
        if (nan) break;
        std::memcpy(pose, upd, sizeof(upd));
        done++;
        diff_all();
    }
    std::memcpy(ref, pose, sizeof(pose));
    *steps = done;
    *min_margin = margin;
    *loss = *rot_err = *t_err = 0;
    *correct = 0;
    if (gt) {
        double eR[9], et[3];
        cv2our(ref, ref + 3, eR, et);
        *loss = max_loss(gt, gt + 9, eR, et, rot_err, t_err);
        *correct = (*rot_err < 5 && *t_err < 50) ? 1 : 0;
    }
    return 0;
}

}  // extern "C"
