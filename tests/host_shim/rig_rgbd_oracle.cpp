// rig_rgbd_oracle.cpp -- test helper (tests/rig_rgbd_oracle.py builds it): a CPU restatement in fp64 of one RGB-D rig's
// refinement (dsac_set_rig_cell_depth_device, INTEGRATION.md "RGB-D rigs").  It compiles the unmodified oracle sources and
// the RGB rig restatement (rig_oracle.cpp: its composition, Cam and rig_diff_map) into the same library, with the flags of
// the oracle's parity build, and follows rgbd_oracle.cpp's refine_rgbd with each camera's selection in turn: per step
// the cells of each camera in permutation order whose error is below thr2d and that have depth in that camera's frame,
// at most inlier_count per camera; fewer than 50 in all stop; the pose update is orc_kabsch from the scene coordinates to
// the rig-frame eye points Rc^T (e - tc) (e - tc exactly for Rc = I).  With C = 1 and a zero extrinsic every product
// with Rc = I and every sum with tc = 0 is exact, so the result is refine_rgbd's bit for bit.
#include "rig_oracle.cpp"

extern "C" {

// One rig of C cameras refined from `start` [6]: coords [C][N][3], pix [C][N][2], intr [C][3], ext [C][6] (cam_from_rig,
// cv), eye [C][N][3] (NaN without depth).  Outputs: ref [6], inlier_map [C][N], steps, and min_margin, the smallest
// |error - thr2d| over the cells with depth the selections tested (threshold ties).
int rig_rgbd_refine(const orc_config* cfgp, int C, const int16_t* coords, const int32_t* pix, const double* intr, const double* ext,
                    const double* eye, const double* start, double* ref, int32_t* inlier_map, int32_t* steps, double* min_margin) {
    const orc_config& cfg = *cfgp;
    if (C < 1 || C > RIG_MAX_C) return -1;
    Cam cams[RIG_MAX_C];
    bool ident[RIG_MAX_C];
    for (int c = 0; c < C; c++) {
        cams[c].f = intr[c * 3]; cams[c].cx = intr[c * 3 + 1]; cams[c].cy = intr[c * 3 + 2];
        rodrigues_v2m(ext + c * 6, cams[c].R, nullptr);
        for (int k = 0; k < 3; k++) cams[c].t[k] = ext[c * 6 + 3 + k];
        ident[c] = true;
        for (int k = 0; k < 9; k++) ident[c] = ident[c] && cams[c].R[k] == (k % 4 == 0 ? 1.0 : 0.0);
    }
    double pose[6];
    std::memcpy(pose, start, sizeof(pose));
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
    std::vector<double> a, b;
    double margin = std::numeric_limits<double>::infinity();
    int done = 0;
    for (int rStep = 0; rStep < cfg.ref_steps; rStep++) {
        for (int i = 0; i < ORC_N; i++) idxs[i] = i;
        std::shuffle(idxs.begin(), idxs.end(), randG);
        a.clear();
        b.clear();
        for (int c = 0; c < C; c++) {
            const int16_t* co = coords + (size_t)c * ORC_N * 3;
            const double* ey = eye + (size_t)c * ORC_N * 3;
            const double* Rc = cams[c].R;
            int count = 0;
            for (int k = 0; k < ORC_N && count < cfg.inlier_count; k++) {
                const int cell = idxs[k];
                if (!(ey[cell * 3 + 2] > 0.0)) continue;   // (NaN: no depth)
                const float e = diffs[(size_t)c * ORC_N + cell];
                margin = std::min(margin, std::fabs((double)e - (double)cfg.thr2d));
                if (e < (float)cfg.thr2d) {
                    const double d[3] = {ey[cell * 3] - cams[c].t[0], ey[cell * 3 + 1] - cams[c].t[1], ey[cell * 3 + 2] - cams[c].t[2]};
                    for (int q = 0; q < 3; q++) {
                        a.push_back(co[cell * 3 + q]);
                        b.push_back(ident[c] ? d[q] : Rc[q] * d[0] + Rc[3 + q] * d[1] + Rc[6 + q] * d[2]);
                    }
                    inlier_map[(size_t)c * ORC_N + cell] += 1;
                    count++;
                }
            }
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
        diff_all();
    }
    std::memcpy(ref, pose, sizeof(pose));
    *steps = done;
    *min_margin = margin;
    return 0;
}

}  // extern "C"
