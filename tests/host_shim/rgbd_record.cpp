// rgbd_record.cpp -- test helper (tests/test_gpu_pose_uncertainty.py builds it): the RGB-D Kabsch refinement replay of
// rgbd_oracle.cpp's refine_rgbd, restated to record the cells its last accepted step fitted -- the set S the pose
// covariance of an RGB-D pass is taken over.  It compiles rgbd_oracle.cpp (and through it the unmodified oracle sources)
// into the same library with the flags of the oracle's parity build, and repeats refine_rgbd's replay mode operation by
// operation, so its pose is refine_rgbd's bit for bit.
#include "rgbd_oracle.cpp"

extern "C" {
// refine() of an RGB-D pass from the cv pose init over the permutations perm [n_perm][N], with the camera (cfg f, cx, cy):
// pose_out (cv), the cells of the last accepted step in selection order sel [<= inlier_count] and their number *count (0:
// no step accepted).  eye [N][3], NaN without depth.  Returns the steps done.
int rrec_refine_record(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const double* eye, const int32_t* perm,
                       int n_perm, const double init[6], double pose_out[6], int32_t* sel, int32_t* count) {
    const orc_config& cfg = *cfgp;
    const Frame fr{coords, pix, cfg.f, cfg.cx, cfg.cy};
    double pose[6];
    std::memcpy(pose, init, sizeof(pose));
    std::vector<float> diff(ORC_N);
    orc_diff_map(fr.coords, fr.pix, pose, pose + 3, fr.f, fr.cx, fr.cy, diff.data());
    int done = 0;
    *count = 0;
    std::vector<double> a, b;
    std::vector<int32_t> cells;
    for (int rStep = 0; rStep < cfg.ref_steps; rStep++) {
        if (rStep >= n_perm) break;
        const int32_t* pp = perm + rStep * ORC_N;
        a.clear();
        b.clear();
        cells.clear();
        for (int k = 0; k < ORC_N; k++) {
            const int c = pp[k];
            if (diff[c] < (float)cfg.thr2d && has_depth(eye, c)) {
                for (int q = 0; q < 3; q++) { a.push_back(fr.coords[c * 3 + q]); b.push_back(eye[c * 3 + q]); }
                cells.push_back(c);
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
        *count = n;
        for (int i = 0; i < n; i++) sel[i] = cells[i];
        orc_diff_map(fr.coords, fr.pix, pose, pose + 3, fr.f, fr.cx, fr.cy, diff.data());
    }
    std::memcpy(pose_out, pose, sizeof(pose));
    return done;
}
}
