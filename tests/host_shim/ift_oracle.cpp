// ift_oracle.cpp -- test helper (tests/ift_oracle.py builds it): the oracle's refinement replay, restated to record the
// cells its last accepted step fitted -- the set S the implicit-function derivatives of dsac_set_coord_derivatives
// (DSAC_DERIV_IMPLICIT) are taken over.  It compiles the unmodified oracle sources into the same library (with the flags
// of oracle/Makefile's parity build) and repeats refine_loop's operations in the same order, so its pose is orc_refine's
// bit for bit.
#include "dsac_oracle.cpp"

extern "C" {
// refine() from the cv pose init over the permutations perm [n_perm][N]: pose_out (cv), the cells of the last accepted
// step in selection order sel [<= inlier_count] and their number *count (0: no step accepted).  Returns the steps done.
int ior_refine_record(const orc_config* cfgp, const int16_t* coords, const int32_t* pix, const int32_t* perm, int n_perm,
                      const double init[6], double pose_out[6], int32_t* sel, int32_t* count) {
    const orc_config& cfg = *cfgp;
    double pose[6];
    std::memcpy(pose, init, sizeof(pose));
    std::vector<float> diff(ORC_N);
    orc_diff_map(coords, pix, pose, pose + 3, cfg.f, cfg.cx, cfg.cy, diff.data());
    int done = 0;
    *count = 0;
    std::vector<float> lobj, limg;
    std::vector<int32_t> cells;
    for (int rStep = 0; rStep < cfg.ref_steps; rStep++) {
        if (rStep >= n_perm) break;
        const int32_t* p = perm + rStep * ORC_N;
        lobj.clear();
        limg.clear();
        cells.clear();
        for (int k = 0; k < ORC_N; k++) {
            const int c = p[k];
            if (diff[c] < (float)cfg.thr2d) {
                limg.push_back((float)pix[c * 2]);
                limg.push_back((float)pix[c * 2 + 1]);
                for (int q = 0; q < 3; q++) lobj.push_back((float)coords[c * 3 + q]);
                cells.push_back(c);
            }
            if ((int)(limg.size() / 2) >= cfg.inlier_count) break;
        }
        const int n = (int)(limg.size() / 2);
        if (n < 50) break;
        double upd[6];
        std::memcpy(upd, pose, sizeof(upd));
        solve_pnp_iterative(n, lobj.data(), limg.data(), cfg.f, cfg.cx, cfg.cy, upd, upd + 3);
        bool nan = false;
        for (int i = 0; i < 6; i++)
            if (upd[i] != upd[i]) nan = true;
        if (nan) break;
        std::memcpy(pose, upd, sizeof(upd));
        done++;
        *count = n;
        for (int i = 0; i < n; i++) sel[i] = cells[i];
        orc_diff_map(coords, pix, pose, pose + 3, cfg.f, cfg.cx, cfg.cy, diff.data());
    }
    std::memcpy(pose_out, pose, sizeof(pose));
    return done;
}
}
