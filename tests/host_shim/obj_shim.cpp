// Host build of the pre-training data path's arithmetic (dsac_b200/csrc/objtrain.cuh, DSAC_HOST_ONLY) for CPU-side
// checks against tests/obj_oracle.py and against libstdc++ / gcc themselves.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include <random>
#include "../../dsac_b200/csrc/objtrain.cuh"

extern "C" {
// cam: the dsac_rgbd_camera layout (ObjCam has the same fields in the same order)
void shim_obj_coords(const dsac::ObjCam* cam, const uint16_t* depth, const double* pose, int16_t* out) {
    dsac::ObjPose p;
    dsac::obj_pose(pose, &p);
    for (int y = 0; y < cam->height; y++)
        for (int x = 0; x < cam->width; x++) {
            const size_t i = (size_t)y * cam->width + x;
            dsac::obj_coord(*cam, p, x, y, depth[i], out + 3 * i);
        }
}
// getDepth's scatter in the reference's own order (x outer, y inner, the last write wins), with the product's mapping
int shim_register_depth(const dsac::ObjCam* cam, const uint16_t* raw, uint16_t* out) {
    const int W = cam->width, H = cam->height;
    int dropped = 0;
    for (size_t i = 0; i < (size_t)W * H; i++) out[i] = cam->raw_data ? 0 : raw[i];
    if (!cam->raw_data) return 0;
    for (int x = 0; x < W; x++)
        for (int y = 0; y < H; y++) {
            const uint16_t d = raw[(size_t)y * W + x];
            if (d == 0) continue;
            int nx, ny;
            dsac::map_depth_to_rgb(*cam, x, y, d, &nx, &ny);
            if (nx < 0 || ny < 0 || nx >= W || ny >= H) { dropped++; continue; }
            out[(size_t)ny * W + nx] = d;
        }
    return dropped;
}
void shim_inv_rotation(const double* m, double* r) { dsac::obj_inv_rotation(m, r); }
void shim_mm_to_m(int n, const int16_t* v, float* out) {
    for (int i = 0; i < n; i++) out[i] = dsac::mm_to_m(v[i]);
}
// the product's conversions next to what gcc makes of the reference's casts, on values it cannot fold
void shim_cvt(int n, const double* v, int32_t* d2i, int32_t* f2i, int16_t* d2s_ref, int16_t* f2s_ref, int16_t* d2s,
              int16_t* f2s) {
    for (int i = 0; i < n; i++) {
        volatile double dv = v[i];
        volatile float fv = (float)v[i];
        d2i[i] = dsac::cvtt_d2i(dv);
        f2i[i] = dsac::cvtt_f2i(fv);
        d2s[i] = dsac::low16(dsac::cvtt_d2i(dv));
        f2s[i] = dsac::low16(dsac::cvtt_f2i(fv));
        d2s_ref[i] = (short)dv;
        f2s_ref[i] = (short)fv;
    }
}
// lemire_draw over std::mt19937(seed) next to std::uniform_int_distribution<int>(0, range - 1) on a second engine
int shim_lemire_vs_std(uint32_t seed, uint32_t range, int n, uint32_t* mine, uint32_t* theirs) {
    std::mt19937 a(seed), b(seed);
    for (int i = 0; i < n; i++) {
        mine[i] = dsac::lemire_draw(range, [&]() { return (uint32_t)a(); });
        std::uniform_int_distribution<int> dist(0, (int)range - 1);
        theirs[i] = (uint32_t)dist(b);
    }
    return a == b ? 1 : 0;
}
}
