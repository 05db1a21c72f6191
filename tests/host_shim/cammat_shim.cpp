// Host build of the score path's dataset camera (dsac_b200/csrc/scoretrain.cuh score_cam, DSAC_HOST_ONLY) next to
// getCamMat() and getObj's principal point as the reference spells them, for CPU-side checks.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/scoretrain.cuh"

extern "C" {
// cam: the dsac_rgbd_camera layout (ObjCam has the same fields in the same order)
void shim_score_cam(const dsac::ObjCam* cam, double* f, float* cx, float* cy) {
    const dsac::ScoreCam c = dsac::score_cam(*cam);
    *f = c.f;
    *cx = c.cx;
    *cy = c.cy;
}
// GlobalProperties::getCamMat() (properties.cpp:308-311): int imageWidth / 2, then + float xShift
void shim_ref_getcammat(const dsac::ObjCam* cam, float* f, float* cx, float* cy) {
    const int imageWidth = cam->width, imageHeight = cam->height;
    const float xShift = cam->x_shift, yShift = cam->y_shift;
    volatile float centerX = imageWidth / 2 + xShift;
    volatile float centerY = imageHeight / 2 + yShift;
    *f = cam->focal;
    *cx = centerX;
    *cy = centerY;
}
// pxToEye's principal point (dataset.cpp:51-52): imageWidth / 2.f + xShift
void shim_ref_getobj_centre(const dsac::ObjCam* cam, float* cx, float* cy) {
    volatile float centerX = cam->width / 2.f + cam->x_shift;
    volatile float centerY = cam->height / 2.f + cam->y_shift;
    *cx = centerX;
    *cy = centerY;
}
}
