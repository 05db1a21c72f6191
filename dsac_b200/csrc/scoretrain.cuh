// scoretrain.cuh -- the data path of the score CNN's pre-training (the reference's train_score.cpp) on the device:
//   * k_score_draw:  assembleData's random draw (train_score.cpp:166-230): per image the frame (irand), the sampling grid
//                    (stochasticSubSample, cnn.h:348-374) and, per hypothesis, the drift level and getRandHyp (:48-72)
//   * k_score_maps:  per (image, hypothesis) poseGT * getRandHyp, the 40x40 reprojection-error image of getDiffMap
//                    (cnn.h:384-427) with K2's arithmetic, the label -temperature * max(angle deg, |dt| mm / 10) and the
//                    5 deg / 50 mm flag; k_score_maps_cam with each frame's getCamMat() camera from the per-dataset table
// The random draws and the pose arithmetic are DSAC_HD functions, so that the host build (tests/host_shim/score_shim.cpp)
// can be checked against the numpy restatement and against libstdc++'s own distributions on a machine without a GPU.
// Every double operation of the draw is spelled with a round-to-nearest intrinsic on the device (objtrain.cuh's OT_*),
// so that nothing is contracted into an FMA the x86 reference never executes.
#pragma once
#include "objtrain.cuh"
#include "train.cuh"

namespace dsac {

#if defined(__CUDA_ARCH__)
#define SC_DSQRT(a) __dsqrt_rn(a)
#else
#define SC_DSQRT(a) sqrt(a)
#endif

constexpr int SCORE_GRID_MAX = 48;     // bounds kept by the entry point (which accepts only 40-iteration loops)
constexpr double SCORE_PI = 3.1415926; // types.h:33: getRandHyp's degrees -> radians (not CV_PI)

// stochasticSubSample's float loop over one axis of a frame `size` pixels wide (patchSize 42, targetSize 40): the upper
// bound of every cell in loop order (the lower bound of cell k > 0 is the upper bound of cell k - 1, of cell 0 it is 21).
// Returns the number of iterations; bounds past max are not stored.  size must exceed 42 (else the loop never ends).
DSAC_HD int score_grid_bounds(int size, float* bounds, int max) {
    const float stride = OT_FDIV((float)(size - 42), (float)DSAC_GRID_CONST);
    const float end = (float)(size - 42 / 2 + 1);
    int n = 0;
    for (float v = OT_FADD(stride, (float)(42 / 2)); v <= end; v = OT_FADD(v, stride)) {
        if (n < max) bounds[n] = v;
        n++;
    }
    return n;
}

// uniform_real_distribution<double>(a, b) of a generate_canonical value: (b - a) * canonical + a
DSAC_HD double uniform_real(double canon, double a, double b) { return OT_DADD(OT_DMUL(canon, OT_DSUB(b, a)), a); }

template <class Next>
DSAC_HD double canonical_draw(Next&& next) {
    const uint32_t w0 = next();
    const uint32_t w1 = next();
    return canonical53(w0, w1);
}

// dgauss: a fresh std::normal_distribution<double>(mean, stddev) per call, so libstdc++'s polar method
// (bits/random.tcc) runs from scratch and its saved second value is discarded.  Each attempt takes 4 words.
template <class Next>
DSAC_HD double normal_draw(double mean, double stddev, Next&& next) {
    double x, y, r2;
    do {
        x = OT_DSUB(OT_DMUL(2.0, canonical_draw(next)), 1.0);
        y = OT_DSUB(OT_DMUL(2.0, canonical_draw(next)), 1.0);
        r2 = OT_DADD(OT_DMUL(x, x), OT_DMUL(y, y));
    } while (r2 > 1.0 || r2 == 0.0);
    const double mult = SC_DSQRT(OT_DDIV(OT_DMUL(-2.0, log(r2)), r2));
    return OT_DADD(OT_DMUL(OT_DMUL(y, mult), stddev), mean);
}

// getRandHyp(gaussRot, gaussTrans) as the 6-vector it hands to Hypothesis(v): rotation vector (radians), translation
// (mm).  GCC evaluates a constructor's three arguments right to left, so z is drawn before y before x, for the
// translation and for the axis.  The axis lies in the positive octant; the sign comes from the Gaussian angle.
template <class Next>
DSAC_HD void score_rand_hyp(float gauss_rot, float gauss_trans, Next&& next, double v[6]) {
    const double tz = normal_draw(0.0, (double)gauss_trans, next);
    const double ty = normal_draw(0.0, (double)gauss_trans, next);
    const double tx = normal_draw(0.0, (double)gauss_trans, next);
    double az = uniform_real(canonical_draw(next), 0.0, 1.0);
    double ay = uniform_real(canonical_draw(next), 0.0, 1.0);
    double ax = uniform_real(canonical_draw(next), 0.0, 1.0);
    const double inv = OT_DDIV(1.0, SC_DSQRT(OT_DADD(OT_DADD(OT_DMUL(ax, ax), OT_DMUL(ay, ay)), OT_DMUL(az, az))));
    ax = OT_DMUL(ax, inv); ay = OT_DMUL(ay, inv); az = OT_DMUL(az, inv);
    const double angle = normal_draw(0.0, (double)gauss_rot, next);
    const double deg = SCORE_PI / 180.0;
    v[0] = OT_DMUL(OT_DMUL(ax, angle), deg);
    v[1] = OT_DMUL(OT_DMUL(ay, angle), deg);
    v[2] = OT_DMUL(OT_DMUL(az, angle), deg);
    v[3] = tx; v[4] = ty; v[5] = tz;
}

// One (image, hypothesis) of assembleData's loop body, without the error image: poseGT = Hypothesis(info) (Q19: the
// rotation through float, the centre through float(t / 1000) times 1e3), poseNoise = poseGT * Hypothesis(v) as the 4x4
// product, the label and the flag from calcAngularDistance (poseNoise's invRotation: OpenCV's closed form) and the norm of
// the translation difference, and the projection rows of our2cv(poseNoise) as K1 builds them for K2 (rows f R0 | f t0,
// f R1 | f t1, R2 | t2 of the rotation cv::projectPoints rebuilds from the Rodrigues vector, in float).
struct ScoreSample {
    float P[12];
    double label;
    int correct;
};
DSAC_HD void score_sample(const double* gt_jp, const double v[6], double f, float temperature, ScoreSample* out) {
    double Rg[9], Rh[9], Rn[9], tn[3];
    for (int k = 0; k < 9; k++) Rg[k] = (double)(float)gt_jp[k];
    ObjPose gp;
    obj_pose(gt_jp, &gp);   // gp.t: the centre * 1e3 as Hypothesis(info) keeps it
    // Hypothesis(v): the identity below |r| = 1e-5, cv::Rodrigues above
    const double len = SC_DSQRT(OT_DADD(OT_DADD(OT_DMUL(v[0], v[0]), OT_DMUL(v[1], v[1])), OT_DMUL(v[2], v[2])));
    if (len > 1e-5) {
        rodrigues_v2m(v, Rh);
    } else {
        for (int k = 0; k < 9; k++) Rh[k] = (k % 4 == 0) ? 1.0 : 0.0;
    }
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++)
            Rn[3 * i + j] = OT_DADD(OT_DADD(OT_DMUL(Rg[3 * i], Rh[j]), OT_DMUL(Rg[3 * i + 1], Rh[3 + j])),
                                    OT_DMUL(Rg[3 * i + 2], Rh[6 + j]));
        tn[i] = OT_DADD(OT_DADD(OT_DADD(OT_DMUL(Rg[3 * i], v[3]), OT_DMUL(Rg[3 * i + 1], v[4])), OT_DMUL(Rg[3 * i + 2], v[5])),
                        gp.t[i]);
    }
    // calcAngularDistance: trace(poseGT.rotation * poseNoise.invRotation)
    double Ri[9];
    obj_inv_rotation(Rn, Ri);
    double trace = 0;
    for (int i = 0; i < 3; i++)
        trace = OT_DADD(trace, OT_DADD(OT_DADD(OT_DMUL(Rg[3 * i], Ri[i]), OT_DMUL(Rg[3 * i + 1], Ri[3 + i])),
                                       OT_DMUL(Rg[3 * i + 2], Ri[6 + i])));
    const double ang = rot_err_deg(trace);
    const double d0 = OT_DSUB(gp.t[0], tn[0]), d1 = OT_DSUB(gp.t[1], tn[1]), d2 = OT_DSUB(gp.t[2], tn[2]);
    const double dt = SC_DSQRT(OT_DADD(OT_DADD(OT_DMUL(d0, d0), OT_DMUL(d1, d1)), OT_DMUL(d2, d2)));
    const double tcm = OT_DDIV(dt, 10.0);
    out->label = OT_DMUL((double)(-temperature), ang < tcm ? tcm : ang);
    out->correct = (ang < 5 && dt < 50) ? 1 : 0;
    // our2cv: rows 1 and 2 negated, cv::Rodrigues to a vector; getDiffMap's cv::projectPoints rebuilds the matrix
    double rm[9], rvec[3], R[9];
    for (int k = 0; k < 9; k++) rm[k] = k < 3 ? Rn[k] : -Rn[k];
    // cv::Rodrigues first projects its input onto the nearest rotation (U V^T of its SVD); rodrigues_m2v assumes an
    // orthonormal matrix.  Rn is orthonormal only to float precision (poseGT's rotation is float), and near 180 degrees
    // -- Rn near the identity -- the axis amplifies that error.  Two steps of Newton's polar iteration R <- (R + R^-T) / 2
    // give the same projection to double precision (the error squares per step, from ~1e-7).
    for (int it = 0; it < 2; it++) {
        double inv[9];
        obj_inv_rotation(rm, inv);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) rm[3 * i + j] = 0.5 * (rm[3 * i + j] + inv[3 * j + i]);
    }
    rodrigues_m2v(rm, rvec);
    rodrigues_v2m(rvec, R);
    const double t[3] = {tn[0], -tn[1], -tn[2]};
    for (int r = 0; r < 2; r++) {
        for (int c = 0; c < 3; c++) out->P[4 * r + c] = (float)(f * R[3 * r + c]);
        out->P[4 * r + 3] = (float)(f * t[r]);
    }
    for (int c = 0; c < 3; c++) out->P[8 + c] = (float)R[6 + c];
    out->P[11] = (float)t[2];
}

// The camera train_score.cpp projects with, getCamMat() (properties.cpp:308-311, train_score.cpp:178), of a dataset
// camera: the focal length, and a principal point of the INTEGER width / 2 (and height / 2) plus the float shift, in
// float.  getObj's principal point is width / 2.f + x_shift instead (dataset.cpp:51); the two differ on odd frame sizes
// (DESIGN.md quirk Q27).  k_score_maps takes dsac_config's camera in the same form: f, and cx / cy rounded to float.
struct ScoreCam {
    double f;
    float cx, cy;
};
DSAC_HD ScoreCam score_cam(const ObjCam& c) {
    return ScoreCam{(double)c.focal, OT_FADD((float)(c.width / 2), c.x_shift), OT_FADD((float)(c.height / 2), c.y_shift)};
}

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)

// ----------------------------------------------------------------------------- assembleData's draw
struct ScoreDrawParams {
    int n_frames, n_images, hyps, n_streams;
    int nx, ny;                                          // iterations of stochasticSubSample's x and y loops
    float xb[SCORE_GRID_MAX], yb[SCORE_GRID_MAX];        // score_grid_bounds of the frame width and height
    uint32_t* state;   // [T][625] std::mt19937 words + position, read and written back
    int32_t* img;      // [n_images]
    int32_t* pix;      // [n_images][1600][2] (x, y), cell y * 40 + x
    int32_t* drift;    // [n_images * hyps]
    double* noise;     // [n_images * hyps][6] getRandHyp's rotation vector and translation
};

// One warp per stream t (std::mt19937(seed + t) of ThreadRand), on the two-block window of k_obj_draw (ObjStream).
// Stream 0 draws, per image, the frame and the grid, then every stream draws its static-schedule chunk of the image's
// hypotheses (the omp parallel for runs once per image, so stream 0 interleaves frame, grid and hypotheses image by
// image).  Sequential draws are made by all lanes in step from the same words (the window's advance needs the whole
// warp); the grid's cells take 4 words each at fixed positions, so lane l converts cell c0 + l.
__global__ void __launch_bounds__(32 * OBJ_DRAW_WARPS) k_score_draw(ScoreDrawParams p) {
    __shared__ uint32_t sbuf[OBJ_DRAW_WARPS][2][MT_N];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * OBJ_DRAW_WARPS + warp;
    if (t >= p.n_streams) return;
    uint32_t* st = p.state + (size_t)t * OBJ_STATE_WORDS;
    ObjStream s;
    s.blk[0] = sbuf[warp][0]; s.blk[1] = sbuf[warp][1]; s.lane = lane;
    for (int k = lane; k < MT_N; k += 32) s.blk[0][k] = st[k];
    __syncwarp();
    int pos = (int)st[MT_N];
    for (int q = lane; q < MT_N - MT_M; q += 32) {
        uint32_t x[3];
        const int nw = mt_regenerate_words(s.blk[0], q, x);
        for (int w = 0; w < nw; w++) s.blk[1][q + w * (MT_N - MT_M)] = x[w];
    }
    __syncwarp();

    auto next = [&]() -> uint32_t { s.ensure(&pos, pos + 1); return s.word(pos++); };
    int h0, hc;
    stream_chunk(p.hyps, p.n_streams, t, &h0, &hc);
    const int cells = p.nx * p.ny;
    for (int i = 0; i < p.n_images; i++) {
        if (t == 0) {
            const int f = (int)s.draw(&pos, (uint32_t)p.n_frames);
            if (lane == 0) p.img[i] = f;
            int32_t* px = p.pix + (size_t)i * DSAC_N_CONST * 2;
            for (int c0 = 0; c0 < cells; c0 += 32) {
                const int m = min(32, cells - c0);
                s.ensure(&pos, pos + 4 * m);
                const int c = c0 + lane, sx = c / p.ny, sy = c - sx * p.ny;
                if (lane < m && sx < DSAC_GRID_CONST && sy < DSAC_GRID_CONST) {
                    const int q = pos + 4 * lane;
                    const double x0 = sx ? p.xb[sx - 1] : 21.f, x1 = p.xb[sx];
                    const double y0 = sy ? p.yb[sy - 1] : 21.f, y1 = p.yb[sy];
                    const int cx = (int)uniform_real(canonical53(s.word(q), s.word(q + 1)), x0, x1);
                    const int cy = (int)uniform_real(canonical53(s.word(q + 2), s.word(q + 3)), y0, y1);
                    px[(sy * DSAC_GRID_CONST + sx) * 2] = cx;
                    px[(sy * DSAC_GRID_CONST + sx) * 2 + 1] = cy;
                }
                pos += 4 * m;
            }
        }
        for (int h = h0; h < h0 + hc; h++) {
            const size_t k = (size_t)i * p.hyps + h;
            const int drift = (int)s.draw(&pos, 2u);   // irand(0, 2)
            double v[6];
            if (drift == 0) score_rand_hyp(2.f, 2.f, next, v);
            else score_rand_hyp(10.f, 100.f, next, v);
            if (lane == 0) {
                p.drift[k] = drift;
                for (int j = 0; j < 6; j++) p.noise[k * 6 + j] = v[j];
            }
        }
    }
    __syncwarp();
    const bool second = pos > MT_N;
    const uint32_t* b = second ? s.blk[1] : s.blk[0];
    for (int k = lane; k < MT_N; k += 32) st[k] = b[k];
    if (lane == 0) st[MT_N] = (uint32_t)(second ? pos - MT_N : pos);
}

// ----------------------------------------------------------------------------- error images and labels
struct ScoreMapsParams {
    const int32_t* img;      // [n_images]
    const double* gt_jp;     // [F][12]
    const int16_t* coords;   // [n_images][1600][3] mm
    const int32_t* pix;      // [n_images][1600][2]
    const double* noise;     // [n_images * hyps][6]
    int hyps;
    double f;
    float cxf, cyf, temperature;
    const ObjCam* cams;      // [n_cams] per-dataset cameras, indexed by img (k_score_maps_cam only)
    int n_cams;
    float* maps;             // [n_images * hyps][1600]
    double* labels;          // [n_images * hyps]
    int32_t* correct;        // [n_images * hyps] or null
};

constexpr int SM_THREADS = 320;
constexpr int SM_PTS = DSAC_N_CONST / SM_THREADS;

// One CTA per (image, hypothesis): thread 0 builds the noisy pose, its label and its projection rows; every thread then
// projects 5 of the 1600 cells with score_pair_error, the function K2 applies to the forward's diffmaps.
// TABLE: the camera is score_cam of frame img[i]'s entry in the per-dataset table; an img[i] outside the table is not
// read and gives a NaN map and label and correct = 0.
template <bool TABLE>
__device__ __forceinline__ void score_maps_body(const ScoreMapsParams& p) {
    __shared__ float s_P[12];
    const size_t k = blockIdx.x;
    const int i = (int)(k / (size_t)p.hyps);
    double f = p.f;
    float cxf = p.cxf, cyf = p.cyf;
    if constexpr (TABLE) {
        const int fr = p.img[i];
        if (fr < 0 || fr >= p.n_cams) {
            float* out = p.maps + k * DSAC_N_CONST;
            for (int pt = threadIdx.x; pt < DSAC_N_CONST; pt += SM_THREADS) out[pt] = __int_as_float(0x7fffffff);
            if (threadIdx.x == 0) {
                p.labels[k] = __longlong_as_double(0x7fffffffffffffffll);
                if (p.correct) p.correct[k] = 0;
            }
            return;
        }
        const ScoreCam sc = score_cam(p.cams[fr]);
        f = sc.f; cxf = sc.cx; cyf = sc.cy;
    }
    if (threadIdx.x == 0) {
        ScoreSample smp;
        score_sample(p.gt_jp + (size_t)p.img[i] * 12, p.noise + k * 6, f, p.temperature, &smp);
        for (int j = 0; j < 12; j++) s_P[j] = smp.P[j];
        p.labels[k] = smp.label;
        if (p.correct) p.correct[k] = smp.correct;
    }
    __syncthreads();
    const int16_t* c = p.coords + (size_t)i * DSAC_N_CONST * 3;
    const int2* px = reinterpret_cast<const int2*>(p.pix + (size_t)i * DSAC_N_CONST * 2);
    float* out = p.maps + k * DSAC_N_CONST;
#pragma unroll
    for (int j = 0; j < SM_PTS; j++) {
        const int pt = threadIdx.x + j * SM_THREADS;
        const int2 q = __ldg(px + pt);
        float az;
        out[pt] = score_pair_error<true>(s_P[0], s_P[1], s_P[2], s_P[3], s_P[4], s_P[5], s_P[6], s_P[7], s_P[8], s_P[9],
                                         s_P[10], s_P[11], (float)__ldg(c + pt * 3), (float)__ldg(c + pt * 3 + 1),
                                         (float)__ldg(c + pt * 3 + 2), (float)q.x - cxf, (float)q.y - cyf, &az);
    }
}
__global__ void __launch_bounds__(SM_THREADS) k_score_maps(ScoreMapsParams p) { score_maps_body<false>(p); }
__global__ void __launch_bounds__(SM_THREADS) k_score_maps_cam(ScoreMapsParams p) { score_maps_body<true>(p); }

#endif  // device code

}  // namespace dsac
