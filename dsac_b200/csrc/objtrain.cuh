// objtrain.cuh -- the data path of the coordinate CNN's pre-training (the reference's train_obj.cpp) on the device:
//   * k_register_depth:   Dataset::getDepth with rawData (dataset.h:180-202, mapDepthToRGB :93-111)
//   * k_obj_coords:       Dataset::getObj (dataset.h:226-255): pxToEye (dataset.cpp:37-56) then Hypothesis::invTransform
//   * k_obj_draw:         assembleData's random draw (train_obj.cpp:47-102): image index, then accepted patch centres
//   * k_gather_patches_at: the patch gather of upstream.cuh at per-patch (frame, x, y) into a device-resident dataset
// The first three have _cam instantiations that take each frame's camera from the per-dataset table
// (dsac_set_dataset_cameras); the instantiations without it are the single-camera code.
// The per-pixel arithmetic is in DSAC_HD functions, so that the host build (tests/host_shim) can be checked against the
// numpy restatement on a machine without a GPU.  Every operation is spelled with a round-to-nearest intrinsic on the
// device so that nvcc cannot contract it into an FMA the x86 reference never executes.
#pragma once
#include "sampler.cuh"
#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
#include "upstream.cuh"
#endif

namespace dsac {

#if defined(__CUDA_ARCH__)
#define OT_DADD(a, b) __dadd_rn((a), (b))
#define OT_DSUB(a, b) __dsub_rn((a), (b))
#define OT_DMUL(a, b) __dmul_rn((a), (b))
#define OT_DDIV(a, b) __ddiv_rn((a), (b))
#define OT_FADD(a, b) __fadd_rn((a), (b))
#define OT_FSUB(a, b) __fsub_rn((a), (b))
#define OT_FDIV(a, b) __fdiv_rn((a), (b))
#else
#define OT_DADD(a, b) ((a) + (b))
#define OT_DSUB(a, b) ((a) - (b))
#define OT_DMUL(a, b) ((a) * (b))
#define OT_DDIV(a, b) ((a) / (b))
#define OT_FADD(a, b) ((a) + (b))
#define OT_FSUB(a, b) ((a) - (b))
#define OT_FDIV(a, b) ((a) / (b))
#endif

constexpr int OBJ_HALF = 42 / 2;            // inputSize / 2 (train_obj.cpp:77-78)
constexpr int OBJ_STATE_WORDS = MT_N + 1;   // one stream's std::mt19937: 624 state words and the position _M_p

struct ObjCam {
    float focal, x_shift, y_shift;                      // the RGB camera (dP.focalLength, xShift, yShift)
    float secondary_focal, raw_x_shift, raw_y_shift;    // the depth camera (dP.secondaryFocalLength, rawXShift, rawYShift)
    double sensor_trans[16];                            // depth -> RGB, row-major 4x4 (dP.sensorTrans)
    int raw_data, width, height;                        // dP.rawData, dP.imageWidth, dP.imageHeight
};

// x86-64 truncating conversions as gcc emits them for (int) / (short) of a float or double: cvttss2si / cvttsd2si to 32
// bits, which yields INT_MIN for NaN and out-of-range values; (short) then keeps the low 16 bits.  The device's own
// conversions saturate instead, so the range test comes first.
DSAC_HD int cvtt_f2i(float v) {
    if (!(v > -2147483904.f && v < 2147483648.f)) return (int)0x80000000u;
    return (int)v;
}
DSAC_HD int cvtt_d2i(double v) {
    if (!(v > -2147483649.0 && v < 2147483648.0)) return (int)0x80000000u;
    return (int)v;
}
DSAC_HD int16_t low16(int v) { return (int16_t)(uint16_t)((uint32_t)v & 0xffffu); }

// cv::Vec3f /= 1000 (train_obj.cpp:95): OpenCV's Vec::operator/=(int) multiplies by the double 1./alpha and converts the
// double product back with saturate_cast<float> (a plain rounding conversion), so it is not v / 1000.f.
DSAC_HD float mm_to_m(int16_t v) { return (float)OT_DMUL((double)(float)v, 1. / 1000); }

// The inverse of the ground-truth rotation as cv::Mat::inv computes it for a 3x3 CV_64F matrix: OpenCV's closed form
// (d = 1/det3, cofactors times d), not an elimination.
DSAC_HD void obj_inv_rotation(const double* m, double r[9]) {
    const double c00 = OT_DSUB(OT_DMUL(m[4], m[8]), OT_DMUL(m[5], m[7]));
    const double c10 = OT_DSUB(OT_DMUL(m[3], m[8]), OT_DMUL(m[5], m[6]));
    const double c20 = OT_DSUB(OT_DMUL(m[3], m[7]), OT_DMUL(m[4], m[6]));
    double d = OT_DADD(OT_DSUB(OT_DMUL(m[0], c00), OT_DMUL(m[1], c10)), OT_DMUL(m[2], c20));
    d = OT_DDIV(1., d);
    r[0] = OT_DMUL(c00, d);
    r[1] = OT_DMUL(OT_DSUB(OT_DMUL(m[2], m[7]), OT_DMUL(m[1], m[8])), d);
    r[2] = OT_DMUL(OT_DSUB(OT_DMUL(m[1], m[5]), OT_DMUL(m[2], m[4])), d);
    r[3] = OT_DMUL(OT_DSUB(OT_DMUL(m[5], m[6]), OT_DMUL(m[3], m[8])), d);
    r[4] = OT_DMUL(OT_DSUB(OT_DMUL(m[0], m[8]), OT_DMUL(m[2], m[6])), d);
    r[5] = OT_DMUL(OT_DSUB(OT_DMUL(m[2], m[3]), OT_DMUL(m[0], m[5])), d);
    r[6] = OT_DMUL(c20, d);
    r[7] = OT_DMUL(OT_DSUB(OT_DMUL(m[1], m[6]), OT_DMUL(m[0], m[7])), d);
    r[8] = OT_DMUL(OT_DSUB(OT_DMUL(m[0], m[4]), OT_DMUL(m[1], m[3])), d);
}

// One frame's ground truth in the form getObj uses it: Hypothesis(info) keeps translation = center * 1e3 (mm) and
// invRotation = rotation.inv().  pose: the jp pose [12] of dsac_forward's gt_jp = row-major rotation, then the
// translation in mm.  jp::info_t holds the rotation and the centre (metres) in float (types.h), so the rotation is
// rounded to float and the translation taken through float(t / 1000), which recovers the pose file's float centre.
struct ObjPose {
    double rinv[9], t[3];
};
DSAC_HD void obj_pose(const double* pose, ObjPose* p) {
    double r[9];
    for (int k = 0; k < 9; k++) r[k] = (double)(float)pose[k];
    obj_inv_rotation(r, p->rinv);
    for (int k = 0; k < 3; k++) p->t[k] = OT_DMUL((double)(float)OT_DDIV(pose[9 + k], 1000.), 1e3);
}

// getObj at one pixel of the registered depth image: zero for depth 0; otherwise pxToEye in float with (short)
// conversions, Point3d, p - translation, invRotation * p (gemm order: 0 + a0 b0 + a1 b1 + a2 b2), and (short) of each
// double.
DSAC_HD void obj_coord(const ObjCam& c, const ObjPose& p, int x, int y, uint16_t depth, int16_t out[3]) {
    if (depth == 0) { out[0] = out[1] = out[2] = 0; return; }
    const float fd = OT_FDIV(c.focal, (float)depth);
    const float cx = OT_FADD((float)c.width / 2.f, c.x_shift), cy = OT_FADD((float)c.height / 2.f, c.y_shift);
    const int16_t e0 = low16(cvtt_f2i(OT_FDIV(OT_FSUB((float)x, cx), fd)));
    const int16_t e1 = low16(cvtt_f2i(-OT_FDIV(OT_FSUB((float)y, cy), fd)));
    const int16_t e2 = low16(-(int)depth);
    const double q[3] = {OT_DSUB((double)e0, p.t[0]), OT_DSUB((double)e1, p.t[1]), OT_DSUB((double)e2, p.t[2])};
    for (int r = 0; r < 3; r++) {
        double s = OT_DMUL(p.rinv[3 * r], q[0]);
        s = OT_DADD(s, OT_DMUL(p.rinv[3 * r + 1], q[1]));
        s = OT_DADD(s, OT_DMUL(p.rinv[3 * r + 2], q[2]));
        out[r] = low16(cvtt_d2i(s));
    }
}

DSAC_HD bool on_obj(const int16_t v[3]) { return v[0] != 0 || v[1] != 0 || v[2] != 0; }

// mapDepthToRGB for one nonzero raw depth: the depth arrives as a short (so >= 32768 is negative), is back-projected in
// double with the depth camera, moved by sensorTrans (gemm order, eye(3) = 1) and projected with the RGB camera;
// (int)(... + 0.5) truncates toward zero.  Writes the target pixel.
DSAC_HD void map_depth_to_rgb(const ObjCam& c, int x, int y, uint16_t raw, int* nx, int* ny) {
    const double depth = (double)(int16_t)raw;
    const double sf = OT_DDIV((double)c.secondary_focal, depth);
    double eye[4];
    eye[0] = OT_DDIV(OT_DSUB((double)x, OT_DADD((double)c.width / 2.0, (double)c.raw_x_shift)), sf);
    eye[1] = -OT_DDIV(OT_DSUB((double)y, OT_DADD((double)c.height / 2.0, (double)c.raw_y_shift)), sf);
    eye[2] = -depth;
    eye[3] = 1.0;
    double m[2];
    for (int r = 0; r < 2; r++) {
        double s = OT_DMUL(c.sensor_trans[4 * r], eye[0]);
        for (int k = 1; k < 4; k++) s = OT_DADD(s, OT_DMUL(c.sensor_trans[4 * r + k], eye[k]));
        m[r] = s;
    }
    const double f = OT_DDIV((double)c.focal, depth);
    const double cx = (double)OT_FADD((float)c.width / 2.f, c.x_shift), cy = (double)OT_FADD((float)c.height / 2.f, c.y_shift);
    *nx = cvtt_d2i(OT_DADD(OT_DADD(OT_DMUL(m[0], f), cx), 0.5));
    *ny = cvtt_d2i(OT_DADD(OT_DADD(-OT_DMUL(m[1], f), cy), 0.5));
}

// One libstdc++ uniform_int_distribution draw over `range` values (range >= 1) from a 32-bit generator: Lemire's
// multiply-and-reject (bits/uniform_int_dist.h, _S_nd).  `next` yields the generator's words.
template <class Next>
DSAC_HD uint32_t lemire_draw(uint32_t range, Next&& next) {
    uint64_t product = (uint64_t)next() * range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
        const uint32_t threshold = (0u - range) % range;
        while (low < threshold) {
            product = (uint64_t)next() * range;
            low = (uint32_t)product;
        }
    }
    return (uint32_t)(product >> 32);
}

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)

// ----------------------------------------------------------------------------- registration
// Pass 1 (one thread per source pixel): the target of each nonzero depth.  The reference writes in the order x outer,
// y inner, so the last source pixel in that order wins; the 64-bit key ((x * rows + y) << 16) | depth ordered by
// atomicMax keeps exactly that one.  Targets outside the image (undefined behaviour in the reference) are dropped and
// counted per frame.  With raw_data = 0 the depth passes through.
// TABLE: the per-dataset camera table (dsac_set_dataset_cameras) gives each frame its own mapping; `c` still holds the
// frame size and raw_data, which every entry shares.
template <bool TABLE>
__device__ __forceinline__ void register_depth_body(const ObjCam& c, const ObjCam* __restrict__ cams, int n,
                                                    const uint16_t* __restrict__ raw, uint64_t* __restrict__ keys,
                                                    uint16_t* __restrict__ out, int32_t* __restrict__ dropped) {
    const int W = c.width, H = c.height;
    const size_t plane = (size_t)W * H;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plane * n) return;
    const int f = (int)(i / plane);
    const int pix = (int)(i - (size_t)f * plane), y = pix / W, x = pix - y * W;
    const uint16_t d = raw[i];
    if (!c.raw_data) { out[i] = d; return; }
    if (d == 0) return;
    int nx, ny;
    if constexpr (TABLE) map_depth_to_rgb(cams[f], x, y, d, &nx, &ny);
    else map_depth_to_rgb(c, x, y, d, &nx, &ny);
    if (nx < 0 || ny < 0 || nx >= W || ny >= H) {
        if (dropped) atomicAdd(dropped + f, 1);
        return;
    }
    const unsigned long long key = ((unsigned long long)((uint32_t)x * (uint32_t)H + (uint32_t)y) << 16) | d;
    atomicMax(reinterpret_cast<unsigned long long*>(keys) + (size_t)f * plane + (size_t)ny * W + nx, key);
}
__global__ void k_register_depth(ObjCam c, int n, const uint16_t* __restrict__ raw, uint64_t* __restrict__ keys,
                                 uint16_t* __restrict__ out, int32_t* __restrict__ dropped) {
    register_depth_body<false>(c, nullptr, n, raw, keys, out, dropped);
}
__global__ void k_register_depth_cam(ObjCam c, const ObjCam* __restrict__ cams, int n, const uint16_t* __restrict__ raw,
                                     uint64_t* __restrict__ keys, uint16_t* __restrict__ out, int32_t* __restrict__ dropped) {
    register_depth_body<true>(c, cams, n, raw, keys, out, dropped);
}

// Pass 2: the registered depth is the winning key's low 16 bits (0 where nothing landed).
__global__ void k_register_finish(size_t count, const uint64_t* __restrict__ keys, uint16_t* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = (uint16_t)(keys[i] & 0xffffu);
}

// ----------------------------------------------------------------------------- getObj
// A listed frame outside [0, n_frames) yields a zero image (the entry point documents it; RGBDScene refuses such lists).
// TABLE: the camera of frame idx[k] from the per-dataset table, read only for a frame inside the dataset.
template <bool TABLE>
__device__ __forceinline__ void obj_coords_body(const ObjCam& c, const ObjCam* __restrict__ cams, int n_frames, int n,
                                                const int32_t* __restrict__ idx, const uint16_t* __restrict__ depth,
                                                const double* __restrict__ poses, int16_t* __restrict__ out) {
    const int W = c.width, H = c.height;
    const size_t plane = (size_t)W * H;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plane * n) return;
    const int k = (int)(i / plane);
    const int f = idx ? idx[k] : k;
    if (f < 0 || f >= n_frames) { out[i * 3] = out[i * 3 + 1] = out[i * 3 + 2] = 0; return; }
    const int pix = (int)(i - (size_t)k * plane), y = pix / W, x = pix - y * W;
    ObjPose p;
    obj_pose(poses + (size_t)f * 12, &p);
    int16_t v[3];
    if constexpr (TABLE) obj_coord(cams[f], p, x, y, depth[(size_t)f * plane + pix], v);
    else obj_coord(c, p, x, y, depth[(size_t)f * plane + pix], v);
    out[i * 3] = v[0]; out[i * 3 + 1] = v[1]; out[i * 3 + 2] = v[2];
}
__global__ void k_obj_coords(ObjCam c, int n_frames, int n, const int32_t* __restrict__ idx, const uint16_t* __restrict__ depth,
                             const double* __restrict__ poses, int16_t* __restrict__ out) {
    obj_coords_body<false>(c, nullptr, n_frames, n, idx, depth, poses, out);
}
__global__ void k_obj_coords_cam(ObjCam c, const ObjCam* __restrict__ cams, int n_frames, int n, const int32_t* __restrict__ idx,
                                 const uint16_t* __restrict__ depth, const double* __restrict__ poses, int16_t* __restrict__ out) {
    obj_coords_body<true>(c, cams, n_frames, n, idx, depth, poses, out);
}

// ----------------------------------------------------------------------------- ThreadRand state
__global__ void k_obj_rng_init(uint32_t seed, int T, uint32_t* __restrict__ state) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    uint32_t* s = state + (size_t)t * OBJ_STATE_WORDS;
    mt_seed(s, seed + (uint32_t)t);   // ThreadRand::init: generators[i].seed(i + seed)
    s[MT_N] = MT_N;                   // a freshly seeded engine twists before its first word
}

// ----------------------------------------------------------------------------- assembleData's draw
struct ObjDrawParams {
    ObjCam cam;                // the camera; with a table, its frame size (which every entry shares)
    const ObjCam* cams;        // [n_frames] per-dataset cameras (k_obj_draw_cam only)
    const uint16_t* depth;     // [F][H][W] registered depth
    const double* poses;       // [F][12] jp poses
    int n_frames, n_images, n_patches, n_streams, max_attempts;
    uint32_t* state;           // [T][625] std::mt19937 words + position, read and written back
    int32_t* img;              // [n_images * n_patches]
    int32_t* centre;           // [n_images * n_patches][2] (x, y); (-1, -1) for a patch an exhausted image could not draw
    float* label;              // [n_images * n_patches][3] metres
    uint32_t* status;          // [n_images] DSAC_ST_OBJ_DRAW_EXHAUSTED
};

constexpr int OBJ_DRAW_WARPS = 4;

// A warp's window on its stream: two consecutive 624-word blocks of raw (untempered) state, addressed by a position
// relative to the first.  advance() drops the first block and twists the one after the second in its place.
struct ObjStream {
    uint32_t* blk[2];
    int lane;
    __device__ uint32_t word(int p) const { return mt_temper(p < MT_N ? blk[0][p] : blk[1][p - MT_N]); }
    __device__ void advance() {
        __syncwarp();   // every lane is done reading the block about to be overwritten
        uint32_t* so = blk[1];
        uint32_t* dst = blk[0];
        for (int t = lane; t < MT_N - MT_M; t += 32) {
            uint32_t x[3];
            const int nw = mt_regenerate_words(so, t, x);
            for (int w = 0; w < nw; w++) dst[t + w * (MT_N - MT_M)] = x[w];
        }
        __syncwarp();
        blk[0] = so; blk[1] = dst;
    }
    // make words up to position q (exclusive) addressable; every lane calls it with the same arguments
    __device__ void ensure(int* pos, int q) {
        while (q > 2 * MT_N) { advance(); *pos -= MT_N; q -= MT_N; }
    }
    __device__ uint32_t draw(int* pos, uint32_t range) {
        return lemire_draw(range, [&]() { ensure(pos, *pos + 1); return word((*pos)++); });
    }
};

// One warp per stream t (std::mt19937(seed + t) of ThreadRand); the stream owns images by libgomp's static schedule.
// Per image: irand(0, F), then n_patches accepted centres, each from a loop of irand(21, W - 21), irand(21, H - 21) until
// the centre's label is on the object.  The draw counts depend on the data, so a warp evaluates 32 candidate pairs at once
// -- lane l takes the words pos + 2l, pos + 2l + 1 -- and keeps the accepted ones in order (ballot, prefix count).  That
// pairing holds only while no word is a Lemire rejection; the first lane whose pair contains one ends the batch there and
// the pair at that point is drawn sequentially (rejections are rare: threshold / 2^32 per word).  A patch that is still
// unmet after max_attempts (>= 32) pairs ends its image with DSAC_ST_OBJ_DRAW_EXHAUSTED; the reference would loop forever.
// TABLE: once the warp has drawn an image's frame it loads that frame's camera for the labels; the words consumed are
// the same.
template <bool TABLE>
__device__ __forceinline__ void obj_draw_body(const ObjDrawParams& p) {
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
    // block 1 = the twist of block 0 (the same routine as advance, into the second buffer)
    for (int q = lane; q < MT_N - MT_M; q += 32) {
        uint32_t x[3];
        const int nw = mt_regenerate_words(s.blk[0], q, x);
        for (int w = 0; w < nw; w++) s.blk[1][q + w * (MT_N - MT_M)] = x[w];
    }
    __syncwarp();

    int i0, cnt;
    stream_chunk(p.n_images, p.n_streams, t, &i0, &cnt);
    const ObjCam& c = p.cam;
    const uint32_t rx = (uint32_t)(c.width - 2 * OBJ_HALF), ry = (uint32_t)(c.height - 2 * OBJ_HALF);
    const uint32_t thx = (0u - rx) % rx, thy = (0u - ry) % ry;
    const size_t plane = (size_t)c.width * c.height;
    const unsigned lt = (1u << lane) - 1u;
    for (int i = i0; i < i0 + cnt; i++) {
        const int f = (int)s.draw(&pos, (uint32_t)p.n_frames);
        ObjPose pose;
        obj_pose(p.poses + (size_t)f * 12, &pose);
        ObjCam fc;   // TABLE: the fields getObj reads, of frame f
        if constexpr (TABLE) {
            const ObjCam* t = p.cams + f;
            fc.focal = t->focal; fc.x_shift = t->x_shift; fc.y_shift = t->y_shift;
            fc.width = c.width; fc.height = c.height;
        }
        const ObjCam& lc = TABLE ? fc : c;
        const uint16_t* dep = p.depth + (size_t)f * plane;
        const size_t out0 = (size_t)i * p.n_patches;
        int done = 0, attempts = 0;
        bool exhausted = false;
        auto emit = [&](int slot, int x, int y, const int16_t v[3]) {
            p.img[out0 + slot] = f;
            p.centre[(out0 + slot) * 2] = x; p.centre[(out0 + slot) * 2 + 1] = y;
            for (int k = 0; k < 3; k++) p.label[(out0 + slot) * 3 + k] = mm_to_m(v[k]);
        };
        while (done < p.n_patches) {
            s.ensure(&pos, pos + 64);
            const int q = pos + 2 * lane;
            const uint64_t px = (uint64_t)s.word(q) * rx, py = (uint64_t)s.word(q + 1) * ry;
            const bool rej = ((uint32_t)px < thx) || ((uint32_t)py < thy);
            const int x = (int)(px >> 32) + OBJ_HALF, y = (int)(py >> 32) + OBJ_HALF;
            int16_t v[3];
            obj_coord(lc, pose, x, y, dep[(size_t)y * c.width + x], v);
            const bool acc = !rej && on_obj(v);
            const unsigned rmask = __ballot_sync(0xffffffffu, rej);
            const int r = rmask ? __ffs(rmask) - 1 : 32;
            unsigned amask = __ballot_sync(0xffffffffu, acc) & (r == 32 ? 0xffffffffu : ((1u << r) - 1u));
            if (amask) {
                const int a0 = __ffs(amask) - 1;
                if (attempts + a0 >= p.max_attempts) { pos += 2 * (p.max_attempts - attempts); exhausted = true; break; }
                const int need = p.n_patches - done;
                while (__popc(amask) > need) amask &= ~(1u << (31 - __clz(amask)));
                if ((amask >> lane) & 1u) emit(done + __popc(amask & lt), x, y, v);
                const int last = 31 - __clz(amask);
                done += __popc(amask);
                if (done == p.n_patches) { pos += 2 * (last + 1); break; }
                pos += 2 * r;
                attempts = r - 1 - last;
            } else {
                const int k = min(r, p.max_attempts - attempts);
                pos += 2 * k;
                attempts += k;
                if (attempts == p.max_attempts) { exhausted = true; break; }
            }
            if (r < 32) {   // the pair with a rejected word, drawn word by word
                const int sx = (int)s.draw(&pos, rx) + OBJ_HALF;
                const int sy = (int)s.draw(&pos, ry) + OBJ_HALF;
                attempts++;
                int16_t w[3];
                obj_coord(lc, pose, sx, sy, dep[(size_t)sy * c.width + sx], w);
                if (on_obj(w)) {
                    if (lane == 0) emit(done, sx, sy, w);
                    done++;
                    attempts = 0;
                } else if (attempts == p.max_attempts && done < p.n_patches) {
                    exhausted = true;
                    break;
                }
            }
        }
        if (exhausted) {
            const int16_t z[3] = {0, 0, 0};
            for (int k = done + lane; k < p.n_patches; k += 32) emit(k, -1, -1, z);
        }
        if (lane == 0) p.status[i] = exhausted ? 8u /* DSAC_ST_OBJ_DRAW_EXHAUSTED */ : 0u;
    }
    // hand the engine back as std::mt19937 holds it: the block of the last word consumed and the index after it
    __syncwarp();
    const bool second = pos > MT_N;
    const uint32_t* b = second ? s.blk[1] : s.blk[0];
    for (int k = lane; k < MT_N; k += 32) st[k] = b[k];
    if (lane == 0) st[MT_N] = (uint32_t)(second ? pos - MT_N : pos);
}
__global__ void __launch_bounds__(32 * OBJ_DRAW_WARPS) k_obj_draw(ObjDrawParams p) { obj_draw_body<false>(p); }
__global__ void __launch_bounds__(32 * OBJ_DRAW_WARPS) k_obj_draw_cam(ObjDrawParams p) { obj_draw_body<true>(p); }

// ----------------------------------------------------------------------------- patch gather at listed centres
struct GatherAtParams {
    const uint8_t* frames;    // [F][height][width][3] BGR
    int width, height, n_frames;
    const int32_t* frame;     // [n] frame of each patch
    const int32_t* centre;    // [n][2] (x, y)
    float mean;
    float* patches;           // [n][3][42][42]
    uint32_t* status;         // [1] or null: DSAC_ST_BORDER_PATCH
};

// k_gather_patches with the frame and centre read per patch: the same row loads, byte -> float conversion, shared
// memory layout and bulk store, so a patch is bit for bit what k_gather_patches makes at that centre.  assembleData
// copies patch(y, x) = image(cy - 21 + y, cx - 21 + x) (train_obj.cpp:83-91), the same window.
__global__ void __launch_bounds__(UP_THREADS) k_gather_patches_at(GatherAtParams p) {
    __shared__ __align__(128) float sf[UP_ELEMS];
    const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int fr = p.frame[n], ox = p.centre[2 * n], oy = p.centre[2 * n + 1];
    const int half = UP_PATCH / 2;
    const bool border = fr < 0 || fr >= p.n_frames || (ox < half) || (oy < half) || (ox > p.width - half) ||
                        (oy > p.height - half);
    float* out = p.patches + (size_t)n * UP_ELEMS;
    if (border) {
        if (tid == 0 && p.status) atomicOr(p.status, 4u /* DSAC_ST_BORDER_PATCH */);
        float4* out4 = reinterpret_cast<float4*>(out);
        for (int q = tid; q < UP_ELEMS / 4; q += UP_THREADS) __stcs(out4 + q, make_float4(0.f, 0.f, 0.f, 0.f));
        return;
    }
    const size_t row_bytes = (size_t)p.width * 3;
    const uint8_t* row0 = p.frames + ((size_t)fr * p.height + (oy - half)) * row_bytes + (size_t)(ox - half) * 3;
    int off[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int e = 4 * lane + j, x = e / 3, c = e - 3 * x;
        off[j] = c * UP_PLANE + x;
    }
    uint32_t w0[UP_ROWS_PER_WARP], w1x[UP_ROWS_PER_WARP], sh8[UP_ROWS_PER_WARP];
#pragma unroll
    for (int k = 0; k < UP_ROWS_PER_WARP; k++) {
        const int r = warp + k * (UP_THREADS / 32);
        w0[k] = 0u; w1x[k] = 0u; sh8[k] = 0u;
        if (r < UP_PATCH) {
            const uint8_t* src = row0 + (size_t)r * row_bytes;
            const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u);
            const uint8_t* base = src - sh;
            w0[k] = __ldg(reinterpret_cast<const uint32_t*>(base) + lane);
            if (lane == 31 && sh == 3u) w1x[k] = (uint32_t)__ldg(base + 128);
            sh8[k] = sh * 8u;
        }
    }
    const float magic = 8388608.f;
#pragma unroll
    for (int k = 0; k < UP_ROWS_PER_WARP; k++) {
        const int r = warp + k * (UP_THREADS / 32);
        uint32_t nb = __shfl_down_sync(0xffffffffu, w0[k], 1);
        if (lane == 31) nb = w1x[k];
        if (r < UP_PATCH) {
            const uint32_t v = __funnelshift_r(w0[k], nb, sh8[k]);
            float* dst = sf + r * UP_PATCH;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (j < 2 || lane < 31) {
                    const float fb = __uint_as_float(0x4B000000u | ((v >> (8 * j)) & 0xffu)) - magic;
                    dst[off[j]] = fb - p.mean;
                }
            }
        }
    }
    __syncthreads();
    if (tid == 0) up_bulk_store(out, sf, (uint32_t)(UP_ELEMS * sizeof(float)));
}

#endif  // device code

}  // namespace dsac
