"""Freezes tests/golden/ref_obj.npz: what the reference's OWN train_obj.cpp and jp::Dataset compute on small synthetic
RGB-D datasets -- registered depth (getDepth), scene coordinates (getObj), the pose reader's jp::info_t, two consecutive
assembleData rounds for T = 1 and 3 OpenMP threads, and the batch permutation.

    DSAC_REFERENCE=/path/to/reference/core python tests/golden/make_ref_obj.py

The reference is compiled unmodified (tests/golden/ref_obj/ref_train_obj.cpp includes train_obj.cpp with main renamed)
against the API shims of oracle/shim and the png++ stand-in of tests/golden/ref_obj, which serves pixel buffers
registered by path.  Frames are coded (tests/obj_oracle.coded_bgr), so a patch's pixels give its frame and centre back;
raw depth comes from tests/obj_oracle.fixture_depth (integer hashing), so the tests rebuild the inputs without storing
them.  Large outputs are kept as SHA-256 digests of their bytes, with the first rows beside them."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import obj_oracle as OO   # noqa: E402

N_IMAGES, N_PATCHES = 10, 48
CASES = [  # name, W, H, F, sensorTrans, rawData, x_shift, draw thread counts
    ("small_identity", 128, 96, 5, "identity", 1, 0.0, (1, 3)),
    ("small_7scenes", 128, 96, 5, "7scenes", 1, 0.5, (1, 3)),
    ("small_raw0", 128, 96, 4, "7scenes", 0, 0.0, (3,)),
    ("vga_7scenes", 640, 480, 4, "7scenes", 1, 0.0, (1, 3)),
]
SEED = 1305


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def sensor_trans(kind):
    if kind == "identity":
        return np.eye(4)
    b = open(os.path.join(HERE, "sensorTrans_7scenes.dat"), "rb").read()
    return np.frombuffer(b[8:], np.float64).reshape(4, 4).copy()


def build(ref, out_dir):
    so = os.path.join(out_dir, "libref_train_obj.so")
    odir = os.path.join(ROOT, "oracle")
    subprocess.check_call(["make", "-C", odir, "-s", "libdsac_oracle.so"])
    srcs = [os.path.join(ref, f) for f in ("Hypothesis.cpp", "properties.cpp", "thread_rand.cpp", "util.cpp", "read_data.cpp",
                                           "dataset.cpp")]
    cmd = ["g++", "-O2", "-std=c++11", "-fPIC", "-fopenmp", "-ffp-contract=off", "-w",
           "-I" + os.path.join(HERE, "ref_obj"), "-I" + os.path.join(odir, "shim"), "-I" + ref, "-I" + odir,
           "-I" + os.path.join(odir, "ref_harness"), "-shared", "-o", so, os.path.join(HERE, "ref_obj", "ref_train_obj.cpp"),
           *srcs, "-L" + odir, "-ldsac_oracle", "-Wl,-rpath," + odir]
    subprocess.check_call(cmd)
    return C.CDLL(so)


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def main():
    ref = os.environ.get("DSAC_REFERENCE", "")
    if not os.path.exists(os.path.join(ref, "train_obj.cpp")):
        sys.exit("DSAC_REFERENCE must name the core/ directory of a checkout of the reference")
    from scipy.spatial.transform import Rotation
    tmp = tempfile.mkdtemp()
    lib = build(ref, tmp)
    out = {"n_images": np.int32(N_IMAGES), "n_patches": np.int32(N_PATCHES), "seed": np.uint32(SEED)}
    rng = np.random.default_rng(20170721)
    cwd = os.getcwd()
    os.chdir(tmp)   # no translation.txt here: the pose reader uses the pose files as they are
    try:
        for name, W, H, F, trans, raw_data, xs, threads in CASES:
            base = os.path.join(tmp, name)
            for d in ("rgb_noseg", "depth_noseg", "poses"):
                os.makedirs(os.path.join(base, d))
            bgr = OO.coded_bgr(F, H, W)
            raw = OO.fixture_depth(F, H, W, salt=len(name))
            st = sensor_trans(trans)
            cam = dict(focal=525.0, x_shift=xs, y_shift=-xs, secondary_focal=585.0, raw_x_shift=0.0, raw_y_shift=0.0,
                       sensor_trans=st, raw_data=raw_data, width=W, height=H)
            # getDepth writes a target outside the image out of bounds (undefined behaviour that corrupts the heap):
            # such source pixels are set to 0 here, and the mask is kept so that the tests rebuild the same input
            ys, xs_ = np.mgrid[0:H, 0:W]
            outside = np.zeros((F, H, W), bool)
            if raw_data:
                for f in range(F):
                    nx, ny = OO.map_depth_to_rgb(cam, xs_, ys, raw[f])
                    outside[f] = (raw[f] != 0) & ((nx < 0) | (ny < 0) | (nx >= W) | (ny >= H))
            raw[outside] = 0
            out[name + "/zeroed"] = np.packbits(outside)
            for f in range(F):
                stem = "frame-%06d" % f
                cpath = base + "/rgb_noseg/" + stem + ".color.png"
                dpath = base + "/depth_noseg/" + stem + ".depth.png"
                open(cpath, "wb").close()
                open(dpath, "wb").close()
                lib.ref_obj_register_bgr(cpath.encode(), W, H, p(np.ascontiguousarray(bgr[f])))
                lib.ref_obj_register_depth(dpath.encode(), W, H, p(np.ascontiguousarray(raw[f])))
                M = np.eye(4)
                M[:3, :3] = Rotation.from_rotvec(rng.uniform(-1.5, 1.5, 3)).as_matrix()
                M[:3, 3] = rng.uniform(-1.5, 1.5, 3)
                with open(base + "/poses/" + stem + ".pose.txt", "w") as fh:
                    for row in M:
                        fh.write(" ".join("%.9e" % v for v in row) + "\n")
            lib.ref_obj_camera(C.c_float(525), C.c_float(xs), C.c_float(-xs), C.c_float(585), C.c_float(0), C.c_float(0),
                               p(np.ascontiguousarray(st)), raw_data, W, H)
            assert lib.ref_obj_dataset(base.encode()) == F
            reg = np.zeros((F, H, W), np.uint16)
            co = np.zeros((F, H, W, 3), np.int16)
            rot = np.zeros((F, 9), np.float32)
            cen = np.zeros((F, 3), np.float32)
            for f in range(F):
                lib.ref_obj_depth(f, p(reg[f]))
                lib.ref_obj_coords(f, p(co[f]))
                assert lib.ref_obj_info(f, p(rot[f]), p(cen[f])) == 1
            out[name + "/camera"] = np.array([525, xs, -xs, 585, 0, 0, raw_data, W, H], np.float64)
            out[name + "/sensor_trans"] = st
            out[name + "/rotation"] = rot
            out[name + "/center"] = cen
            out[name + "/depth_sha"] = np.stack([digest(reg[f]) for f in range(F)])
            out[name + "/coords_sha"] = np.stack([digest(co[f]) for f in range(F)])
            out[name + "/depth_rows"] = reg[:, :4].copy()
            out[name + "/coords_rows"] = co[:, :2].copy()
            n = N_IMAGES * N_PATCHES
            for T in threads:
                lib.ref_obj_threads(SEED, T)
                for rnd in range(2):
                    corner = np.zeros((n, 3), np.float32)
                    centre = np.zeros((n, 3), np.float32)
                    lab = np.zeros((n, 3), np.float32)
                    lib.ref_obj_assemble(N_IMAGES, N_PATCHES, p(corner), p(centre), p(lab))
                    fr, x0, y0 = OO.decode_bgr(corner.astype(np.uint8))
                    fr2, xc, yc = OO.decode_bgr(centre.astype(np.uint8))
                    assert (fr == fr2).all() and (xc == x0 + 21).all() and (yc == y0 + 21).all()
                    key = "%s/T%d/round%d" % (name, T, rnd)
                    out[key + "/img"] = fr.astype(np.int32)
                    out[key + "/centre"] = np.stack([xc, yc], 1).astype(np.int32)
                    out[key + "/label"] = lab
            print(name, "done", flush=True)
        perm = np.zeros(51200, np.int32)
        lib.ref_obj_permutation(51200, p(perm))
        out["permutation_sha"] = digest(perm)
        out["permutation_head"] = perm[:64].copy()
    finally:
        os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "ref_obj.npz"), **out)
    print("wrote", os.path.join(HERE, "ref_obj.npz"), os.path.getsize(os.path.join(HERE, "ref_obj.npz")), "bytes")


if __name__ == "__main__":
    main()
