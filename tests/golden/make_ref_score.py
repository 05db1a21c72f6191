"""Freezes tests/golden/ref_score.npz: what the reference's OWN train_score.cpp and jp::Dataset compute -- getRandHyp
sequences (which pin the order in which gcc evaluates its constructor arguments) and two consecutive assembleData rounds
for T = 1, 3 and 16 OpenMP threads on small synthetic datasets and at 640x480.

    DSAC_REFERENCE=/path/to/reference/core python tests/golden/make_ref_score.py

The reference is compiled unmodified (tests/golden/ref_score/ref_train_score.cpp includes train_score.cpp with main
renamed) against the API shims of oracle/shim and the png++ stand-in of tests/golden/ref_obj, which serves pixel buffers
registered by path.  Frames are coded (tests/obj_oracle.coded_bgr), so the coordinate CNN's stub sees each patch's frame
and centre and returns a scene coordinate the tests recompute (tests/test_score_ref_fixture.py)."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import obj_oracle as OO   # noqa: E402

N_IMAGES, HYPS = 2, 5
CASES = [  # name, W, H, F, draw thread counts
    ("small", 128, 96, 4, (1, 3, 16)),
    ("vga", 640, 480, 3, (3,)),
]
SEED = 1305
HYP_SEEDS, HYP_N = (1305, 7), 64
FOCAL = 525.0


def build(ref, out_dir):
    so = os.path.join(out_dir, "libref_train_score.so")
    odir = os.path.join(ROOT, "oracle")
    subprocess.check_call(["make", "-C", odir, "-s", "libdsac_oracle.so"])
    srcs = [os.path.join(ref, f) for f in ("Hypothesis.cpp", "properties.cpp", "thread_rand.cpp", "util.cpp", "read_data.cpp",
                                           "dataset.cpp")]
    cmd = ["g++", "-O2", "-std=c++11", "-fPIC", "-fopenmp", "-ffp-contract=off", "-w",
           "-I" + os.path.join(HERE, "ref_obj"), "-I" + os.path.join(odir, "shim"), "-I" + ref, "-I" + odir,
           "-shared", "-o", so, os.path.join(HERE, "ref_score", "ref_train_score.cpp"),
           *srcs, "-L" + odir, "-ldsac_oracle", "-Wl,-rpath," + odir]
    subprocess.check_call(cmd)
    return C.CDLL(so)


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def main():
    ref = os.environ.get("DSAC_REFERENCE", "")
    if not os.path.exists(os.path.join(ref, "train_score.cpp")):
        sys.exit("DSAC_REFERENCE must name the core/ directory of a checkout of the reference")
    from scipy.spatial.transform import Rotation
    tmp = tempfile.mkdtemp()
    lib = build(ref, tmp)
    lib.ref_score_camera.argtypes = [C.c_float, C.c_int, C.c_int]
    lib.ref_score_rand_hyp.argtypes = [C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    out = {"n_images": np.int32(N_IMAGES), "hyps": np.int32(HYPS), "seed": np.uint32(SEED), "focal": np.float64(FOCAL)}
    for seed in HYP_SEEDS:
        lib.ref_score_threads(seed, 1)
        for rot, trans in ((2.0, 2.0), (10.0, 100.0)):
            t = np.zeros((HYP_N, 3))
            R = np.zeros((HYP_N, 9))
            lib.ref_score_rand_hyp(rot, trans, HYP_N, p(t), p(R))
            key = "randhyp/%d/%g_%g" % (seed, rot, trans)
            out[key + "/trans"] = t
            out[key + "/rot"] = R
    rng = np.random.default_rng(20161216)
    cwd = os.getcwd()
    os.chdir(tmp)   # no translation.txt here: the pose reader uses the pose files as they are
    try:
        for name, W, H, F, threads in CASES:
            base = os.path.join(tmp, name)
            for d in ("rgb_noseg", "depth_noseg", "poses"):
                os.makedirs(os.path.join(base, d))
            bgr = OO.coded_bgr(F, H, W)
            for f in range(F):
                stem = "frame-%06d" % f
                cpath = base + "/rgb_noseg/" + stem + ".color.png"
                open(cpath, "wb").close()
                open(base + "/depth_noseg/" + stem + ".depth.png", "wb").close()
                lib.ref_score_register_bgr(cpath.encode(), W, H, p(np.ascontiguousarray(bgr[f])))
                M = np.eye(4)
                M[:3, :3] = Rotation.from_rotvec(rng.uniform(-1.0, 1.0, 3)).as_matrix()
                M[:3, 3] = rng.uniform(-1.0, 1.0, 3)
                with open(base + "/poses/" + stem + ".pose.txt", "w") as fh:
                    for row in M:
                        fh.write(" ".join("%.9e" % v for v in row) + "\n")
            lib.ref_score_camera(FOCAL, W, H)
            gt = np.zeros((F, 12))
            assert lib.ref_score_dataset(base.encode(), p(gt)) == F
            out[name + "/size"] = np.array([W, H, F], np.int32)
            out[name + "/gt_jp"] = gt
            n = N_IMAGES * HYPS
            for T in threads:
                lib.ref_score_threads(SEED, T)
                for rnd in range(2):
                    maps = np.zeros((n, 1600), np.float32)
                    labels = np.zeros(n)
                    frames = np.zeros(N_IMAGES, np.int32)
                    grid = np.zeros((N_IMAGES, 1600, 2), np.int32)
                    assert lib.ref_score_assemble(N_IMAGES, HYPS, p(maps), p(labels), p(frames), p(grid)) == n
                    key = "%s/T%d/round%d" % (name, T, rnd)
                    out[key + "/maps"] = maps
                    out[key + "/labels"] = labels
                    out[key + "/frames"] = frames
                    out[key + "/grid"] = grid.astype(np.int16)
            print(name, "done", flush=True)
    finally:
        os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "ref_score.npz"), **out)
    print("wrote", os.path.join(HERE, "ref_score.npz"), os.path.getsize(os.path.join(HERE, "ref_score.npz")), "bytes")


if __name__ == "__main__":
    main()
