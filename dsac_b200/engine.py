"""Python host-side binding of the C ABI (include/dsac_b200.h) via ctypes.

This is a thin mirror for tests and bench.py; the C/C++ surface (include/, dsac_b200/host/)
is the drop-in boundary.  There is no CPU fallback: `Engine(...)` raises if the CUDA
library is missing or no device is present.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

GRID = 40
N = GRID * GRID
STAGE_SAMPLE, STAGE_SCORE, STAGE_REFINE, STAGE_EVAL, STAGE_ALL = 1, 2, 4, 8, 15
ST_SAMPLER_EXHAUSTED, ST_REFINE_ABORTED = 1, 2
ST_BAD_WEIGHTS = 32          # DSAC_ST_BAD_WEIGHTS
ST_NO_DEPTH = 64             # DSAC_ST_NO_DEPTH
PASS_SOFTAM, PASS_DSAC, PASS_RIG = 1, 2, 3   # DSAC_PASS_SOFTAM, DSAC_PASS_DSAC, DSAC_PASS_RIG (dsac_last_pass)

# every symbol include/dsac_b200.h declares
EXPORTS = [
    "dsac_default_config", "dsac_engine_create", "dsac_engine_destroy", "dsac_last_error", "dsac_engine_config",
    "dsac_forward", "dsac_forward_submit", "dsac_forward_wait", "dsac_forward_device", "dsac_fetch", "dsac_device_view_get", "dsac_set_cameras", "dsac_set_stages",
    "dsac_set_tail_split", "dsac_launch_count", "dsac_sampler_profile", "dsac_sampler_profile_read", "dsac_debug_spec_result", "dsac_set_score_hook", "dsac_set_score_backward_hook", "dsac_backward", "dsac_backward_device", "dsac_forward_dsac", "dsac_forward_dsac_device",
    "dsac_backward_dsac", "dsac_backward_dsac_device", "dsac_refined_jp6_device", "dsac_backward_pose_device",
    "dsac_backward_dsac_pose_device", "dsac_gather_patches_device", "dsac_coords_from_prediction_device", "dsac_kabsch",
    "dsac_stochastic_subsample",
    "dsac_synth_frames", "dsac_version",
    "dsac_default_rgbd_camera", "dsac_set_dataset_cameras", "dsac_register_depth_device", "dsac_obj_coords_device", "dsac_obj_rng_init_device",
    "dsac_obj_draw_device", "dsac_gather_patches_at_device", "dsac_shuffle_permutation",
    "dsac_score_draw_device", "dsac_score_maps_device", "dsac_shuffle_permutations",
    "dsac_set_sampling_logits_device", "dsac_set_cell_depth_device", "dsac_sampling_table_device", "dsac_sampling_log_prob_device",
    "dsac_sampling_log_prob_backward_device", "dsac_set_coord_derivatives", "dsac_pose_uncertainty_device",
    "dsac_last_pass", "dsac_set_pose_priors_device", "dsac_pose_modes_device", "dsac_forward_rig_device",
    "dsac_backward_rig_device", "dsac_backward_rig_pose_device", "dsac_rig_refined_jp6_device",
    "dsac_rig_pose_uncertainty_device", "dsac_set_rig_pose_priors_device", "dsac_set_rig_cell_depth_device",
    "dsac_set_rig_score_hooks", "dsac_rig_pose_modes_device",
]

ST_OBJ_DRAW_EXHAUSTED = 8    # DSAC_ST_OBJ_DRAW_EXHAUSTED
ST_DEPTH_DROPPED = 16        # DSAC_ST_DEPTH_DROPPED
ST_BAD_PRIOR = 128           # DSAC_ST_BAD_PRIOR
ST_BAD_RIG = 256             # DSAC_ST_BAD_RIG
MAX_RIG_CAMERAS = 8          # DSAC_MAX_RIG_CAMERAS
MAX_PRIORS = 16              # DSAC_MAX_PRIORS
MAX_MODES = 16               # DSAC_MAX_MODES
OBJ_STATE_WORDS = 625        # one ThreadRand stream: std::mt19937's 624 words and its position


class Config(C.Structure):
    _fields_ = [
        ("focal", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
        ("n_hyps", C.c_int32), ("thr2d", C.c_int32), ("inlier_count", C.c_int32), ("ref_steps", C.c_int32),
        ("sub_sample", C.c_double), ("alpha", C.c_double), ("beta", C.c_double),
        ("seed", C.c_uint32), ("n_streams", C.c_int32), ("stream_skip", C.c_uint32), ("max_candidates", C.c_int32),
        ("fix_q4", C.c_int32), ("grad_clamp", C.c_double),
        ("write_diffmaps", C.c_int32), ("device", C.c_int32), ("max_frames", C.c_int32), ("hyps_per_cta", C.c_int32),
    ]


class RGBDCamera(C.Structure):
    """dsac_rgbd_camera: the RGB camera, the depth camera, sensorTrans (row-major 4x4), rawData and the frame size."""
    _fields_ = [
        ("focal", C.c_float), ("x_shift", C.c_float), ("y_shift", C.c_float),
        ("secondary_focal", C.c_float), ("raw_x_shift", C.c_float), ("raw_y_shift", C.c_float),
        ("sensor_trans", C.c_double * 16), ("raw_data", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
    ]


def default_rgbd_camera(**kw):
    """dsac_default_rgbd_camera with fields overridden by keyword (sensor_trans: any 4x4 / 16-element array)."""
    cam = RGBDCamera()
    rc = load().dsac_default_rgbd_camera(C.byref(cam))
    assert rc == 0
    for k, v in kw.items():
        if k == "sensor_trans":
            v = np.asarray(v, np.float64).reshape(16)
            for i in range(16):
                cam.sensor_trans[i] = float(v[i])
        else:
            setattr(cam, k, v)
    return cam


def camera_table(cams):
    """A sequence of RGBDCamera as the contiguous dsac_rgbd_camera array dsac_set_dataset_cameras reads (a ctypes array
    of RGBDCamera is returned as it is)."""
    if isinstance(cams, C.Array) and cams._type_ is RGBDCamera:
        return cams
    return (RGBDCamera * len(cams))(*cams)


def shuffle_permutation(n, seed=5489):
    """dsac_shuffle_permutation: std::shuffle(iota(n), std::mt19937(seed)), libstdc++'s permutation."""
    out = np.empty(n, np.int32)
    rc = load().dsac_shuffle_permutation(n, seed, _p(out))
    if rc != 0:
        raise ValueError("dsac_shuffle_permutation: bad arguments")
    return out


def shuffle_permutations(n, seed=5489, first_round=0, n_rounds=1):
    """dsac_shuffle_permutations: [n_rounds][n], the permutations of rounds first_round .. of one continuing
    std::mt19937(seed), each a std::shuffle of a fresh iota(n) (train_score.cpp's batch order)."""
    out = np.empty((n_rounds, n), np.int32)
    rc = load().dsac_shuffle_permutations(n, seed, first_round, n_rounds, _p(out))
    if rc != 0:
        raise ValueError("dsac_shuffle_permutations: bad arguments")
    return out


_OUT_FIELDS = ["hyp_pose", "img_idx", "cand_idx", "scores", "sf", "diffmaps", "entropy", "avg_pose", "ref_pose",
               "inlier_map", "ref_steps_done", "n_perm_steps", "loss", "rot_err", "t_err", "correct", "n_candidates",
               "status"]


class ForwardOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _OUT_FIELDS]


class DeviceView(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("diffmaps", "hyp_pose", "scores", "sf", "avg_pose", "ref_pose", "img_idx")]


_BW_FIELDS = ["dloss_dobj", "dloss_dref", "dref_dhyp", "dref_dobj", "score_grads", "dpnp"]


class BackwardOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _BW_FIELDS]


_DSAC_FIELDS = ["hyp_pose", "img_idx", "sf", "entropy", "ref_pose", "losses", "inlier_maps", "steps_done", "expected_loss",
                "hyp_idx", "rot_err", "t_err", "correct", "status"]


class DsacOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _DSAC_FIELDS]


_UNC_FIELDS = ("cov_jp6", "cov_xi", "sigma2", "n_fit", "support", "ok")


class PoseUncertaintyOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _UNC_FIELDS]


_MODES_FIELDS = ("n_modes", "hyp", "pose", "score", "mass", "members", "steps_done", "cov_xi", "sigma2", "n_fit", "support", "ok")


class PoseModesOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _MODES_FIELDS]


_RIG_FIELDS = ("hyp_pose", "rig_hyp", "scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map", "steps_done", "status",
               "loss", "rot_err", "t_err", "correct")


class RigOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _RIG_FIELDS]


_RIG_BW_FIELDS = ("dloss_dref", "dref_dhyp", "score_grads", "dref_dobj")


class RigBackwardOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _RIG_BW_FIELDS]


SCORE_HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p)
SCORE_BACKWARD_HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p)

_lib = None


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """dlopen libdsac_b200.so (building it with nvcc first if needed)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    alt = os.environ.get("DSAC_B200_LIB")   # development aid (tools/sweep.py): another BUILD of the same CUDA library
    if alt:
        path = alt
    elif build_if_missing:
        _build.build()
    if not os.path.exists(path):
        raise RuntimeError("%s is missing: build it with `python -m dsac_b200.build` (no CPU fallback exists)" % path)
    lib = C.CDLL(path)
    lib.dsac_last_error.restype = C.c_char_p
    lib.dsac_last_error.argtypes = [C.c_void_p]
    lib.dsac_version.restype = C.c_char_p
    lib.dsac_launch_count.restype = C.c_int64
    lib.dsac_launch_count.argtypes = [C.c_void_p]
    lib.dsac_engine_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    lib.dsac_engine_destroy.argtypes = [C.c_void_p]
    lib.dsac_engine_destroy.restype = None
    lib.dsac_forward.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                 C.POINTER(ForwardOut)]
    lib.dsac_forward_submit.argtypes = lib.dsac_forward.argtypes
    lib.dsac_forward_wait.argtypes = [C.c_void_p]
    lib.dsac_forward_device.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_void_p]
    lib.dsac_fetch.argtypes = [C.c_void_p, C.c_int32, C.POINTER(ForwardOut), C.c_void_p]
    lib.dsac_device_view_get.argtypes = [C.c_void_p, C.POINTER(DeviceView)]
    lib.dsac_sampler_profile.argtypes = [C.c_void_p, C.c_int32]
    lib.dsac_sampler_profile_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_debug_spec_result.argtypes = [C.c_void_p, C.c_void_p]
    lib.dsac_set_cameras.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_set_stages.argtypes = [C.c_void_p, C.c_uint32]
    lib.dsac_set_sampling_logits_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_set_cell_depth_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_set_pose_priors_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    lib.dsac_set_coord_derivatives.argtypes = [C.c_void_p, C.c_int32]
    lib.dsac_sampling_table_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.dsac_sampling_log_prob_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_sampling_log_prob_backward_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_set_tail_split.argtypes = [C.c_void_p, C.c_int32]
    lib.dsac_set_score_hook.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_set_score_backward_hook.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_backward.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                  C.POINTER(BackwardOut)]
    lib.dsac_forward_dsac.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                      C.POINTER(DsacOut)]
    lib.dsac_backward_dsac.argtypes = [C.c_void_p, C.c_int32, C.POINTER(BackwardDsacOut)]
    lib.dsac_backward_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    lib.dsac_forward_dsac_device.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                             C.c_int32, C.POINTER(DsacOut), C.c_void_p]
    lib.dsac_backward_dsac_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(BackwardDsacOut), C.c_void_p, C.c_float,
                                              C.c_void_p]
    lib.dsac_refined_jp6_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_pose_uncertainty_device.argtypes = [C.c_void_p, C.c_int32, C.POINTER(PoseUncertaintyOut), C.c_void_p]
    lib.dsac_last_pass.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.dsac_pose_modes_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_double, C.POINTER(PoseModesOut),
                                           C.c_void_p]
    lib.dsac_forward_rig_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_void_p, C.c_void_p, C.POINTER(RigOut), C.c_void_p]
    lib.dsac_backward_rig_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                             C.POINTER(RigBackwardOut), C.c_void_p]
    lib.dsac_backward_rig_pose_device.argtypes = lib.dsac_backward_rig_device.argtypes
    lib.dsac_rig_refined_jp6_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_rig_pose_uncertainty_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(PoseUncertaintyOut), C.c_void_p]
    lib.dsac_rig_pose_modes_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double,
                                               C.POINTER(PoseModesOut), C.c_void_p]
    lib.dsac_set_rig_pose_priors_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_double,
                                                    C.c_void_p]
    lib.dsac_set_rig_cell_depth_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_set_rig_score_hooks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_backward_pose_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    lib.dsac_backward_dsac_pose_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(BackwardDsacOut),
                                                   C.c_void_p, C.c_float, C.c_void_p]
    lib.dsac_gather_patches_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                               C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_coords_from_prediction_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_kabsch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_stochastic_subsample.argtypes = [C.c_uint32, C.c_int32, C.c_int32, C.c_void_p]
    lib.dsac_synth_frames.argtypes = [C.c_uint32, C.c_uint32, C.c_int32, C.c_int64, C.c_int32, C.c_double, C.c_double,
                                      C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    lib.dsac_default_rgbd_camera.argtypes = [C.POINTER(RGBDCamera)]
    lib.dsac_set_dataset_cameras.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_register_depth_device.argtypes = [C.c_void_p, C.POINTER(RGBDCamera), C.c_int32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_obj_coords_device.argtypes = [C.c_void_p, C.POINTER(RGBDCamera), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_obj_rng_init_device.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dsac_obj_draw_device.argtypes = [C.c_void_p, C.POINTER(RGBDCamera), C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
    lib.dsac_gather_patches_at_device.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_shuffle_permutation.argtypes = [C.c_int32, C.c_uint32, C.c_void_p]
    lib.dsac_score_draw_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_score_maps_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsac_shuffle_permutations.argtypes = [C.c_int32, C.c_uint32, C.c_int32, C.c_int32, C.c_void_p]
    _lib = lib
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def default_config(**kw):
    c = Config()
    load().dsac_default_config(C.byref(c))
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


def stochastic_subsample(seed=1305, width=640, height=480):
    pix = np.empty((N, 2), np.int32)
    rc = load().dsac_stochastic_subsample(seed, width, height, _p(pix))
    assert rc == 0
    return pix


def synth_frames(n_frames, frame0=0, data_seed=20170721, sampler_seed=1305, n_streams=1, rho=0.5, sigma=25.0,
                 traj=False, focal=525.0, cx=320.0, cy=240.0):
    """Synthetic frames of SURVEY.md section 8(d): (coords int16 [n,N,3], pix int32 [n,N,2], gt_cv [n,6], gt_jp [n,12])."""
    coords = np.empty((n_frames, N, 3), np.int16)
    pix = np.empty((n_frames, N, 2), np.int32)
    gt_cv = np.empty((n_frames, 6))
    gt_jp = np.empty((n_frames, 12))
    rc = load().dsac_synth_frames(data_seed, sampler_seed, n_streams, frame0, n_frames, rho, sigma, int(traj), focal, cx,
                                  cy, _p(coords), _p(pix), _p(gt_cv), _p(gt_jp))
    assert rc == 0
    return coords, pix, gt_cv, gt_jp


class ForwardResult:
    """Host copies of the processImage outputs for a batch of frames."""

    def __init__(self, n, H, want_diffmaps):
        self.hyp_pose = np.zeros((n, H, 6))
        self.img_idx = np.zeros((n, H, 4), np.int32)
        self.cand_idx = np.zeros((n, H), np.int32)
        self.scores = np.zeros((n, H))
        self.sf = np.zeros((n, H))
        self.diffmaps = np.zeros((n, H, N), np.float32) if want_diffmaps else None
        self.entropy = np.zeros(n)
        self.avg_pose = np.zeros((n, 6))
        self.ref_pose = np.zeros((n, 6))
        self.inlier_map = np.zeros((n, N), np.int32)
        self.ref_steps_done = np.zeros(n, np.int32)
        self.n_perm_steps = np.zeros(n, np.int32)
        self.loss = np.zeros(n)
        self.rot_err = np.zeros(n)
        self.t_err = np.zeros(n)
        self.correct = np.zeros(n, np.int32)
        self.n_candidates = np.zeros(n, np.int64)
        self.status = np.zeros(n, np.uint32)
        self.raw = ForwardOut()
        for k in _OUT_FIELDS:
            setattr(self.raw, k, _p(getattr(self, k)))


class DsacResult:
    """Host copies of the DSAC-variant processImage outputs (core/cnn.h:1028-1257)."""

    def __init__(self, n, H, want_inlier_maps):
        self.hyp_pose = np.zeros((n, H, 6)); self.img_idx = np.zeros((n, H, 4), np.int32); self.sf = np.zeros((n, H))
        self.entropy = np.zeros(n); self.ref_pose = np.zeros((n, H, 6)); self.losses = np.zeros((n, H))
        self.inlier_maps = np.zeros((n, H, N), np.int32) if want_inlier_maps else None
        self.steps_done = np.zeros((n, H), np.int32); self.expected_loss = np.zeros(n); self.hyp_idx = np.zeros(n, np.int32)
        self.rot_err = np.zeros(n); self.t_err = np.zeros(n); self.correct = np.zeros(n, np.int32); self.status = np.zeros(n, np.uint32)
        self.raw = DsacOut()
        for k in _DSAC_FIELDS:
            setattr(self.raw, k, _p(getattr(self, k)))


_BWD_FIELDS = ("dloss_dobj", "path1", "path2", "score_grads", "n_selected", "n_refine_jobs")


class BackwardDsacOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _BWD_FIELDS]


class BackwardDsacResult:
    """dsac_backward_dsac outputs (train_ransac.cpp:304-381)."""

    def __init__(self, n, H):
        self.dloss_dobj = np.zeros((n, N, 3)); self.path1 = np.zeros((n, N, 3)); self.path2 = np.zeros((n, N, 3))
        self.score_grads = np.zeros((n, H)); self.n_selected = np.zeros(n, np.int32); self.n_refine_jobs = np.zeros(n, np.int32)
        self.raw = BackwardDsacOut()
        for k in _BWD_FIELDS:
            setattr(self.raw, k, _p(getattr(self, k)))


class BackwardResult:
    def __init__(self, n, H, full=True):
        self.dloss_dobj = np.zeros((n, N, 3))
        self.dloss_dref = np.zeros((n, 6))
        self.dref_dhyp = np.zeros((n, 6, 6))
        self.dref_dobj = np.zeros((n, 6, N * 3)) if full else None
        self.score_grads = np.zeros((n, H))
        self.dpnp = np.zeros((n, H, 6, 12)) if full else None
        self.raw = BackwardOut()
        for k in _BW_FIELDS:
            setattr(self.raw, k, _p(getattr(self, k)))


class Engine:
    """One engine per GPU (dsac_engine_create / dsac_engine_destroy)."""

    def __init__(self, cfg=None, **kw):
        self.lib = load()
        self.cfg = cfg if cfg is not None else default_config(**kw)
        if cfg is not None:
            for k, v in kw.items():
                setattr(self.cfg, k, v)
        h = C.c_void_p()
        rc = self.lib.dsac_engine_create(C.byref(self.cfg), C.byref(h))
        if rc != 0:
            raise RuntimeError("dsac_engine_create failed (%d): %s" % (rc, self.lib.dsac_last_error(None).decode()))
        self.h = h
        self._hook = None
        self._rig_hooks = None   # the trampolines of set_rig_score_hooks
        self._dataset_cameras = None   # bytes of the dataset camera table installed by set_dataset_cameras, or None
        self.passes = 0   # forward passes started on this engine: the engine holds one pass, autograd.py checks it is still its own

    def close(self):
        if getattr(self, "h", None):
            self.lib.dsac_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("dsac call failed (%d): %s" % (rc, self.lib.dsac_last_error(self.h).decode()))

    @property
    def launches(self):
        return int(self.lib.dsac_launch_count(self.h))

    def set_stages(self, mask):
        self._check(self.lib.dsac_set_stages(self.h, mask))

    def sampler_profile(self, enable=True):
        self._check(self.lib.dsac_sampler_profile(self.h, int(enable)))

    def sampler_profile_read(self):
        """(ms[4], counts[4]) of the last profiled forward: generation+selection, filter, solve, tail; candidates, flagged,
        accepted, rounds."""
        ms = (C.c_double * 4)()
        cnt = (C.c_uint64 * 4)()
        self._check(self.lib.dsac_sampler_profile_read(self.h, ms, cnt))
        return list(ms), [int(x) for x in cnt]

    def spec_result(self):
        """Windows stitched per stream by the speculative first round of the last pass (0: abandoned / not used)."""
        out = (C.c_int32 * 8)()
        self._check(self.lib.dsac_debug_spec_result(self.h, out))
        return [int(x) for x in out]

    def set_cameras(self, cams, stream=None):
        """dsac_set_cameras: cams float64 [n][3] = (focal, cx, cy) of frame i of the following passes (a host array or CPU
        tensor), which must then have n frames; None: back to the config's camera.  stream: a cudaStream_t as int."""
        if cams is None:
            self._check(self.lib.dsac_set_cameras(self.h, 0, None, None))
            return
        cams = np.ascontiguousarray(cams, np.float64)
        if cams.ndim != 2 or cams.shape[1] != 3:
            raise ValueError("cameras must be float64 [n][3] (focal, cx, cy), got %s" % (cams.shape,))
        self._check(self.lib.dsac_set_cameras(self.h, cams.shape[0], _p(cams), C.c_void_p(stream) if stream else None))

    def set_cell_depth_device(self, n, d_depth, stream=None):
        """dsac_set_cell_depth_device: float32 [n][1600] depth in mm per cell on the device (raw pointer as int) makes the
        following passes RGB-D passes; d_depth None / 0 returns to RGB."""
        self._check(self.lib.dsac_set_cell_depth_device(self.h, n if d_depth else 0, C.c_void_p(d_depth) if d_depth else None,
                                                        C.c_void_p(stream) if stream else None))

    def set_pose_priors_device(self, n, k, d_poses, d_info=None, gate=0.0, stream=None):
        """dsac_set_pose_priors_device: k cv poses per frame, float64 [n][k][6] on the device (raw pointer as int), take the
        last k hypothesis slots of the following passes; d_info (float64 [n][k][6][6] information matrices, or None) gates
        the sampled hypotheses at the chi^2 bound `gate` (INTEGRATION.md, "Pose priors").  d_poses None / 0 clears them."""
        self._check(self.lib.dsac_set_pose_priors_device(self.h, n if d_poses else 0, k if d_poses else 0,
                                                         C.c_void_p(d_poses) if d_poses else None,
                                                         C.c_void_p(d_info) if d_info else None, float(gate),
                                                         C.c_void_p(stream) if stream else None))

    def set_coord_derivatives(self, mode):
        """dsac_set_coord_derivatives: "central" (the reference's central differences, the default) or "implicit" (the
        implicit-function derivatives of the refinement and of the minimal solve; INTEGRATION.md)."""
        modes = {"central": 0, "implicit": 1}
        if mode not in modes:
            raise ValueError("coordinate derivatives must be 'central' or 'implicit', got %r" % (mode,))
        self._check(self.lib.dsac_set_coord_derivatives(self.h, modes[mode]))

    def set_sampling_logits_device(self, n, d_logits, stream=None):
        """dsac_set_sampling_logits_device: float32 [n][1600] logits on the device (raw pointer as int) guide the sampler of
        the following passes, which must then have n frames; d_logits None: back to the reference's uniform sampler."""
        self._check(self.lib.dsac_set_sampling_logits_device(self.h, n if d_logits else 0, C.c_void_p(d_logits) if d_logits else None,
                                                             C.c_void_p(stream) if stream else None))

    def sampling_table_device(self, n, d_q):
        """dsac_sampling_table_device: the integer weights [n][1600] (uint32) the sampler draws from."""
        self._check(self.lib.dsac_sampling_table_device(self.h, n, C.c_void_p(d_q)))

    def sampling_log_prob_device(self, n, d_logp, stream=None):
        """dsac_sampling_log_prob_device: float64 [n] log-probability of the last (guided) pass's draw."""
        self._check(self.lib.dsac_sampling_log_prob_device(self.h, n, C.c_void_p(d_logp), C.c_void_p(stream) if stream else None))

    def sampling_log_prob_backward_device(self, n, d_grad_logp, d_grad_logits, stream=None):
        """dsac_sampling_log_prob_backward_device: float32 [n][1600] = d_grad_logp[f] * d log p_f / d logits_f."""
        self._check(self.lib.dsac_sampling_log_prob_backward_device(self.h, n, C.c_void_p(d_grad_logp), C.c_void_p(d_grad_logits),
                                                                    C.c_void_p(stream) if stream else None))

    def set_tail_split(self, mode):
        """0: off, 1: forward_device + blocking forward (default), 2: submitted passes too (scheduling only)."""
        self._check(self.lib.dsac_set_tail_split(self.h, mode))

    def forward(self, coords, pix, gt_jp=None, frame0=0, want_diffmaps=False, out=None):
        """dsac_forward with HOST buffers (numpy arrays)."""
        coords = np.ascontiguousarray(coords, np.int16).reshape(-1, N, 3)
        n = coords.shape[0]
        pix = np.ascontiguousarray(pix, np.int32)
        shared = 1 if pix.size == N * 2 else 0
        assert shared or pix.size == n * N * 2
        gt = np.ascontiguousarray(gt_jp, np.float64).reshape(n, 12) if gt_jp is not None else None
        res = out if out is not None else ForwardResult(n, self.cfg.n_hyps, want_diffmaps)
        self.passes += 1
        self._check(self.lib.dsac_forward(self.h, n, frame0, _p(coords), _p(pix), shared, _p(gt), C.byref(res.raw)))
        return res

    def forward_submit(self, coords, pix, gt_jp=None, frame0=0, out=None, want_diffmaps=False):
        """dsac_forward_submit: enqueue a pass and return; the arrays must stay alive (ideally pinned) until forward_wait()."""
        coords = np.ascontiguousarray(coords, np.int16).reshape(-1, N, 3)
        n = coords.shape[0]
        pix = np.ascontiguousarray(pix, np.int32)
        shared = 1 if pix.size == N * 2 else 0
        gt = np.ascontiguousarray(gt_jp, np.float64).reshape(n, 12) if gt_jp is not None else None
        res = out if out is not None else ForwardResult(n, self.cfg.n_hyps, want_diffmaps)
        self._pending = (coords, pix, gt, res)
        self.passes += 1
        self._check(self.lib.dsac_forward_submit(self.h, n, frame0, _p(coords), _p(pix), shared, _p(gt), C.byref(res.raw)))
        return res

    def forward_wait(self):
        self._check(self.lib.dsac_forward_wait(self.h))
        pending = getattr(self, "_pending", None)
        self._pending = None
        return pending[3] if pending else None

    def forward_device(self, n, d_coords, d_pix, pix_shared=0, d_gt=None, frame0=0, stream=None):
        """dsac_forward_device with raw device pointers (ints)."""
        self.passes += 1
        self._check(self.lib.dsac_forward_device(self.h, n, frame0, C.c_void_p(d_coords), C.c_void_p(d_pix), pix_shared,
                                                 C.c_void_p(d_gt) if d_gt else None, C.c_void_p(stream) if stream else None))

    def fetch(self, n, want_diffmaps=False, stream=None, out=None):
        res = out if out is not None else ForwardResult(n, self.cfg.n_hyps, want_diffmaps)
        self._check(self.lib.dsac_fetch(self.h, n, C.byref(res.raw), C.c_void_p(stream) if stream else None))
        return res

    def fetch_device(self, n, stream=None, **ptrs):
        """dsac_fetch into the given device pointers (ints; fields of dsac_forward_out except n_candidates); synchronises
        `stream`."""
        raw = ForwardOut()
        for k, v in ptrs.items():
            if k not in _OUT_FIELDS or k == "n_candidates":
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_fetch(self.h, n, C.byref(raw), C.c_void_p(stream) if stream else None))

    def device_view(self):
        v = DeviceView()
        self._check(self.lib.dsac_device_view_get(self.h, C.byref(v)))
        return v

    def set_score_hook(self, fn):
        """fn(d_diffmaps:int, n:int, H:int, d_scores:int, stream:int) -> int, called with device pointers."""
        if fn is None:
            self._hook = None
            self._check(self.lib.dsac_set_score_hook(self.h, None, None))
            return

        def tramp(dm, n, H, sc, stream, user):
            return int(fn(dm or 0, n, H, sc or 0, stream or 0))

        self._hook = SCORE_HOOK(tramp)
        self._check(self.lib.dsac_set_score_hook(self.h, C.cast(self._hook, C.c_void_p), None))

    def set_score_backward_hook(self, fn):
        """fn(d_diffmaps:int, d_score_grads:int, n:int, H:int, d_diffmap_grads:int, stream:int) -> int (device pointers):
        the seam's adjoint (lua_calls.h:312-341); must be registered together with the forward hook."""
        if fn is None:
            self._bw_hook = None
            self._check(self.lib.dsac_set_score_backward_hook(self.h, None, None))
            return

        def tramp(dm, sg, n, H, out, stream, user):
            return int(fn(dm or 0, sg or 0, n, H, out or 0, stream or 0))

        self._bw_hook = SCORE_BACKWARD_HOOK(tramp)
        self._check(self.lib.dsac_set_score_backward_hook(self.h, C.cast(self._bw_hook, C.c_void_p), None))

    def forward_dsac(self, coords, pix, gt_jp, random_draw=True, frame0=0, want_inlier_maps=False):
        """dsac_forward_dsac: the DSAC / RANSAC variant (draw + refine all hypotheses + expected loss)."""
        coords = np.ascontiguousarray(coords, np.int16).reshape(-1, N, 3)
        n = coords.shape[0]
        pix = np.ascontiguousarray(pix, np.int32)
        shared = 1 if pix.size == N * 2 else 0
        gt = np.ascontiguousarray(gt_jp, np.float64).reshape(n, 12) if gt_jp is not None else None
        res = DsacResult(n, self.cfg.n_hyps, want_inlier_maps)
        self.passes += 1
        self._check(self.lib.dsac_forward_dsac(self.h, n, frame0, _p(coords), _p(pix), shared, _p(gt), int(random_draw),
                                               C.byref(res.raw)))
        return res

    def backward(self, coords, pix, gt_jp, full=True):
        coords = np.ascontiguousarray(coords, np.int16).reshape(-1, N, 3)
        n = coords.shape[0]
        pix = np.ascontiguousarray(pix, np.int32)
        shared = 1 if pix.size == N * 2 else 0
        gt = np.ascontiguousarray(gt_jp, np.float64).reshape(n, 12)
        res = BackwardResult(n, self.cfg.n_hyps, full)
        self._check(self.lib.dsac_backward(self.h, n, _p(coords), _p(pix), shared, _p(gt), C.byref(res.raw)))
        return res

    def backward_dsac(self, n):
        """dsac_backward_dsac: gradients of the expected loss of the DSAC variant; follows forward_dsac over n frames."""
        res = BackwardDsacResult(n, self.cfg.n_hyps)
        self._check(self.lib.dsac_backward_dsac(self.h, n, C.byref(res.raw)))
        return res

    def backward_device(self, n, d_loss_grad=None, d_dloss_dobj=None, d_dloss_dpred=None, clamp=0.0, stream=None):
        """dsac_backward_device (raw device pointers as ints): soft-argmax backward of the preceding forward pass."""
        self._check(self.lib.dsac_backward_device(self.h, n, C.c_void_p(d_loss_grad) if d_loss_grad else None,
                                                  C.c_void_p(d_dloss_dobj) if d_dloss_dobj else None,
                                                  C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None, C.c_float(clamp),
                                                  C.c_void_p(stream) if stream else None))

    def forward_dsac_device(self, n, d_coords, d_pix, pix_shared=0, d_gt=None, random_draw=True, frame0=0, stream=None, **ptrs):
        """dsac_forward_dsac_device (raw device pointers as ints); ptrs: device destinations of dsac_dsac_out fields."""
        raw = DsacOut()
        for k, v in ptrs.items():
            if k not in _DSAC_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self.passes += 1
        self._check(self.lib.dsac_forward_dsac_device(self.h, n, frame0, C.c_void_p(d_coords), C.c_void_p(d_pix), pix_shared,
                                                      C.c_void_p(d_gt) if d_gt else None, int(random_draw), C.byref(raw),
                                                      C.c_void_p(stream) if stream else None))

    def backward_dsac_device(self, n, d_loss_grad=None, d_dloss_dpred=None, clamp=0.0, stream=None, **ptrs):
        """dsac_backward_dsac_device (raw device pointers as ints); ptrs: device destinations of dsac_backward_dsac_out fields."""
        raw = BackwardDsacOut()
        for k, v in ptrs.items():
            if k not in _BWD_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_backward_dsac_device(self.h, n, C.c_void_p(d_loss_grad) if d_loss_grad else None, C.byref(raw),
                                                       C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None, C.c_float(clamp),
                                                       C.c_void_p(stream) if stream else None))

    def refined_jp6_device(self, n, d_jp6, stream=None):
        """dsac_refined_jp6_device (raw device pointers as ints): jp 6-vectors of the preceding pass's refined poses,
        [n][6] after a soft-argmax forward, [n][H][6] after a DSAC-variant forward."""
        self._check(self.lib.dsac_refined_jp6_device(self.h, n, C.c_void_p(d_jp6), C.c_void_p(stream) if stream else None))

    def pose_uncertainty_device(self, n, stream=None, **ptrs):
        """dsac_pose_uncertainty_device (raw device pointers as ints); ptrs: device destinations of the fields of
        dsac_pose_uncertainty_out (cov_jp6, cov_xi, sigma2, n_fit, support, ok), one entry per refined pose of the preceding
        pass: [n] after a soft-argmax forward, [n][H] after a DSAC-variant forward."""
        raw = PoseUncertaintyOut()
        for k, v in ptrs.items():
            if k not in _UNC_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_pose_uncertainty_device(self.h, n, C.byref(raw), C.c_void_p(stream) if stream else None))

    def pose_modes_device(self, n, max_modes, rot_rad, trans_mm, stream=None, **ptrs):
        """dsac_pose_modes_device (raw device pointers as ints): the distinct refined poses of each frame's hypothesis pool
        after the preceding pass over n frames (INTEGRATION.md, "Pose modes"); ptrs: device destinations of the fields of
        dsac_pose_modes_out (n_modes [n]; hyp, pose, score, mass, members, steps_done, cov_xi, sigma2, n_fit, support, ok
        [n][max_modes](...))."""
        raw = PoseModesOut()
        for k, v in ptrs.items():
            if k not in _MODES_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_pose_modes_device(self.h, n, max_modes, float(rot_rad), float(trans_mm), C.byref(raw),
                                                    C.c_void_p(stream) if stream else None))

    def forward_rig_device(self, n, n_cameras, d_coords, d_pix, d_cam_from_rig, pix_shared=0, d_gt_rig=None, frame0=0,
                           stream=None, **ptrs):
        """dsac_forward_rig_device (raw device pointers as ints): one pose per rig of n_cameras cameras over n frames
        (INTEGRATION.md, "Multi-camera rigs"); ptrs: device destinations of the fields of dsac_rig_out."""
        raw = RigOut()
        for k, v in ptrs.items():
            if k not in _RIG_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self.passes += 1
        self._check(self.lib.dsac_forward_rig_device(self.h, n, n_cameras, frame0, C.c_void_p(d_coords), C.c_void_p(d_pix),
                                                     pix_shared, C.c_void_p(d_cam_from_rig), C.c_void_p(d_gt_rig) if d_gt_rig else None,
                                                     C.byref(raw), C.c_void_p(stream) if stream else None))

    def _rig_diag(self, ptrs):
        raw = RigBackwardOut()
        for k, v in ptrs.items():
            if k not in _RIG_BW_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        return raw

    def backward_rig_device(self, n, d_loss_grad=None, d_dloss_dobj=None, d_dloss_dpred=None, clamp=0.0, stream=None, **ptrs):
        """dsac_backward_rig_device (raw device pointers as ints): the loss form of the rig backward after forward_rig_device
        over n frames (INTEGRATION.md, "Rig gradients"); d_loss_grad [R] (None: 1); ptrs: device destinations of the fields
        of dsac_rig_backward_out (dloss_dref, dref_dhyp, score_grads, dref_dobj)."""
        raw = self._rig_diag(ptrs)
        self._check(self.lib.dsac_backward_rig_device(self.h, n, C.c_void_p(d_loss_grad) if d_loss_grad else None,
                                                      C.c_void_p(d_dloss_dobj) if d_dloss_dobj else None,
                                                      C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None, C.c_float(clamp),
                                                      C.byref(raw), C.c_void_p(stream) if stream else None))

    def backward_rig_pose_device(self, n, d_grad_ref, d_dloss_dobj=None, d_dloss_dpred=None, clamp=0.0, stream=None, **ptrs):
        """dsac_backward_rig_pose_device (raw device pointers as ints): the rig backward seeded by dOuter/d(refined rig jp6)
        [R][6]; ptrs as backward_rig_device."""
        raw = self._rig_diag(ptrs)
        self._check(self.lib.dsac_backward_rig_pose_device(self.h, n, C.c_void_p(d_grad_ref) if d_grad_ref else None,
                                                           C.c_void_p(d_dloss_dobj) if d_dloss_dobj else None,
                                                           C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None, C.c_float(clamp),
                                                           C.byref(raw), C.c_void_p(stream) if stream else None))

    def rig_refined_jp6_device(self, n, d_jp6, stream=None):
        """dsac_rig_refined_jp6_device (raw device pointers as ints): jp 6-vectors [R][6] of the refined rig poses of the
        preceding forward_rig_device over n frames."""
        self._check(self.lib.dsac_rig_refined_jp6_device(self.h, n, C.c_void_p(d_jp6) if d_jp6 else None,
                                                         C.c_void_p(stream) if stream else None))

    def set_rig_pose_priors_device(self, n, n_cameras, k, d_poses, d_info=None, gate=0.0, stream=None):
        """dsac_set_rig_pose_priors_device: k cv rig poses per rig, float64 [n / n_cameras][k][6] on the device (raw pointer as
        int), join the pools of the following forward_rig_device passes over n frames of n_cameras cameras; d_info (float64
        [n / n_cameras][k][6][6] information matrices in the rig chart, or None) gates every camera's sampled hypotheses at
        the chi^2 bound `gate` (INTEGRATION.md, "Rig tracking").  d_poses None / 0 clears them."""
        self._check(self.lib.dsac_set_rig_pose_priors_device(self.h, n if d_poses else 0, n_cameras if d_poses else 0,
                                                             k if d_poses else 0, C.c_void_p(d_poses) if d_poses else None,
                                                             C.c_void_p(d_info) if d_info else None, float(gate),
                                                             C.c_void_p(stream) if stream else None))

    def set_rig_cell_depth_device(self, n, n_cameras, d_depth, stream=None):
        """dsac_set_rig_cell_depth_device: float32 [n][1600] depth in mm per cell of every camera frame on the device (raw
        pointer as int) makes the following forward_rig_device passes over n frames of n_cameras cameras RGB-D rigs
        (INTEGRATION.md, "RGB-D rigs").  d_depth None / 0 clears it."""
        self._check(self.lib.dsac_set_rig_cell_depth_device(self.h, n if d_depth else 0, n_cameras if d_depth else 0,
                                                            C.c_void_p(d_depth) if d_depth else None,
                                                            C.c_void_p(stream) if stream else None))

    def set_rig_score_hooks(self, fn, bw_fn):
        """dsac_set_rig_score_hooks: score every rig pass's pool with fn and differentiate it with bw_fn (INTEGRATION.md,
        "Rig score hooks"); the callables of set_score_hook and set_score_backward_hook, called with n camera frames and
        P = n_cameras * n_hyps pool slots (ScoreCNN and its backward as they are).  (None, None) clears them."""
        if fn is None and bw_fn is None:
            self._check(self.lib.dsac_set_rig_score_hooks(self.h, None, None, None))
            self._rig_hooks = None
            return
        if fn is None or bw_fn is None:
            raise ValueError("set_rig_score_hooks: the forward and the backward hook are set together; (None, None) clears them")

        def tramp(dm, n, P, sc, stream, user):
            return int(fn(dm or 0, n, P, sc or 0, stream or 0))

        def bw_tramp(dm, sg, n, P, out, stream, user):
            return int(bw_fn(dm or 0, sg or 0, n, P, out or 0, stream or 0))

        hooks = (SCORE_HOOK(tramp), SCORE_BACKWARD_HOOK(bw_tramp))
        self._check(self.lib.dsac_set_rig_score_hooks(self.h, C.cast(hooks[0], C.c_void_p), C.cast(hooks[1], C.c_void_p), None))
        self._rig_hooks = hooks   # the engine calls them until they are replaced or cleared

    def rig_pose_uncertainty_device(self, n, n_cameras, stream=None, **ptrs):
        """dsac_rig_pose_uncertainty_device (raw device pointers as ints): the covariance of each refined rig pose of the
        preceding forward_rig_device over n frames of n_cameras cameras; ptrs: device destinations of the fields of
        dsac_pose_uncertainty_out, one entry per rig ([R] and [R][6][6], R = n / n_cameras)."""
        raw = PoseUncertaintyOut()
        for k, v in ptrs.items():
            if k not in _UNC_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_rig_pose_uncertainty_device(self.h, n, n_cameras, C.byref(raw), C.c_void_p(stream) if stream else None))

    def rig_pose_modes_device(self, n, n_cameras, max_modes, rot_rad, trans_mm, stream=None, **ptrs):
        """dsac_rig_pose_modes_device (raw device pointers as ints): the distinct refined rig poses of each rig's pool after
        the preceding forward_rig_device over n frames of n_cameras cameras (INTEGRATION.md, "Rig pose modes"); ptrs: device
        destinations of the fields of dsac_pose_modes_out, per rig (n_modes [R]; the others [R][max_modes](...),
        R = n / n_cameras; hyp is the pool slot c * n_hyps + h)."""
        raw = PoseModesOut()
        for k, v in ptrs.items():
            if k not in _MODES_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_rig_pose_modes_device(self.h, n, n_cameras, max_modes, float(rot_rad), float(trans_mm),
                                                        C.byref(raw), C.c_void_p(stream) if stream else None))

    def last_pass(self, n):
        """dsac_last_pass: "softam", "dsac" or "rig", the kind of the pass over n frames the engine holds (what
        pose_uncertainty_device reads after the first two); raises if it holds none."""
        kind = C.c_int32(0)
        self._check(self.lib.dsac_last_pass(self.h, n, C.byref(kind)))
        return {PASS_SOFTAM: "softam", PASS_DSAC: "dsac", PASS_RIG: "rig"}[kind.value]

    def backward_pose_device(self, n, d_grad_ref, d_dloss_dobj=None, d_dloss_dpred=None, clamp=0.0, stream=None):
        """dsac_backward_pose_device (raw device pointers as ints): soft-argmax backward seeded by dOuter/d(refined jp6)."""
        self._check(self.lib.dsac_backward_pose_device(self.h, n, C.c_void_p(d_grad_ref),
                                                       C.c_void_p(d_dloss_dobj) if d_dloss_dobj else None,
                                                       C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None, C.c_float(clamp),
                                                       C.c_void_p(stream) if stream else None))

    def backward_dsac_pose_device(self, n, d_grad_ref=None, d_grad_sf=None, d_dloss_dpred=None, clamp=0.0, stream=None, **ptrs):
        """dsac_backward_dsac_pose_device (raw device pointers as ints): DSAC-variant backward seeded by dOuter/d(refined
        jp6) [n][H][6] and dOuter/dsf [n][H], either None; ptrs: device destinations of dsac_backward_dsac_out fields."""
        raw = BackwardDsacOut()
        for k, v in ptrs.items():
            if k not in _BWD_FIELDS:
                raise KeyError(k)
            setattr(raw, k, v)
        self._check(self.lib.dsac_backward_dsac_pose_device(self.h, n, C.c_void_p(d_grad_ref) if d_grad_ref else None,
                                                            C.c_void_p(d_grad_sf) if d_grad_sf else None, C.byref(raw),
                                                            C.c_void_p(d_dloss_dpred) if d_dloss_dpred else None,
                                                            C.c_float(clamp), C.c_void_p(stream) if stream else None))

    def gather_patches_device(self, n, d_frames, width, height, d_pix, pix_shared, d_patches, mean=127.0, d_status=None, stream=None):
        """dsac_gather_patches_device (raw device pointers as ints): BGR frames -> normalised 3x42x42 CNN patches."""
        self._check(self.lib.dsac_gather_patches_device(self.h, n, C.c_void_p(d_frames), width, height, C.c_void_p(d_pix), pix_shared,
                                                        C.c_float(mean), C.c_void_p(d_patches), C.c_void_p(d_status) if d_status else None,
                                                        C.c_void_p(stream) if stream else None))

    def coords_from_prediction_device(self, n, d_pred, d_coords, stream=None):
        """dsac_coords_from_prediction_device: float metres -> int16 millimetres (cv::saturate_cast<short>)."""
        self._check(self.lib.dsac_coords_from_prediction_device(self.h, n, C.c_void_p(d_pred), C.c_void_p(d_coords),
                                                                C.c_void_p(stream) if stream else None))

    def kabsch(self, a, b):
        a = np.ascontiguousarray(a, np.float64)
        b = np.ascontiguousarray(b, np.float64)
        n, m = a.shape[0], a.shape[1]
        R = np.zeros((n, 9))
        t = np.zeros((n, 3))
        self._check(self.lib.dsac_kabsch(self.h, n, m, _p(a), _p(b), _p(R), _p(t)))
        return R.reshape(n, 3, 3), t

    # ------------------------------------------------------------------ coordinate-CNN pre-training data path
    # Raw device pointers as ints; `cam` is an RGBDCamera, or None for the dataset camera table (set_dataset_cameras);
    # stream: a cudaStream_t as int or None.

    def set_dataset_cameras(self, cams, stream=None):
        """dsac_set_dataset_cameras: cams, a sequence of RGBDCamera, one per dataset frame, becomes the table that
        cam=None means in the pre-training calls and that score_maps_device projects with; None clears it."""
        if cams is None:
            self._check(self.lib.dsac_set_dataset_cameras(self.h, 0, None, None))
            self._dataset_cameras = None
            return
        table = camera_table(cams)
        self._check(self.lib.dsac_set_dataset_cameras(self.h, len(cams), C.cast(table, C.c_void_p),
                                                      C.c_void_p(stream) if stream else None))
        self._dataset_cameras = bytes(table)

    def use_dataset_cameras(self, cams, stream=None):
        """set_dataset_cameras(cams) unless this wrapper installed the same table last (None: no table), so that
        several scenes can take turns on one engine without copying their tables on every call."""
        key = None if cams is None else bytes(camera_table(cams))
        if key != self._dataset_cameras:
            self.set_dataset_cameras(cams, stream)

    @staticmethod
    def _cam(cam):
        return C.byref(cam) if cam is not None else None

    def register_depth_device(self, cam, n, d_raw, d_depth, d_dropped=None, d_status=None, stream=None):
        """dsac_register_depth_device: raw depth [n][H][W] uint16 -> depth registered to the RGB camera."""
        self._check(self.lib.dsac_register_depth_device(self.h, self._cam(cam), n, C.c_void_p(d_raw), C.c_void_p(d_depth),
                                                        C.c_void_p(d_dropped) if d_dropped else None,
                                                        C.c_void_p(d_status) if d_status else None,
                                                        C.c_void_p(stream) if stream else None))

    def obj_coords_device(self, cam, n_frames, n, d_depth, d_poses, d_coords, d_idx=None, stream=None):
        """dsac_obj_coords_device: getObj images [n][H][W][3] int16 (mm) of frames d_idx[0..n) (None: 0..n) of a
        dataset of n_frames frames."""
        self._check(self.lib.dsac_obj_coords_device(self.h, self._cam(cam), n_frames, n, C.c_void_p(d_idx) if d_idx else None,
                                                    C.c_void_p(d_depth), C.c_void_p(d_poses), C.c_void_p(d_coords),
                                                    C.c_void_p(stream) if stream else None))

    def obj_rng_init_device(self, seed, n_streams, d_state, stream=None):
        """dsac_obj_rng_init_device: ThreadRand::init(seed) for n_streams threads into d_state [n_streams][625] uint32."""
        self._check(self.lib.dsac_obj_rng_init_device(self.h, C.c_uint32(seed), n_streams, C.c_void_p(d_state),
                                                      C.c_void_p(stream) if stream else None))

    def obj_draw_device(self, cam, n_frames, d_depth, d_poses, n_images, n_patches, n_streams, max_attempts, d_state,
                        d_img, d_centre, d_label, d_status, stream=None):
        """dsac_obj_draw_device: one round of assembleData's draw."""
        self._check(self.lib.dsac_obj_draw_device(self.h, self._cam(cam), n_frames, C.c_void_p(d_depth), C.c_void_p(d_poses),
                                                  n_images, n_patches, n_streams, max_attempts, C.c_void_p(d_state),
                                                  C.c_void_p(d_img), C.c_void_p(d_centre), C.c_void_p(d_label),
                                                  C.c_void_p(d_status), C.c_void_p(stream) if stream else None))

    def gather_patches_at_device(self, n, d_frames, n_frames, width, height, d_frame, d_centre, d_patches, mean=127.0,
                                 d_status=None, stream=None):
        """dsac_gather_patches_at_device: patches [n][3][42][42] around listed (frame, x, y) of device-resident frames."""
        self._check(self.lib.dsac_gather_patches_at_device(self.h, n, C.c_void_p(d_frames), n_frames, width, height,
                                                           C.c_void_p(d_frame), C.c_void_p(d_centre), C.c_float(mean),
                                                           C.c_void_p(d_patches), C.c_void_p(d_status) if d_status else None,
                                                           C.c_void_p(stream) if stream else None))

    # ------------------------------------------------------------------ score-CNN pre-training data path

    def score_draw_device(self, n_frames, width, height, n_images, hyps_per_image, n_streams, d_state, d_img, d_pix,
                          d_drift, d_noise, stream=None):
        """dsac_score_draw_device: one round of train_score.cpp's assembleData draw (frames, grids, drift levels and
        getRandHyp vectors) on ThreadRand state d_state [n_streams][625]."""
        self._check(self.lib.dsac_score_draw_device(self.h, n_frames, width, height, n_images, hyps_per_image, n_streams,
                                                    C.c_void_p(d_state), C.c_void_p(d_img), C.c_void_p(d_pix),
                                                    C.c_void_p(d_drift), C.c_void_p(d_noise),
                                                    C.c_void_p(stream) if stream else None))

    def score_maps_device(self, n_images, hyps_per_image, d_img, d_gt_jp, d_coords, d_pix, d_noise, temperature, d_maps,
                          d_labels, d_correct=None, stream=None):
        """dsac_score_maps_device: reprojection-error images [n][1600], labels [n] and the 5 deg / 50 mm flags of a
        draw's perturbed ground-truth poses against the coordinate CNN's grids; with a dataset camera table installed,
        image i is projected with the camera of frame img[i] (getCamMat), else with the config's camera."""
        self._check(self.lib.dsac_score_maps_device(self.h, n_images, hyps_per_image, C.c_void_p(d_img), C.c_void_p(d_gt_jp),
                                                    C.c_void_p(d_coords), C.c_void_p(d_pix), C.c_void_p(d_noise),
                                                    C.c_float(temperature), C.c_void_p(d_maps), C.c_void_p(d_labels),
                                                    C.c_void_p(d_correct) if d_correct else None,
                                                    C.c_void_p(stream) if stream else None))
