"""ctypes binding of libdsk.so (the C ABI in include/dsk.h) and the in-tree nvcc build recipe.

The product path has no fallback: if the shared library is missing or an entry point fails, a
RuntimeError is raised (north star: "no CPU fallback, no multi-backend dispatch").
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdsk.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")

NUM_CONV = 12
DSK_F16, DSK_BF16 = 0, 1
DSK_EVAL, DSK_TRAIN = 0, 1
DSK_GE2E_SOFTMAX, DSK_GE2E_CONTRAST = 0, 1
DSK_LINKAGE_AVERAGE, DSK_LINKAGE_COMPLETE = 0, 1
DSK_AHC_MAX_N = 32768
DSK_NORM_NONE, DSK_NORM_LENGTH, DSK_NORM_PLDA = 0, 1, 2
DSK_F64_MAX_DIM = 4096
DSK_PLDA_MAX_ROWS = 4194240
DSK_VBX_MAX_SPEAKERS = 128
DSK_SC_MAX_SPEAKERS, DSK_SC_MAX_P = 32, 64
DSK_SPEED_MAX_DEN, DSK_SPEED_TAPS, DSK_SPEED_MAX_FACTORS = 32, 50, 8
DSK_AAM_MAX_C, DSK_AAM_MAX_SUBCENTRES, DSK_AAM_MAX_TOPK = 65536, 16, 64

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))) + [
        os.path.join(INCLUDE, "dsk.h")
    ]


HASH_PATH = LIB_PATH + ".srchash"


def _source_hash() -> str:
    import hashlib

    h = hashlib.sha1()
    for s in _sources():
        h.update(os.path.basename(s).encode())
        with open(s, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def needs_build() -> bool:
    """True when lib/libdsk.so is missing or was built from different source CONTENT (file times are not trusted:
    the tree is copied between machines, and N ranks may import it at once)."""
    if not os.path.exists(LIB_PATH):
        return True
    try:
        with open(HASH_PATH) as f:
            return f.read().strip() != _source_hash()
    except OSError:
        return True


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into lib/libdsk.so (nvcc cross-compiles without a GPU).  Safe under concurrent
    callers: an exclusive file lock serialises them and the library is renamed into place."""
    if not force and not needs_build():
        return LIB_PATH
    import fcntl

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libdsk.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not needs_build():  # another process built it while this one waited
            return LIB_PATH
        tmp = LIB_PATH + f".tmp{os.getpid()}"
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp, os.path.join(CSRC, "dsk_api.cu")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            if os.path.exists(tmp):
                os.remove(tmp)
            raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
        os.replace(tmp, LIB_PATH)
        with open(HASH_PATH, "w") as f:
            f.write(_source_hash())
        if verbose:
            print(r.stderr)
    return LIB_PATH


class DskWeights(ctypes.Structure):
    _fields_ = [
        ("conv_w", c_void_p * NUM_CONV),
        ("bn_gamma", c_void_p * NUM_CONV),
        ("bn_beta", c_void_p * NUM_CONV),
        ("bn_running_mean", c_void_p * NUM_CONV),
        ("bn_running_var", c_void_p * NUM_CONV),
        ("fc_w", c_void_p),
        ("fc_b", c_void_p),
        ("embedding_size", c_int32),
    ]


class DskGrads(ctypes.Structure):
    _fields_ = [
        ("conv_w", c_void_p * NUM_CONV),
        ("bn_gamma", c_void_p * NUM_CONV),
        ("bn_beta", c_void_p * NUM_CONV),
        ("fc_w", c_void_p),
        ("fc_b", c_void_p),
    ]


class DskBackwardCapture(ctypes.Structure):
    _fields_ = [
        ("gy", c_void_p * NUM_CONV),
        ("G", c_void_p * NUM_CONV),
        ("gres", c_void_p * NUM_CONV),
        ("g_fc", c_void_p),
        ("fc_out", c_void_p),
        ("dP", c_void_p),
        ("loss_scale", c_void_p),
    ]


# name -> (restype, argtypes); must list every symbol declared in include/dsk.h
SIGNATURES = {
    "dsk_last_error": (c_char_p, []),
    "dsk_version": (c_int32, []),
    "dsk_create": (c_int32, [POINTER(c_void_p), c_int32, c_int32]),
    "dsk_destroy": (c_int32, [c_void_p]),
    "dsk_load_weights": (c_int32, [c_void_p, POINTER(DskWeights), c_void_p]),
    "dsk_load_weights_train": (c_int32, [c_void_p, POINTER(DskWeights), c_void_p]),
    "dsk_share_weights": (c_int32, [c_void_p, c_void_p]),
    "dsk_rescnn_forward": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int32, c_void_p]),
    "dsk_rescnn_forward_train": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, POINTER(c_void_p), c_void_p]),
    "dsk_rescnn_backward": (c_int32, [c_void_p, c_void_p, c_void_p, POINTER(DskGrads), c_void_p]),
    "dsk_train_ctx_read": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_debug_backward_plan": (c_int32, [c_void_p, c_void_p, c_int32, POINTER(c_int32)]),
    "dsk_debug_read_eval_activation": (c_int32, [c_void_p, c_int32, c_void_p, c_int64, POINTER(c_int32), c_void_p]),
    "dsk_train_ctx_release": (c_int32, [c_void_p, c_void_p]),
    "dsk_set_loss_scale": (c_int32, [c_void_p, c_float]),
    "dsk_sync_forward_begin": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, POINTER(c_void_p), c_void_p]),
    "dsk_sync_backward_begin": (c_int32, [c_void_p, c_void_p, c_void_p, POINTER(DskGrads), c_void_p]),
    "dsk_sync_records": (c_int32, [c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_int64)]),
    "dsk_sync_stage": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, POINTER(c_int32), c_void_p]),
    "dsk_bn_act_sync_train_forward": (c_int32, [c_void_p] * 10 + [c_int32, c_int32, c_int32, c_void_p]),
    "dsk_set_profiling": (c_int32, [c_void_p, c_int32]),
    "dsk_get_launch_times": (c_int32, [c_void_p, c_void_p, c_int32, POINTER(c_int32)]),
    "dsk_conv2d_nhwc": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32,
                                  c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_float, c_void_p]),
    "dsk_conv2d_dgrad_nhwc": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                        c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "dsk_conv2d_wgrad_nhwc": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                        c_int32, c_int32, c_int32, c_float, c_void_p]),
    "dsk_bn_act_train_forward": (c_int32, [c_void_p] * 10 + [c_int64, c_int32, c_void_p]),
    "dsk_bn_act_train_backward": (c_int32, [c_void_p] * 11 + [c_int64, c_int32, c_float, c_void_p]),
    "dsk_conv3x3_padded": (c_int32, [c_void_p] * 7 + [c_int32, c_int32, c_int32, c_int32, c_int32, c_float, c_int32, c_void_p]),
    "dsk_conv5x5s2_planar": (c_int32, [c_void_p] * 6 + [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_float, c_void_p]),
    "dsk_debug_set_backward_capture": (c_int32, [c_void_p, POINTER(DskBackwardCapture)]),
    "dsk_padded_positions": (c_int64, [c_int32, c_int32, c_int32]),
    "dsk_pack_conv_weight": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "dsk_nchw_f32_to_nhwc16": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "dsk_nhwc16_to_nchw_f32": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "dsk_pairwise_distance": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_pairwise_distance_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                            c_void_p, c_void_p]),
    "dsk_triplet_loss": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "dsk_triplet_loss_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                       c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_margin_select": (c_int32, [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_void_p]),
    "dsk_gather_rows": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int64, c_void_p, c_void_p]),
    "dsk_allpairs_topk_tc": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "dsk_allpairs_topk": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "dsk_batch_hard_triplet": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float] + [c_void_p] * 7),
    "dsk_batch_hard_triplet_bwd": (c_int32, [c_void_p] * 5 + [c_int32, c_int32, c_float, c_void_p, c_void_p, c_void_p,
                                                              c_void_p]),
    "dsk_batch_hard_select_rows": (c_int32, [c_void_p] * 3 + [c_int32] * 4 + [c_void_p] * 6),
    "dsk_batch_hard_mean": (c_int32, [c_void_p] * 3 + [c_int32, c_float, c_void_p, c_void_p]),
    "dsk_batch_hard_triplet_bwd_rows": (c_int32, [c_void_p] * 6 + [c_int32] * 4 + [c_float] + [c_void_p] * 3),
    "dsk_aam_softmax": (c_int32, [c_void_p] * 4 + [c_int32] * 3 + [c_float, c_float] + [c_void_p] * 4),
    "dsk_aam_softmax_bwd": (c_int32, [c_void_p] * 6 + [c_int32] * 3 + [c_float, c_float] + [c_void_p] * 4),
    "dsk_aam_softmax_sc": (c_int32, [c_void_p] * 4 + [c_int32] * 4 + [c_float, c_float, c_int32, c_float]
                           + [c_void_p] * 6),
    "dsk_aam_softmax_sc_bwd": (c_int32, [c_void_p] * 8 + [c_int32] * 4 + [c_float, c_float, c_int32, c_float]
                               + [c_void_p] * 4),
    "dsk_aam_subcentre_cos": (c_int32, [c_void_p] * 3 + [c_int32] * 4 + [c_void_p] * 2),
    "dsk_aam_shard_cos": (c_int32, [c_void_p] * 4 + [c_int32] * 7 + [c_void_p] * 4),
    "dsk_aam_shard_merge": (c_int32, [c_void_p] * 3 + [c_int32] * 6 + [c_float] * 3 + [c_void_p] * 4),
    "dsk_aam_shard_partials": (c_int32, [c_void_p] * 4 + [c_int32] * 7 + [c_float] * 3 + [c_void_p] * 3),
    "dsk_aam_shard_finish": (c_int32, [c_void_p] * 3 + [c_int32] * 4 + [c_void_p] * 5),
    "dsk_aam_shard_bwd": (c_int32, [c_void_p] * 9 + [c_int32] * 6 + [c_float, c_float, c_int32, c_float]
                          + [c_void_p] * 4),
    "dsk_aam_shard_bwd_rows": (c_int32, [c_void_p] * 2 + [c_int32] * 3 + [c_void_p] * 2),
    "dsk_ge2e": (c_int32, [c_void_p, c_void_p, c_int32, c_int32] + [c_void_p] * 3 + [c_int32, c_int32] + [c_void_p] * 2
                 + [c_int32] + [c_void_p] * 4),
    "dsk_ge2e_bwd": (c_int32, [c_void_p, c_void_p, c_int32, c_int32] + [c_void_p] * 3 + [c_int32, c_int32]
                     + [c_void_p] * 2 + [c_int32] + [c_void_p] * 7),
    "dsk_ge2e_rows": (c_int32, [c_void_p, c_void_p, c_int32, c_int32] + [c_void_p] * 3 + [c_int32, c_int32]
                      + [c_void_p] * 2 + [c_int32] * 3 + [c_void_p] * 4),
    "dsk_ge2e_mean": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_ge2e_dcos_rows": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                     c_void_p, c_int32, c_void_p, c_int32, c_int32] + [c_void_p] * 5),
    "dsk_ge2e_bwd_rows": (c_int32, [c_void_p, c_void_p, c_int32, c_int32] + [c_void_p] * 3 + [c_int32]
                          + [c_void_p] * 2 + [c_int32] * 2 + [c_void_p] * 2),
    "dsk_cosine_matrix": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_topk_mean_std": (c_int32, [c_void_p, c_int32, c_int32, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    "dsk_cohort_stats": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32] + [c_void_p] * 3),
    "dsk_score_trials": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_int64] + [c_void_p] * 5),
    "dsk_topk_indices": (c_int32, [c_void_p, c_int32, c_int32, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    "dsk_cosine_topk": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32] + [c_void_p] * 3),
    "dsk_class_centroids": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_int32, c_void_p, c_void_p]),
    "dsk_ahc": (c_int32, [c_void_p, c_int32, c_int64, c_int32, c_int32, c_double, c_void_p, POINTER(c_int32), c_void_p,
                          POINTER(c_int32), c_void_p]),
    "dsk_spectral_cluster": (c_int32, [c_void_p, c_int32, c_int64, c_void_p, c_int32, c_int32, c_int32, c_int32]
                             + [c_void_p] * 8),
    "dsk_class_sums_f64": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                     c_void_p]),
    "dsk_gram_f64": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    "dsk_affine_norm_f64": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "dsk_plda_score_trials": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                        c_void_p]),
    "dsk_plda_score_matrix": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_int64,
                                        c_void_p]),
    "dsk_vbx": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_double, c_double,
                          c_double, c_double, c_int32, c_double] + [c_void_p] * 6),
    "dsk_linear_forward": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_linear_backward": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "dsk_cross_entropy": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_cross_entropy_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_adagrad_step": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_double, c_double, c_double, c_double,
                                   c_int64, c_float, c_void_p, c_void_p]),
    "dsk_set_defer_running_stats": (c_int32, [c_void_p, c_int32]),
    "dsk_train_ctx_commit_stats": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "dsk_pipeline_create": (c_int32, [POINTER(c_void_p), c_void_p, c_int32, c_int32]),
    "dsk_pipeline_destroy": (c_int32, [c_void_p]),
    "dsk_pipeline_submit": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, POINTER(c_int64)]),
    "dsk_pipeline_submit_device": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, POINTER(c_int64)]),
    "dsk_pipeline_join": (c_int32, [c_void_p, c_void_p]),
    "dsk_pipeline_wait": (c_int32, [c_void_p, c_int64]),
    "dsk_pipeline_sync": (c_int32, [c_void_p]),
    "dsk_pipeline_lane_stream": (c_int32, [c_void_p, c_int32, POINTER(c_void_p)]),
    "dsk_fbank_num_frames": (c_int64, [c_int64, c_int32]),
    "dsk_fbank": (c_int32, [c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_fbank_frame_offsets": (c_int32, [c_void_p, c_int32, c_int32, c_void_p]),
    "dsk_fbank_batch": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "dsk_fbank_crops": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int32,
                                  c_void_p, c_int32, c_void_p, c_void_p]),
    "dsk_fbank_batch_vad": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_double, c_double,
                                      c_int32, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_frame_runs": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int64, c_int64, c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "dsk_gather_runs": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p,
                                  c_void_p]),
    "dsk_fbank_filterbank": (c_int32, [c_int32, c_void_p]),
    "dsk_wave_augment": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p,
                                   c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_int32] + [c_void_p] * 5),
    "dsk_speed_filter": (c_int32, [c_int32, c_int32, c_void_p]),
    "dsk_wave_augment_speed": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                         c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_int32]
                               + [c_void_p] * 5 + [c_int32] + [c_void_p] * 3),
    "dsk_fbank_segments": (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_int32,
                                     c_void_p, c_int32, c_void_p, c_void_p]),
    "dsk_threshold_counts": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load libdsk.so (building it first if it is missing or its sources changed). Raises if unavailable — no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        try:
            build()
        except Exception as e:  # a GPU box without nvcc must ship the prebuilt .so
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"libdsk.so is missing and could not be built: {e}") from e
            if os.environ.get("DSK_STRICT_BUILD") == "1":
                raise RuntimeError(f"libdsk.so does not match csrc/ and the rebuild failed: {e}") from e
            import warnings

            warnings.warn(f"libdsk.so was built from DIFFERENT sources than csrc/ and the rebuild failed ({e}); "
                          f"loading the stale library (set DSK_STRICT_BUILD=1 to make this an error)", RuntimeWarning)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().dsk_last_error()
        raise RuntimeError(f"libdsk {what} failed ({rc}): {msg.decode() if msg else '?'}")


def cur_stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


def ptr(t) -> int:
    """Raw device pointer of a tensor (None -> NULL)."""
    return 0 if t is None else t.data_ptr()
