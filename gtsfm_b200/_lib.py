"""ctypes binding of libgtsfm_b200.so (include/gtsfm_b200.h).  No fallback: a missing library or GPU raises."""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional

import numpy as np

LIB_PATH = Path(__file__).resolve().parent / "libgtsfm_b200.so"

_lib: Optional[C.CDLL] = None


class B200Error(RuntimeError):
    pass


class LightGlueParams(C.Structure):
    _fields_ = [("depth_confidence", C.c_double), ("width_confidence", C.c_double), ("filter_threshold", C.c_double),
                ("prune_min_kpts", C.c_int), ("fp16_attention", C.c_int)]


class LightGluePair(C.Structure):
    _fields_ = [("kp0", C.c_void_p), ("desc0", C.c_void_p), ("n0", C.c_int), ("kp1", C.c_void_p), ("desc1", C.c_void_p), ("n1", C.c_int),
                ("out_matches", C.c_void_p), ("out_scores", C.c_void_p), ("out_k", C.c_int), ("out_stop_layer", C.c_int),
                ("enc0", C.c_void_p), ("enc1", C.c_void_p)]


class LightGlueImage(C.Structure):
    _fields_ = [("kp", C.c_void_p), ("desc", C.c_void_p), ("n", C.c_int), ("out", C.c_void_p)]


class MnnPair(C.Structure):
    _fields_ = [("desc0", C.c_void_p), ("n0", C.c_int), ("desc1", C.c_void_p), ("n1", C.c_int), ("out_matches", C.c_void_p),
                ("out_dist", C.c_void_p), ("out_k", C.c_int)]


MNN_ERR_RATIO = -4  # b2_mnn_*: ratio test with fewer than 2 descriptors on one side


class SiftKeypoint(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float), ("response", C.c_float),
                ("octave", C.c_int32)]


# numpy twin of b2_sift_keypoint (24 bytes, the fields of cv2.KeyPoint)
SIFT_KEYPOINT_DTYPE = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                                ("response", np.float32), ("octave", np.int32)])


class SiftImage(C.Structure):
    _fields_ = [("image", C.c_void_p), ("mask", C.c_void_p), ("max_keypoints", C.c_int), ("out_keypoints", C.c_void_p),
                ("out_desc", C.c_void_p), ("out_n", C.c_int), ("out_total", C.c_int)]


class OrbImage(C.Structure):  # b2_orb_image: b2_sift_image's layout
    _fields_ = SiftImage._fields_


class D2NetImage(C.Structure):
    _fields_ = [("image", C.c_void_p), ("max_keypoints", C.c_int), ("out_xy", C.c_void_p), ("out_scores", C.c_void_p),
                ("out_desc", C.c_void_p), ("out_n", C.c_int), ("out_total", C.c_int)]


class JpegImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size", C.c_size_t), ("out", C.c_void_p), ("out_pitch", C.c_size_t), ("out_status", C.c_int),
                ("out_rounds", C.c_int)]


SIFT_CAPACITY = -5  # b2_sift_detect_host / b2_orb_detect_host: more keypoints than the capacity; *out_n holds the count needed


class RansacParams(C.Structure):
    _fields_ = [("threshold", C.c_double), ("confidence", C.c_double), ("max_iters", C.c_int), ("seed", C.c_uint64)]


class RansacProblem(C.Structure):  # b2_ransac_problem
    _fields_ = [("kp1", C.c_void_p), ("kp2", C.c_void_p), ("matches", C.c_void_p), ("x1", C.c_void_p), ("x2", C.c_void_p),
                ("k", C.c_int), ("mode", C.c_int), ("max_iters", C.c_int), ("cal1", C.c_double * 3), ("cal2", C.c_double * 3),
                ("threshold", C.c_double), ("mask", C.c_void_p)]


class LinearProblem(C.Structure):  # b2_linear_problem (tests only)
    _fields_ = [("a1", C.c_void_p), ("lda1", C.c_int), ("a2", C.c_void_p), ("lda2", C.c_int), ("b", C.c_void_p), ("ldb", C.c_int),
                ("resid", C.c_void_p), ("ldr", C.c_int), ("c", C.c_void_p), ("ldc", C.c_int), ("c_hi", C.c_void_p), ("c_lo", C.c_void_p),
                ("ldch", C.c_int), ("m", C.c_int), ("n", C.c_int)]


class LinearLaunch(C.Structure):  # b2_linear_launch (tests only)
    _fields_ = [("path", C.c_int), ("k1", C.c_int), ("k2", C.c_int), ("per_problem_b", C.c_int), ("bias", C.c_void_p),
                ("scale", C.c_float), ("relu", C.c_int), ("gelu", C.c_int), ("head_major", C.c_int), ("lo_unscaled", C.c_int),
                ("resid_in_place", C.c_int)]


class ConvLayer(C.Structure):  # b2_conv_layer (tests only)
    _fields_ = [("path", C.c_int), ("dilation", C.c_int), ("pool", C.c_int), ("relu", C.c_int), ("ctas", C.c_int), ("height", C.c_int),
                ("width", C.c_int), ("cin", C.c_int), ("cout", C.c_int), ("in_", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p),
                ("out", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p)]


class RansacResult(C.Structure):  # b2_ransac_result
    _fields_ = [("status", C.c_int), ("num_inliers", C.c_int), ("model", C.c_double * 9), ("R", C.c_double * 9), ("t", C.c_double * 3)]


class RansacCandidate(C.Structure):
    _fields_ = [("model", C.c_double * 9), ("cost", C.c_double), ("ninl", C.c_int), ("valid", C.c_int)]


class RansacTrace(C.Structure):  # b2_ransac_trace (tests only)
    _fields_ = [("batch", C.c_int), ("max_records", C.c_int), ("nsol", C.c_void_p), ("models", C.c_void_p), ("cost", C.c_void_p),
                ("ninl", C.c_void_p), ("selected", C.c_void_p), ("more", C.c_void_p), ("batches", C.c_int), ("ext_go", C.c_int),
                ("records", C.c_int), ("prerefine", RansacCandidate * 8), ("refined", RansacCandidate * 8), ("pick", RansacCandidate),
                ("mask_count", C.c_int), ("votes", C.c_int * 4), ("winner", C.c_int), ("pose_cands", C.c_double * 21)]


class LmedsParams(C.Structure):  # b2_lmeds_params
    _fields_ = [("confidence", C.c_double * 2)]


class LmedsTrace(C.Structure):  # b2_lmeds_trace (tests only)
    _fields_ = [("cap", C.c_int), ("idx", C.c_void_p), ("nsol", C.c_void_p), ("models", C.c_void_p), ("medians", C.c_void_p),
                ("niters", C.c_int), ("drawn", C.c_int), ("slot", C.c_int), ("min_median", C.c_float), ("sigma", C.c_double),
                ("thr", C.c_float), ("count", C.c_int)]


class TwoViewProblem(C.Structure):  # b2_twoview_problem
    _fields_ = [("kp1", C.c_void_p), ("kp2", C.c_void_p), ("matches", C.c_void_p), ("mask", C.c_void_p), ("k", C.c_int),
                ("cal1", C.c_double * 3), ("cal2", C.c_double * 3), ("R", C.c_double * 9), ("t", C.c_double * 3),
                ("out_mask", C.c_void_p), ("out_rows", C.c_void_p)]


class TwoViewParams(C.Structure):  # b2_twoview_params
    _fields_ = [("max_iters", C.c_int), ("min_num_inliers", C.c_int), ("min_inlier_ratio", C.c_double),
                ("ba_reproj_error_threshold", C.c_double), ("tri_reproj_error_threshold", C.c_double),
                ("min_triangulation_angle", C.c_double)]


class TwoViewResult(C.Structure):  # b2_twoview_result
    _fields_ = [("status", C.c_int), ("num_rows", C.c_int), ("num_verified", C.c_int), ("num_tracks", C.c_int),
                ("iterations", C.c_int), ("bundle_adjusted", C.c_int), ("indeterminate", C.c_int), ("trace_len", C.c_int),
                ("R", C.c_double * 9), ("t", C.c_double * 3), ("final_error", C.c_double)]


class TwoViewEvalProblem(C.Structure):  # b2_twoview_eval_problem
    _fields_ = [("kp1", C.c_void_p), ("kp2", C.c_void_p), ("matches", C.c_void_p), ("mask", C.c_void_p), ("k", C.c_int),
                ("has_pose", C.c_int), ("has_gt", C.c_int), ("pad_", C.c_int), ("R", C.c_double * 9), ("t", C.c_double * 3),
                ("wRi1", C.c_double * 9), ("wti1", C.c_double * 3), ("wRi2", C.c_double * 9), ("wti2", C.c_double * 3),
                ("cal1", C.c_double * 3), ("cal2", C.c_double * 3), ("out_d2", C.c_void_p), ("out_inlier", C.c_void_p)]


class TwoViewEvalParams(C.Structure):  # b2_twoview_eval_params
    _fields_ = [("eval_threshold_px", C.c_double)]


class TwoViewEvalResult(C.Structure):  # b2_twoview_eval_result
    _fields_ = [("num_rows", C.c_int), ("num_inliers_gt", C.c_int), ("no_gt", C.c_int), ("no_rows", C.c_int),
                ("inlier_avg_reproj_error_gt", C.c_double), ("outlier_avg_reproj_error_gt", C.c_double),
                ("R_error_deg", C.c_double), ("U_error_deg", C.c_double)]


class ViewGraphParams(C.Structure):  # b2_viewgraph_params
    _fields_ = [("criterion", C.c_int), ("pad_", C.c_int), ("error_threshold_deg", C.c_double)]


VG_MEDIAN, VG_MIN = 0, 1  # B2_VG_MEDIAN, B2_VG_MIN


class TriangulationParams(C.Structure):  # b2_triangulation_params
    _fields_ = [("mode", C.c_int), ("num_hypotheses", C.c_int), ("reproj_error_threshold", C.c_double),
                ("min_triangulation_angle", C.c_double), ("seed", C.c_uint64)]


TRI_NO_RANSAC, TRI_SAMPLE_UNIFORM = 0, 1  # B2_TRI_NO_RANSAC, B2_TRI_SAMPLE_UNIFORM

_vp, _i, _f, _sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
_ip = C.POINTER(C.c_int)

# name -> (restype, argtypes): every symbol include/gtsfm_b200.h declares
SIGNATURES = {
    "b2_version": (_i, []),
    "b2_create": (_i, [_i, C.POINTER(_vp)]),
    "b2_destroy": (None, [_vp]),
    "b2_last_error": (C.c_char_p, [_vp]),
    "b2_launch_count": (C.c_uint64, [_vp]),
    "b2_h2d_bytes": (C.c_uint64, [_vp]),
    "b2_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int64]),
    "b2_profile_start": (_i, [_vp, C.c_char_p]),
    "b2_profile_stop": (_i, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "b2_debug_fetch": (C.c_int64, [_vp, C.c_char_p, _vp, C.c_int64]),
    "b2_debug_linear_host": (_i, [_vp, C.POINTER(LinearLaunch), C.POINTER(LinearProblem), _i]),
    "b2_debug_conv_host": (_i, [_vp, C.POINTER(ConvLayer)]),
    "b2_debug_gemm_segments_host": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "b2_debug_attention_host": (_i, [_vp, _i, _ip, _ip, _i, _f, _i, _vp, _vp, _vp, _vp]),
    "b2_debug_superglue_assign_host": (_i, [_vp, _i, _i, _vp, _i, _i, _f, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip]),
    "b2_debug_lightglue_assign_host": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip,
                                            _ip]),
    "b2_debug_lightglue_argmax_host": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _ip]),
    "b2_debug_lightglue_posenc_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_debug_lightglue_ln_gelu_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_debug_lightglue_rowheads_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_debug_lightglue_prune_host": (_i, [_vp, _i, _vp, _vp, _vp, _f, _f, _vp, _vp]),
    "b2_debug_lightglue_gather_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_debug_lightglue_filter_host": (_i, [_vp, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _ip]),
    "b2_superpoint_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_superpoint_detect_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _f, _i, _i, _vp, _vp, _i, _ip, C.POINTER(C.c_uint64), _vp]),
    "b2_superpoint_describe_dev": (_i, [_vp, C.c_uint64, _vp, _i, _vp, _vp]),
    "b2_superpoint_extract_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _f, _i, _i, _i, _vp, _vp, _vp, _ip, _vp]),
    "b2_superpoint_extract_async_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _f, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b2_superpoint_finish_dev": (_i, [_vp, _vp]),
    "b2_superpoint_detect_host": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _i, _vp, _vp, _i, _ip, C.POINTER(C.c_uint64)]),
    "b2_superpoint_describe_host": (_i, [_vp, C.c_uint64, _vp, _i, _vp]),
    "b2_image_resize_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _i, _i, _vp]),
    "b2_lightglue_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_lightglue_qkv_rows": (_i, [_vp]),
    "b2_lightglue_match_dev": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, C.POINTER(LightGlueParams), _vp, _vp, _ip, _ip, _vp]),
    "b2_lightglue_match_host": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, C.POINTER(LightGlueParams), _vp, _vp, _ip, _ip]),
    "b2_lightglue_match_batched_dev": (_i, [_vp, C.POINTER(LightGluePair), _i, C.POINTER(LightGlueParams), _vp]),
    "b2_lightglue_trace_count": (_i, [_vp]),
    "b2_lightglue_trace_get": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_lightglue_encoded_bytes": (_sz, [_i]),
    "b2_lightglue_encode_batched_dev": (_i, [_vp, C.POINTER(LightGlueImage), _i, C.POINTER(LightGlueParams), _vp]),
    "b2_superglue_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_superglue_match_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _ip, _vp]),
    "b2_superglue_match_host": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _ip]),
    "b2_superglue_trace_count": (_i, [_vp]),
    "b2_superglue_trace_get": (_i, [_vp, _i, _vp, _vp]),
    "b2_netvlad_blob_floats": (_sz, []),
    "b2_netvlad_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_netvlad_describe_dev": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "b2_netvlad_describe_host": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "b2_megaloc_blob_floats": (_sz, []),
    "b2_megaloc_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_megaloc_describe_dev": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "b2_megaloc_describe_host": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "b2_megaloc_describe_u8_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _vp]),
    "b2_megaloc_resize_u8_dev": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _vp]),
    "b2_similarity_pairs_host": (_i, [_vp, _vp, _i, _i, _i, _f, _vp, _vp]),
    "b2_ransac_essential_host": (_i, [_vp, _vp, _vp, _i, C.POINTER(RansacParams), _vp, _vp, _ip, _vp, _vp]),
    "b2_ransac_fundamental_host": (_i, [_vp, _vp, _vp, _i, C.POINTER(RansacParams), _vp, _vp, _ip]),
    "b2_ransac_essential_dev": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, C.POINTER(RansacParams), _vp, _vp, _ip, _vp, _vp, _vp]),
    "b2_ransac_verify_batched_dev": (_i, [_vp, C.POINTER(RansacProblem), _i, C.POINTER(RansacParams), C.POINTER(RansacResult), _vp]),
    "b2_ransac_workspace_bytes": (_sz, [C.POINTER(RansacProblem)]),
    "b2_ransac_plan": (_i, [C.POINTER(RansacProblem), _i, _sz, _ip]),
    "b2_lmeds_verify_batched_dev": (_i, [_vp, C.POINTER(RansacProblem), _i, C.POINTER(LmedsParams), C.POINTER(RansacResult), _vp]),
    "b2_lmeds_workspace_bytes": (_sz, [C.POINTER(RansacProblem), C.POINTER(LmedsParams)]),
    "b2_lmeds_plan": (_i, [C.POINTER(RansacProblem), _i, C.POINTER(LmedsParams), _sz, _ip]),
    "b2_debug_lmeds_trace_host": (_i, [_vp, _i, _vp, _vp, _i, C.POINTER(LmedsParams), _i, C.POINTER(LmedsTrace), C.POINTER(RansacResult), _vp]),
    "b2_twoview_eval_batched_dev": (_i, [_vp, C.POINTER(TwoViewEvalProblem), _i, C.POINTER(TwoViewEvalParams),
                                        C.POINTER(TwoViewEvalResult), _vp]),
    "b2_viewgraph_cycle_filter_host": (_i, [_vp, _vp, _vp, _i, C.POINTER(ViewGraphParams), _vp, _vp, _vp, _vp]),
    "b2_triangulate_tracks_host": (_i, [_vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, _i, C.POINTER(TriangulationParams), _vp, _vp, _vp,
                                        _vp, _vp]),
    "b2_debug_viewgraph_triplets_host": (_i, [_vp, _vp, _vp, _i, C.c_int64, _vp, _vp, C.POINTER(C.c_int64), _vp]),
    "b2_twoview_ba_batched_dev": (_i, [_vp, C.POINTER(TwoViewProblem), _i, C.POINTER(TwoViewParams), C.POINTER(TwoViewResult), _vp]),
    "b2_twoview_ba_workspace_bytes": (_sz, [C.POINTER(TwoViewProblem), C.POINTER(TwoViewParams)]),
    "b2_twoview_ba_plan": (_i, [C.POINTER(TwoViewProblem), _i, C.POINTER(TwoViewParams), _sz, _ip]),
    "b2_debug_twoview_ba_trace_host": (_i, [_vp, C.POINTER(TwoViewProblem), _i, C.POINTER(TwoViewParams), C.POINTER(TwoViewResult), _vp,
                                            _vp]),
    "b2_ransac_sync_count": (C.c_uint64, [_vp]),
    "b2_recover_pose_host": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _ip]),
    "b2_debug_ransac_trace_host": (_i, [_vp, _i, _vp, _vp, _i, C.POINTER(RansacParams), C.POINTER(RansacTrace), _vp, _vp, _ip, _vp, _vp]),
    "b2_debug_recover_pose_host": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _ip, _vp, _vp, _ip]),
    "b2_mnn_match_batched_dev": (_i, [_vp, C.POINTER(MnnPair), _i, _i, _i, C.c_double, _vp]),
    "b2_mnn_match_host": (_i, [_vp, _vp, _i, _vp, _i, _i, _i, C.c_double, _vp, _vp, _ip]),
    "b2_sift_detect_batched_dev": (_i, [_vp, C.POINTER(SiftImage), _i, _i, _i, _i, _sz, _vp]),
    "b2_sift_detect_host": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _ip]),
    "b2_orb_detect_batched_dev": (_i, [_vp, C.POINTER(OrbImage), _i, _i, _i, _i, _sz, _vp]),
    "b2_orb_detect_host": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _ip]),
    "b2_d2net_blob_floats": (_sz, []),
    "b2_d2net_norm_table": (_i, [_vp]),
    "b2_d2net_set_weights": (_i, [_vp, _vp, _sz]),
    "b2_d2net_detect_batched_dev": (_i, [_vp, C.POINTER(D2NetImage), _i, _i, _i, _i, _sz, _vp]),
    "b2_d2net_detect_host": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _ip, _ip]),
    "b2_debug_d2net_avgpool_host": (_i, [_vp, _vp, _i, _i, _vp]),
    "b2_debug_d2net_rank_host": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "b2_jpeg_status_string": (C.c_char_p, [_i]),
    "b2_jpeg_info_host": (_i, [_vp, _sz, _ip, _ip, _ip]),
    "b2_jpeg_decode_batched_dev": (_i, [_vp, C.POINTER(JpegImage), _i, _vp]),
}


def load() -> C.CDLL:
    """dlopen the in-tree library and bind every declared symbol.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise B200Error(f"{LIB_PATH} is missing: run `python -m gtsfm_b200.build` (there is no CPU fallback)")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def ptr(a) -> C.c_void_p:
    """Raw pointer of a C-contiguous numpy array, a torch tensor (data_ptr) or an int address."""
    if a is None:
        return C.c_void_p(0)
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        assert a.is_contiguous(), "tensor must be contiguous"
        return C.c_void_p(a.data_ptr())
    return C.c_void_p(int(a))


class Context:
    """Owns one b2_context (one CUDA device, one internal stream).  Created lazily by the plugins."""

    def __init__(self, device: int = 0):
        self._lib = load()
        h = C.c_void_p()
        rc = self._lib.b2_create(int(device), C.byref(h))
        if rc != 0 or not h:
            raise B200Error(
                f"b2_create(device={device}) failed with {rc}: an sm_90 (H100) GPU is required; there is no CPU fallback")
        self.handle = h
        self.device = device
        self.options = {}  # what set_option was given, by name (the last value)

    def check(self, rc: int, what: str) -> None:
        if rc < 0:
            raise B200Error(f"{what} failed ({rc}): {self._lib.b2_last_error(self.handle).decode()}")

    @property
    def lib(self) -> C.CDLL:
        return self._lib

    def launch_count(self) -> int:
        return int(self._lib.b2_launch_count(self.handle))

    def ransac_sync_count(self) -> int:
        """Stream synchronisations the RANSAC entry points have performed through this context."""
        return int(self._lib.b2_ransac_sync_count(self.handle))

    def set_option(self, name: str, value: int) -> None:
        self.check(self._lib.b2_set_option(self.handle, name.encode(), int(value)), f"set_option({name})")
        self.options[name] = int(value)

    def h2d_bytes(self) -> int:
        return int(self._lib.b2_h2d_bytes(self.handle))

    def profile_start(self, kernel_prefix: str) -> None:
        self.check(self._lib.b2_profile_start(self.handle, kernel_prefix.encode()), "profile_start")

    def profile_stop(self):
        ms, n, w = C.c_double(0), C.c_uint64(0), C.c_double(0)
        self.check(self._lib.b2_profile_stop(self.handle, C.byref(ms), C.byref(n), C.byref(w)), "profile_stop")
        return ms.value, int(n.value), w.value

    def debug_fetch(self, name: str, max_floats: int) -> np.ndarray:
        out = np.empty(max_floats, np.float32)
        n = self._lib.b2_debug_fetch(self.handle, name.encode(), ptr(out), max_floats)
        self.check(int(n), f"debug_fetch({name})")
        return out[:n]

    def close(self) -> None:
        if getattr(self, "handle", None):
            self._lib.b2_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
