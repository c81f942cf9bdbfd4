"""ctypes binding of libk210yolo_b200.so (the C-ABI declared in include/k210_yolo_b200.h).

There is no CPU fallback anywhere in this package: if the shared library has not been built
(``python -c "import __graft_entry__ as g; g.build()"``) importing this module raises, and every
compute entry point raises ``K2YError`` when no CUDA device is usable.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libk210yolo_b200.so")

K2Y_OK = 0
MATH_FP32_SIMT = 0
MATH_TC_3XTF32 = 1
MATH_TC_TF32 = 2
MATH_TC_BF16X3 = 3
MATH_NAMES = {MATH_FP32_SIMT: "fp32_simt", MATH_TC_3XTF32: "tc_3xtf32", MATH_TC_TF32: "tc_tf32", MATH_TC_BF16X3: "tc_bf16x3"}


class K2YError(RuntimeError):
    pass


class LayerInfo(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 64), ("bn_name", ctypes.c_char * 64), ("kind", c_int32),
                ("kh", c_int32), ("kw", c_int32), ("cin", c_int32), ("cout", c_int32), ("stride", c_int32),
                ("has_bias", c_int32)]


class Det(ctypes.Structure):
    _fields_ = [("ymin", c_float), ("xmin", c_float), ("ymax", c_float), ("xmax", c_float),
                ("score", c_float), ("index", c_int32)]


class DetectCfg(ctypes.Structure):
    _fields_ = [("n_layers", c_int32), ("layer_h", c_int32 * 3), ("layer_w", c_int32 * 3),
                ("anchor_num", c_int32), ("class_num", c_int32), ("anchors", c_float * 48),
                ("in_h", c_int32), ("in_w", c_int32), ("obj_thresh", c_float), ("iou_thresh", c_float),
                ("max_per_class", c_int32)]


class RegionCfg(ctypes.Structure):
    _fields_ = [("layer_w", c_int32), ("layer_h", c_int32), ("anchor_num", c_int32), ("classes", c_int32),
                ("net_w", c_int32), ("net_h", c_int32), ("image_w", c_int32), ("image_h", c_int32),
                ("anchors", c_float * 16), ("threshold", c_float), ("nms_value", c_float)]


class JpegInfo(ctypes.Structure):
    _fields_ = [("height", c_int32), ("width", c_int32), ("components", c_int32), ("h_samp", c_int32 * 4), ("v_samp", c_int32 * 4),
                ("restart_interval", c_int32), ("precision", c_int32), ("sof_marker", c_int32), ("gpu_decodable", c_int32),
                ("entropy_offset", c_int32), ("reason", ctypes.c_char * 64)]


class JpegProgressiveInfo(ctypes.Structure):
    _fields_ = [("height", c_int32), ("width", c_int32), ("components", c_int32), ("sof_marker", c_int32), ("scans", c_int32),
                ("levels", c_int32), ("gpu_decodable", c_int32), ("reason", ctypes.c_char * 64)]


class PngInfo(ctypes.Structure):
    _fields_ = [("height", c_int32), ("width", c_int32), ("color_type", c_int32), ("bit_depth", c_int32), ("interlace", c_int32),
                ("idat_chunks", c_int32), ("stream_bytes", c_int64), ("gpu_decodable", c_int32), ("reason", ctypes.c_char * 64)]


# Every symbol include/k210_yolo_b200.h declares (tests/test_abi.py checks the two lists agree).
_SIGNATURES = {
    "k2y_last_error": (c_char_p, []),
    "k2y_version": (c_int, []),
    "k2y_cuda_available": (c_int, []),
    "k2y_net_create": (c_int, [c_char_p, c_int, c_int, c_float, c_int, c_int, c_int, c_int, POINTER(c_void_p)]),
    "k2y_net_destroy": (c_int, [c_void_p]),
    "k2y_net_num_layers": (c_int, [c_void_p, POINTER(c_int)]),
    "k2y_net_layer_info": (c_int, [c_void_p, c_int, POINTER(LayerInfo)]),
    "k2y_net_set_weight": (c_int, [c_void_p, c_char_p, c_char_p, c_void_p, POINTER(c_int64), c_int]),
    "k2y_net_finalize": (c_int, [c_void_p]),
    "k2y_net_set_math": (c_int, [c_void_p, c_int]),
    "k2y_net_get_math": (c_int, [c_void_p, POINTER(c_int)]),
    "k2y_net_set_use_graph": (c_int, [c_void_p, c_int]),
    "k2y_net_num_outputs": (c_int, [c_void_p, POINTER(c_int)]),
    "k2y_net_output_shape": (c_int, [c_void_p, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "k2y_net_workspace_bytes": (c_int, [c_void_p, POINTER(c_size_t)]),
    "k2y_net_bind": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_void_p), c_int]),
    "k2y_net_bind_u8": (c_int, [c_void_p, c_void_p, c_void_p]),
    "k2y_net_bind_input": (c_int, [c_void_p, c_void_p]),
    "k2y_net_bind_heads": (c_int, [c_void_p, POINTER(c_void_p), c_int]),
    "k2y_net_set_sm_limit": (c_int, [c_void_p, c_int]),
    "k2y_net_run": (c_int, [c_void_p, c_int, c_void_p]),
    "k2y_net_predict_host": (c_int, [c_void_p, c_void_p, c_int, POINTER(c_void_p), c_void_p]),
    "k2y_net_launches_per_run": (c_int, [c_void_p, POINTER(c_int)]),
    "k2y_net_schedule_len": (c_int, [c_void_p, POINTER(c_int)]),
    "k2y_net_profile": (c_int, [c_void_p, c_int, c_void_p, POINTER(c_float), c_int]),
    "k2y_net_launch_info": (c_int, [c_void_p, c_int, ctypes.c_char_p, c_int, POINTER(ctypes.c_double), POINTER(ctypes.c_double)]),
    "k2y_net_set_keep_all": (c_int, [c_void_p, c_int]),
    "k2y_net_read_layer": (c_int, [c_void_p, c_char_p, c_int, c_void_p, c_size_t, POINTER(c_int), POINTER(c_int),
                                   POINTER(c_int)]),
    "k2y_conv2d": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 11 +
                   [c_float, c_int, c_void_p]),
    "k2y_detect_workspace_bytes": (c_int, [POINTER(DetectCfg), c_int, POINTER(c_size_t)]),
    "k2y_detect_keras": (c_int, [POINTER(DetectCfg), POINTER(c_void_p), c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_size_t, c_void_p]),
    "k2y_detect_keras_strided": (c_int, [POINTER(DetectCfg), POINTER(c_void_p), c_int, c_void_p, c_void_p, c_void_p,
                                         ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_size_t, c_void_p]),
    "k2y_merge_views_max_records": (c_int, []),
    "k2y_merge_views": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                                ctypes.c_longlong, ctypes.c_longlong, c_void_p]),
    "k2y_merge_views_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong,
                                   c_void_p]),
    "k2y_merge_views_mirror": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int,
                                       c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, ctypes.c_longlong,
                                       ctypes.c_longlong, c_void_p]),
    "k2y_track_state_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "k2y_track_update": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                 ctypes.c_double, c_void_p, c_void_p, c_void_p]),
    "k2y_bytetrack_state_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "k2y_bytetrack_update": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_int, c_int, c_int,
                                     ctypes.c_double, ctypes.c_double, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "k2y_ocsort_state_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "k2y_ocsort_update": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_int, c_int, c_int,
                                  ctypes.c_double, c_int, c_int, ctypes.c_double, c_int, ctypes.c_double, c_int, c_void_p, c_void_p,
                                  c_void_p]),
    "k2y_track_update_streams": (c_int, [c_void_p, c_int, c_size_t, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p,
                                         c_int, c_int, c_int, c_int, c_int, ctypes.c_double, c_void_p, c_void_p, c_void_p]),
    "k2y_bytetrack_update_streams": (c_int, [c_void_p, c_int, c_size_t, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p,
                                             c_void_p, c_int, c_int, c_int, ctypes.c_double, ctypes.c_double, c_int, c_int, c_void_p,
                                             c_void_p, c_void_p]),
    "k2y_ocsort_update_streams": (c_int, [c_void_p, c_int, c_size_t, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p,
                                          c_int, c_int, c_int, ctypes.c_double, c_int, c_int, ctypes.c_double, c_int, ctypes.c_double,
                                          c_int, c_void_p, c_void_p, c_void_p]),
    "k2y_comm_unique_id": (c_int, [c_void_p]),
    "k2y_comm_create": (c_int, [c_void_p, c_int, c_int, c_int, POINTER(c_void_p)]),
    "k2y_comm_destroy": (c_int, [c_void_p]),
    "k2y_comm_info": (c_int, [c_void_p, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "k2y_allgather_detections": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "k2y_region_workspace_bytes": (c_int, [POINTER(RegionCfg), c_int, POINTER(c_size_t)]),
    "k2y_region_run": (c_int, [POINTER(RegionCfg), c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                               c_void_p]),
    "k2y_tc_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "k2y_tc_plan_budget": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "k2y_xywh_to_all": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_int, c_int, POINTER(c_float), c_void_p, c_void_p, c_void_p]),
    "k2y_correct_box": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_float, c_float, c_float, c_float, c_void_p, c_void_p]),
    "k2y_nms_workspace_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "k2y_nms_boxes": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "k2y_expf_eval": (c_int, [c_int, c_void_p, c_void_p, ctypes.c_longlong, c_void_p]),
    "k2y_pr_counts": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_float, c_int, c_void_p, c_void_p]),
    "k2y_letterbox_u8": (c_int, [c_void_p, c_int, c_int, POINTER(ctypes.c_double), c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "k2y_letterbox_u8_batch": (c_int, [c_void_p, c_int, POINTER(ctypes.c_longlong), POINTER(c_int), POINTER(ctypes.c_double), c_void_p,
                                       c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "k2y_letterbox_u8_views": (c_int, [c_void_p, c_int, POINTER(ctypes.c_longlong), POINTER(c_int), POINTER(c_int), POINTER(ctypes.c_double),
                                       c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "k2y_letterbox_u8_views_mirror": (c_int, [c_void_p, c_int, POINTER(ctypes.c_longlong), POINTER(c_int), POINTER(c_int), POINTER(c_int),
                                              POINTER(ctypes.c_double), c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "k2y_jpeg_inspect": (c_int, [c_void_p, c_size_t, POINTER(JpegInfo)]),
    "k2y_jpeg_plan": (c_int, [POINTER(c_void_p), POINTER(c_size_t), c_int, POINTER(ctypes.c_longlong), POINTER(ctypes.c_longlong),
                              c_void_p, c_size_t, POINTER(c_size_t)]),
    "k2y_jpeg_workspace_bytes": (c_int, [c_void_p, POINTER(c_size_t)]),
    "k2y_jpeg_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "k2y_jpeg_progressive_inspect": (c_int, [c_void_p, c_size_t, POINTER(JpegProgressiveInfo)]),
    "k2y_jpeg_progressive_plan": (c_int, [POINTER(c_void_p), POINTER(c_size_t), c_int, POINTER(ctypes.c_longlong),
                                          POINTER(ctypes.c_longlong), c_void_p, c_size_t, POINTER(c_size_t)]),
    "k2y_jpeg_progressive_workspace_bytes": (c_int, [c_void_p, POINTER(c_size_t)]),
    "k2y_jpeg_progressive_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "k2y_png_inspect": (c_int, [c_void_p, c_size_t, POINTER(PngInfo)]),
    "k2y_png_plan": (c_int, [POINTER(c_void_p), POINTER(c_size_t), c_int, POINTER(ctypes.c_longlong), POINTER(ctypes.c_longlong),
                             c_void_p, c_size_t, POINTER(c_size_t)]),
    "k2y_png_workspace_bytes": (c_int, [c_void_p, POINTER(c_size_t)]),
    "k2y_png_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "k2y_jpeg_encode_plan": (c_int, [c_int, POINTER(c_int), POINTER(ctypes.c_longlong), c_int, c_void_p, c_size_t, POINTER(c_size_t)]),
    "k2y_jpeg_encode_header": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t, POINTER(c_size_t)]),
    "k2y_jpeg_encode_workspace_bytes": (c_int, [c_void_p, POINTER(c_size_t), POINTER(c_size_t)]),
    "k2y_jpeg_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "k2y_render_detections": (c_int, [c_void_p, c_int, POINTER(ctypes.c_longlong), POINTER(c_int), POINTER(c_void_p), c_void_p, c_void_p,
                                      ctypes.c_longlong, ctypes.c_longlong, c_int, c_int, c_void_p, c_void_p]),
    "k2y_render_tracks": (c_int, [c_void_p, c_int, POINTER(ctypes.c_longlong), POINTER(c_int), POINTER(c_void_p), c_void_p, c_void_p,
                                  c_void_p, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_longlong, c_int, c_int, c_void_p, c_int,
                                  c_void_p]),
    "k2y_ap_create": (c_int, [c_int, c_int, POINTER(c_float), c_int, c_int, POINTER(c_void_p)]),
    "k2y_ap_destroy": (c_int, [c_void_p]),
    "k2y_ap_match": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong, c_int, c_void_p, c_void_p, c_int,
                             c_void_p]),
    "k2y_ap_result": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(ctypes.c_uint), c_void_p]),
    "k2y_ap_reset": (c_int, [c_void_p, c_void_p]),
    "k2y_ap_tp_flags": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, POINTER(ctypes.c_longlong), c_void_p]),
    "k2y_coco_create": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_int, c_void_p, c_void_p, c_int, POINTER(c_void_p)]),
    "k2y_coco_destroy": (c_int, [c_void_p]),
    "k2y_coco_match": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong, c_int, c_void_p, c_void_p]),
    "k2y_coco_result": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(ctypes.c_uint), c_void_p]),
    "k2y_coco_reset": (c_int, [c_void_p, c_void_p]),
    "k2y_mot_create": (c_int, [c_int, c_int, POINTER(c_void_p)]),
    "k2y_mot_destroy": (c_int, [c_void_p]),
    "k2y_mot_add_sequence": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, POINTER(c_int)]),
    "k2y_mot_update": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_longlong,
                               c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "k2y_mot_result": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(ctypes.c_uint), c_void_p]),
    "k2y_mot_result_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(ctypes.c_uint),
                                  c_void_p]),
}
# include/region_layer.h (ABI-compatible firmware API)
_REGION_ABI = ["region_layer_init", "region_layer_deinit", "region_layer_run", "region_layer_draw_boxes"]


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing — build the CUDA extension first (python -c 'import __graft_entry__ as g; "
            f"g.build()').  k210_yolo_framework_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    for name in _REGION_ABI:
        getattr(lib, name)
    return lib


lib = _load()


def last_error() -> str:
    return lib.k2y_last_error().decode("utf-8", "replace")


def check(rc: int) -> None:
    if rc != K2Y_OK:
        raise K2YError(f"[{rc}] {last_error()}")


def cuda_available() -> bool:
    return bool(lib.k2y_cuda_available())


def require_cuda() -> None:
    if not cuda_available():
        raise K2YError("no usable CUDA device: k210_yolo_framework_b200 runs on H100 (sm_90a) only, no CPU fallback")
