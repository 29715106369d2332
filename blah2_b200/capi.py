"""ctypes binding of the C ABI in include/b200dd.h (blah2_b200/lib/libb200dd.so).

This is the host-side mirror used by tests, bench.py and the Python operator classes in
blah2_b200/process.py.  It never computes anything itself and has NO CPU fallback: if
the native library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libb200dd.so")

OK = 0
ERR_ARG = 1
ERR_GEOMETRY = 2
ERR_CUDA = 3
ERR_CAPACITY = 4
ERR_NONFINITE = 5
FILTER_FAILED = 10
# b200dd_pipeline_stamp's boundaries
STAMP_CHAIN = 0
STAMP_SPECTRUM = 1
STAMP_CLUTTER = 2

DET_CFAR = 1
DET_CENTROID = 2
DET_INTERPOLATE = 3


class B200ddError(RuntimeError):
    def __init__(self, code, text):
        super().__init__(f"b200dd error {code}: {text}")
        self.code = code


class CafParams(C.Structure):
    _fields_ = [("delay_min", C.c_int32), ("delay_max", C.c_int32), ("doppler_min", C.c_int32),
                ("doppler_max", C.c_int32), ("fs", C.c_uint32), ("n_samples", C.c_uint32),
                ("round_hamming", C.c_int32), ("device", C.c_int32)]


class CafGeometry(C.Structure):
    _fields_ = [("n_delay_bins", C.c_uint32), ("n_doppler_bins", C.c_uint32), ("n_corr", C.c_uint32),
                ("nfft", C.c_uint32), ("n_used", C.c_uint32), ("cpi", C.c_double), ("doppler_middle", C.c_double),
                ("range_fft_len", C.c_uint32), ("range_segments", C.c_uint32), ("range_hop", C.c_uint32),
                ("doppler_fft_len", C.c_uint32), ("range_parts", C.c_uint32), ("range_groups", C.c_uint32)]


class DetParams(C.Structure):
    _fields_ = [("pfa", C.c_double), ("n_guard", C.c_int32), ("n_train", C.c_int32), ("min_delay", C.c_int32),
                ("min_doppler", C.c_double), ("n_centroid_delay", C.c_uint32), ("n_centroid_doppler", C.c_uint32),
                ("resolution_doppler", C.c_double), ("interp_delay", C.c_int32), ("interp_doppler", C.c_int32),
                ("device", C.c_int32)]


class PipelineParams(C.Structure):
    _fields_ = [("caf", CafParams), ("clutter_enable", C.c_int32), ("clutter_delay_min", C.c_int32),
                ("clutter_delay_max", C.c_int32), ("detection_enable", C.c_int32), ("det", DetParams)]


class SpectrumGeometry(C.Structure):
    _fields_ = [("decimation", C.c_uint32), ("n_spectrum", C.c_uint32), ("nfft", C.c_uint32),
                ("n_frequency", C.c_uint32), ("fold_chunks", C.c_uint32), ("fold_rows_per_chunk", C.c_uint32)]


class WhPlan(C.Structure):
    _fields_ = [("corr_fft_len", C.c_uint32), ("corr_hop", C.c_uint32), ("corr_segments", C.c_uint32),
                ("corr_ctas", C.c_uint32), ("filter_fft_len", C.c_uint32), ("filter_hop", C.c_uint32),
                ("filter_blocks", C.c_uint32), ("corr_lag_blocks", C.c_uint32), ("filter_partitions", C.c_uint32),
                ("filter_partition_taps", C.c_uint32), ("solve_threads", C.c_uint32),
                ("solve_rows_per_thread", C.c_uint32)]


class TrackerParams(C.Structure):
    _fields_ = [("m", C.c_uint32), ("n", C.c_uint32), ("n_delete", C.c_uint32), ("cpi", C.c_double),
                ("max_acc_init", C.c_double), ("fs", C.c_uint32), ("fc", C.c_uint32)]


class CpiResult(C.Structure):
    _fields_ = [("filter_status", C.c_int32), ("n_detections", C.c_uint32), ("noise_power", C.c_double),
                ("max_power", C.c_double)]


# every symbol include/b200dd.h declares: (name, restype, argtypes)
_VP = C.c_void_p
SIGNATURES = [
    ("b200dd_last_error", C.c_char_p, []),
    ("b200dd_device_count", C.c_int, []),
    ("b200dd_device_name", C.c_int, [C.c_int, C.c_char_p, C.c_int]),
    ("b200dd_next_hamming", C.c_uint32, [C.c_uint32]),
    ("b200dd_caf_create", C.c_int, [C.POINTER(CafParams), C.POINTER(_VP)]),
    ("b200dd_caf_plan", C.c_int, [C.POINTER(CafParams), C.POINTER(CafGeometry), _VP, C.c_uint32, _VP, C.c_uint32]),
    ("b200dd_caf_destroy", None, [_VP]),
    ("b200dd_caf_get_geometry", C.c_int, [_VP, C.POINTER(CafGeometry)]),
    ("b200dd_caf_get_axes", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_caf_process_host", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_caf_process_device", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_caf_range_device", C.c_int, [_VP, _VP, _VP, C.c_uint32, C.c_uint32, _VP, _VP]),
    ("b200dd_caf_doppler_device", C.c_int, [_VP, _VP, C.c_uint32, C.c_uint32, _VP, _VP]),
    ("b200dd_caf_place_tile_device", C.c_int, [_VP, _VP, C.c_uint32, C.c_uint32, _VP, _VP]),
    ("b200dd_caf_place_tiles_device", C.c_int, [_VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_caf_profile_device", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP, _VP, C.POINTER(C.c_float),
                                            C.POINTER(C.c_float)]),
    ("b200dd_caf_debug_range_matrix", C.c_int, [_VP, _VP]),
    ("b200dd_caf_device_map", _VP, [_VP]),
    ("b200dd_caf_stream", _VP, [_VP]),
    ("b200dd_wh_create", C.c_int, [C.c_int32, C.c_int32, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_wh_destroy", None, [_VP]),
    ("b200dd_wh_process_host", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_wh_process_device", C.c_int, [_VP, _VP, _VP, _VP, _VP]),
    ("b200dd_wh_last_status", C.c_int, [_VP]),
    ("b200dd_wh_process_device_f64", C.c_int, [_VP, _VP, _VP, _VP, _VP]),
    ("b200dd_wh_device_status", _VP, [_VP]),
    ("b200dd_wh_profile_device", C.c_int, [_VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                           C.POINTER(C.c_float)]),
    ("b200dd_wh_debug_weights", C.c_int, [_VP, _VP, _VP, _VP]),
    ("b200dd_wh_n_bins", C.c_uint32, [_VP]),
    ("b200dd_wh_get_plan", C.c_int, [_VP, C.POINTER(WhPlan)]),
    ("b200dd_wh_create_chunk", C.c_int, [C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_wh_chunk_halos", C.c_int, [_VP, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("b200dd_wh_chunk_corr_device", C.c_int, [_VP, _VP, _VP, _VP, _VP]),
    ("b200dd_wh_chunk_filter_device", C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    ("b200dd_wh_stream", _VP, [_VP]),
    ("b200dd_det_create", C.c_int, [C.POINTER(DetParams), C.c_uint32, C.c_uint32, C.POINTER(_VP)]),
    ("b200dd_det_destroy", None, [_VP]),
    ("b200dd_det_set_metrics_device", C.c_int, [_VP, _VP, C.c_uint32, C.c_uint32, _VP, _VP]),
    ("b200dd_det_process_device", C.c_int, [_VP, C.c_int, _VP, C.c_uint32, C.c_uint32, _VP, _VP, C.c_double, _VP,
                                            _VP, _VP, C.c_uint32, C.POINTER(C.c_uint32), _VP]),
    ("b200dd_det_chain_device_async", C.c_int, [_VP, C.c_int, _VP, C.c_uint32, C.c_uint32, _VP, _VP, _VP]),
    ("b200dd_det_chain_fetch", C.c_int, [_VP, _VP, _VP, _VP, _VP, C.c_uint32, C.POINTER(C.c_uint32), _VP]),
    ("b200dd_det_process_host", C.c_int, [_VP, C.c_int, _VP, C.c_uint32, C.c_uint32, _VP, _VP, C.c_double, _VP, _VP,
                                          _VP, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("b200dd_det_centroid_host", C.c_int, [_VP, _VP, _VP, _VP, C.c_uint32, _VP, _VP, _VP, C.c_uint32,
                                           C.POINTER(C.c_uint32)]),
    ("b200dd_det_interpolate_host", C.c_int, [_VP, _VP, _VP, _VP, C.c_uint32, _VP, C.c_uint32, C.c_uint32, _VP, _VP,
                                              C.c_double, _VP, _VP, _VP, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("b200dd_spectrum_create", C.c_int, [C.c_uint32, C.c_double, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_spectrum_plan", C.c_int, [C.c_uint32, C.c_double, C.POINTER(SpectrumGeometry), _VP, C.c_uint32]),
    ("b200dd_spectrum_destroy", None, [_VP]),
    ("b200dd_spectrum_get_geometry", C.c_int, [_VP, C.POINTER(SpectrumGeometry)]),
    ("b200dd_spectrum_get_frequency", C.c_int, [_VP, _VP, C.c_uint32]),
    ("b200dd_spectrum_process_host", C.c_int, [_VP, _VP, C.c_uint32, _VP]),
    ("b200dd_spectrum_process_device", C.c_int, [_VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_spectrum_process_device_f64", C.c_int, [_VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_spectrum_fold_slice_device", C.c_int, [_VP, _VP, C.c_uint32, C.c_uint32, _VP, _VP]),
    ("b200dd_spectrum_finish_device", C.c_int, [_VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_spectrum_fetch", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_spectrum_profile_device", C.c_int, [_VP, _VP, C.c_uint32, _VP, C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float)]),
    ("b200dd_spectrum_stream", _VP, [_VP]),
    ("b200dd_pipeline_create", C.c_int, [C.POINTER(PipelineParams), C.POINTER(_VP)]),
    ("b200dd_pipeline_destroy", None, [_VP]),
    ("b200dd_pipeline_get_geometry", C.c_int, [_VP, C.POINTER(CafGeometry)]),
    ("b200dd_pipeline_get_axes", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_pipeline_process_host", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP, C.POINTER(CpiResult), _VP, _VP, _VP,
                                               C.c_uint32]),
    ("b200dd_pipeline_submit_host", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_submit_host_rspduo", C.c_int, [_VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_submit_host_ci8", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_submit_host_cf32", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_submit_device", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_pipeline_prepare_device", C.c_int, [_VP, _VP, _VP, C.c_uint32, _VP, _VP]),
    ("b200dd_pipeline_fetch", C.c_int, [_VP, C.POINTER(CpiResult), _VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_stream", _VP, [_VP]),
    ("b200dd_pipeline_enable_spectrum", C.c_int, [_VP, C.c_double, C.POINTER(C.c_uint32)]),
    ("b200dd_pipeline_fetch_spectrum", C.c_int, [_VP, _VP, C.c_uint32]),
    ("b200dd_pipeline_enable_map_json", C.c_int, [_VP, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_map_json", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_enable_maxhold", C.c_int, [_VP, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_maxhold", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_enable_detection_json", C.c_int, [_VP, C.c_uint32, C.POINTER(C.c_size_t),
                                                        C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_detection_json", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_detection_stash", C.c_int, [_VP, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_enable_tracker", C.c_int, [_VP, C.POINTER(TrackerParams), C.c_uint32, C.c_uint32,
                                                 C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_track_json", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_enable_iqdata_json", C.c_int, [_VP, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_size_t),
                                                     C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_iqdata_json", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_iqdata_stash", C.c_int, [_VP, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_enable_timing_json", C.c_int, [_VP, C.c_uint64, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_timing_json", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_fetch_timing_stash", C.c_int, [_VP, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_debug_timing_values", C.c_int, [_VP, C.POINTER(C.c_char_p), _VP, C.c_uint32,
                                                      C.POINTER(C.c_uint32)]),
    ("b200dd_timing_render_host", C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_char_p), _VP,
                                            C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_timing_max_bytes", C.c_size_t, []),
    ("b200dd_pipeline_share_history", C.c_int, [_VP, C.c_uint32]),
    ("b200dd_pipeline_enable_export", C.c_int, [_VP, C.c_uint32, C.POINTER(C.c_size_t)]),
    ("b200dd_pipeline_export_record", C.c_int, [_VP, C.POINTER(_VP)]),
    ("b200dd_pipeline_submit_record", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_pipeline_submit_map", C.c_int, [_VP, _VP, _VP, _VP, C.c_uint32, _VP]),
    ("b200dd_pipeline_stamp", C.c_int, [_VP, C.c_int, _VP]),
    ("b200dd_mapjson_create", C.c_int, [C.c_uint32, C.c_uint32, _VP, _VP, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_mapjson_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_mapjson_destroy", None, [_VP]),
    ("b200dd_mapjson_render_device", C.c_int, [_VP, _VP, C.c_int, C.c_double, C.c_double, _VP]),
    ("b200dd_mapjson_fetch", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_mapjson_render_host", C.c_int, [_VP, _VP, C.c_double, C.c_double, C.c_uint64, _VP, C.c_size_t,
                                             C.POINTER(C.c_size_t)]),
    ("b200dd_mapjson_format_doubles_host", C.c_int, [_VP, C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_mapjson_format_doubles_device", C.c_int, [_VP, C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t),
                                                       C.c_int32]),
    ("b200dd_mapjson_debug_cell_values", C.c_int, [_VP, _VP, C.c_int, C.c_double, _VP, _VP]),
    ("b200dd_maxhold_create", C.c_int, [C.c_uint32, C.c_uint32, _VP, _VP, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_maxhold_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_maxhold_destroy", None, [_VP]),
    ("b200dd_maxhold_push_device", C.c_int, [_VP, _VP, C.c_int, C.c_double, C.c_double, _VP]),
    ("b200dd_maxhold_fetch", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_maxhold_format_doubles_host", C.c_int, [_VP, C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_maxhold_format_doubles_device", C.c_int, [_VP, C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t),
                                                       C.c_int32]),
    ("b200dd_detjson_create", C.c_int, [C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_detjson_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_detjson_stash_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_detjson_destroy", None, [_VP]),
    ("b200dd_detjson_render_device", C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    ("b200dd_detjson_fetch", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_detjson_fetch_stash", C.c_int, [_VP, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_detjson_render_host", C.c_int, [_VP, _VP, _VP, C.c_uint32, C.c_uint64, C.c_uint32, _VP, C.c_size_t,
                                             C.POINTER(C.c_size_t)]),
    ("b200dd_iqjson_create", C.c_int, [C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_iqjson_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_iqjson_stash_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_iqjson_destroy", None, [_VP]),
    ("b200dd_iqjson_render_device", C.c_int, [_VP, _VP, _VP]),
    ("b200dd_iqjson_fetch", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_iqjson_fetch_stash", C.c_int, [_VP, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_iqjson_render_host", C.c_int, [_VP, C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_uint64, _VP,
                                            C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_iqjson_debug_bin_values", C.c_int, [_VP, _VP, _VP, _VP]),
    ("b200dd_tracker_plan", C.c_int, [C.POINTER(TrackerParams), C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32),
                                      C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    ("b200dd_tracker_create", C.c_int, [C.POINTER(TrackerParams), C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_tracker_destroy", None, [_VP]),
    ("b200dd_tracker_reset", C.c_int, [_VP]),
    ("b200dd_tracker_max_bytes", C.c_size_t, [_VP]),
    ("b200dd_tracker_reserve", C.c_int, [_VP, C.c_uint32, C.c_uint32, _VP]),
    ("b200dd_tracker_usage", C.c_int, [_VP, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), _VP]),
    ("b200dd_tracker_process_device", C.c_int, [_VP, _VP, _VP, _VP, _VP, C.c_uint64, _VP]),
    ("b200dd_tracker_process_host", C.c_int, [_VP, _VP, _VP, _VP, C.c_uint32, C.c_uint64, _VP]),
    ("b200dd_tracker_fetch", C.c_int, [_VP, C.c_uint64, _VP, C.c_size_t, C.POINTER(C.c_size_t), _VP]),
    ("b200dd_tracker_format_doubles_host", C.c_int, [_VP, C.c_uint32, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("b200dd_comm_get_unique_id", C.c_int, [_VP]),
    ("b200dd_comm_create", C.c_int, [C.c_int32, C.c_int32, _VP, C.c_int32, C.POINTER(_VP)]),
    ("b200dd_comm_destroy", None, [_VP]),
    ("b200dd_comm_rank", C.c_int32, [_VP]),
    ("b200dd_comm_world", C.c_int32, [_VP]),
    ("b200dd_comm_stream", _VP, [_VP]),
    ("b200dd_comm_gather_async", C.c_int, [_VP, _VP, _VP, C.c_size_t, C.c_int32, _VP]),
    ("b200dd_comm_gatherv_async", C.c_int, [_VP, _VP, C.c_size_t, _VP, _VP, _VP, C.c_int32, _VP]),
    ("b200dd_comm_allgatherv_async", C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    ("b200dd_comm_allreduce_f64_async", C.c_int, [_VP, _VP, C.c_size_t, _VP]),
    ("b200dd_comm_sendrecv_async", C.c_int, [_VP, _VP, C.c_size_t, C.c_int32, _VP, C.c_size_t, C.c_int32, _VP]),
    ("b200dd_comm_wait_stream", C.c_int, [_VP, _VP]),
    ("b200dd_comm_join", C.c_int, [_VP, _VP]),
    ("b200dd_comm_sync", C.c_int, [_VP]),
    ("b200dd_ubench_fp64_tflops", C.c_int, [C.c_int32, C.POINTER(C.c_double)]),
    ("b200dd_bind_host_to_device", C.c_int, [C.c_int32, C.c_char_p, C.c_int32]),
    ("b200dd_host_alloc", _VP, [C.c_size_t]),
    ("b200dd_host_free", None, [_VP]),
]

_lib = None


def load():
    """Load libb200dd.so (building nothing).  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(f"{LIB_PATH} not found: run `python -m blah2_b200.build` (needs nvcc)")
    lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
    for name, res, args in SIGNATURES:
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().b200dd_last_error().decode("utf-8", "replace")


def check(rc: int, allow=()):
    if rc != OK and rc not in allow:
        raise B200ddError(rc, last_error())
    return rc


def ptr(a):
    """Raw pointer of a numpy array / torch tensor / int."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


def caf_plan(delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming=False, device=-1):
    """Host-only: (CafGeometry, delay axis, doppler axis) as b200dd_caf_create would set them up."""
    lib = load()
    p = CafParams(int(delayMin), int(delayMax), int(dopplerMin), int(dopplerMax), int(fs), int(n),
                  int(bool(roundHamming)), int(device))
    g = CafGeometry()
    check(lib.b200dd_caf_plan(C.byref(p), C.byref(g), None, 0, None, 0))
    delay = np.empty(g.n_delay_bins, dtype=np.int32)
    doppler = np.empty(g.n_doppler_bins, dtype=np.float64)
    check(lib.b200dd_caf_plan(C.byref(p), C.byref(g), ptr(delay), delay.shape[0], ptr(doppler), doppler.shape[0]))
    return g, delay, doppler


def spectrum_plan(n, bandwidth):
    """Host-only: (SpectrumGeometry, frequency vector) as b200dd_spectrum_create would set them up."""
    lib = load()
    g = SpectrumGeometry()
    check(lib.b200dd_spectrum_plan(int(n), float(bandwidth), C.byref(g), None, 0))
    f = np.empty(g.n_frequency, dtype=np.float64)
    check(lib.b200dd_spectrum_plan(int(n), float(bandwidth), C.byref(g), ptr(f), f.shape[0]))
    return g, f


def format_doubles(values, device=None) -> list:
    """The text a map client receives for each double (written at two decimals, read back, written again), as
    the formatter computes it on the host (device=None) or in a kernel on `device`; "" where a value has none."""
    lib = load()
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    n = C.c_size_t()
    out = np.empty(v.size * 25 + 1, dtype=np.uint8)
    if device is None:
        check(lib.b200dd_mapjson_format_doubles_host(ptr(v), v.size, ptr(out), out.size, C.byref(n)))
    else:
        check(lib.b200dd_mapjson_format_doubles_device(ptr(v), v.size, ptr(out), out.size, C.byref(n), int(device)))
    return out[:n.value].tobytes().decode("ascii").split(",") if v.size else []


def format_maxhold_doubles(values, device=None) -> list:
    """The /stash/map text of a max-hold cell whose only held value is each double (its map-document text parsed
    and re-printed by Number::toString), on the host (device=None) or in a kernel on `device`; "" where a value has
    no map-document text or its hundredths lie outside int32."""
    lib = load()
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    n = C.c_size_t()
    out = np.empty(v.size * 13 + 1, dtype=np.uint8)
    if device is None:
        check(lib.b200dd_maxhold_format_doubles_host(ptr(v), v.size, ptr(out), out.size, C.byref(n)))
    else:
        check(lib.b200dd_maxhold_format_doubles_device(ptr(v), v.size, ptr(out), out.size, C.byref(n), int(device)))
    return out[:n.value].tobytes().decode("ascii").split(",") if v.size else []


def tracker_plan(m, n, nDelete, cpi, maxAcc, fs, fc, max_tracks=1 << 16, max_history=64):
    """Host-only: (hypotheses per unassociated detection, document size bound, device bytes of the track state)."""
    lib = load()
    p = TrackerParams(int(m), int(n), int(nDelete), float(cpi), float(maxAcc), int(fs), int(fc))
    nh, mb, db = C.c_uint32(), C.c_size_t(), C.c_size_t()
    check(lib.b200dd_tracker_plan(C.byref(p), int(max_tracks), int(max_history), C.byref(nh), C.byref(mb),
                                  C.byref(db)))
    return int(nh.value), int(mb.value), int(db.value)


def format_track_doubles(values) -> list:
    """The text the track document gives each double (Writer::Double at two decimal places, written once), on the
    host; "" for a non-finite value."""
    lib = load()
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    n = C.c_size_t()
    out = np.empty(v.size * 25 + 1, dtype=np.uint8)
    check(lib.b200dd_tracker_format_doubles_host(ptr(v), v.size, ptr(out), out.size, C.byref(n)))
    return out[:n.value].tobytes().decode("ascii").split(",") if v.size else []


def device_count() -> int:
    return int(load().b200dd_device_count())


def next_hamming(v: int) -> int:
    return int(load().b200dd_next_hamming(int(v)))
