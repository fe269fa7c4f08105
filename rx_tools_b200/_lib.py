"""ctypes loader for librxb200.so (include/rxb200.h).  No fallback: a missing library or a missing
CUDA device raises — the product path never routes through a CPU implementation."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RXB200_LIB", os.path.join(HERE, "librxb200.so"))   # override: A/B builds of the same ABI

OK, EINVAL, ENODEV, ECUDA, ENOMEM, EUNSUPPORTED, ECAPACITY = 0, -1, -2, -3, -4, -5, -6
ERR_NAMES = {EINVAL: "EINVAL", ENODEV: "ENODEV", ECUDA: "ECUDA", ENOMEM: "ENOMEM",
             EUNSUPPORTED: "EUNSUPPORTED", ECAPACITY: "ECAPACITY"}


# the capture handles' input formats (rxb200_*_mix_set_input_format): bytes per complex element of each
IN_CS16, IN_CS8, IN_CU8, IN_CS12 = 0, 1, 2, 3
IN_FORMATS = {"CS16": IN_CS16, "CS8": IN_CS8, "CU8": IN_CU8, "CS12": IN_CS12}
IN_ELEM_BYTES = {IN_CS16: 4, IN_CS8: 2, IN_CU8: 2, IN_CS12: 3}


def in_array(x, fmt: int):
    """A capture call's host buffer in input format fmt as one C array, and its n_int16 (two per complex element):
    int16 for CS16, else the format's raw bytes (uint8)."""
    if fmt == IN_CS16:
        a = np.ascontiguousarray(x, dtype=np.int16).reshape(-1)
        return a, a.size
    a = np.ascontiguousarray(x, dtype=np.uint8).reshape(-1)
    e = IN_ELEM_BYTES[fmt]
    if a.size % e:
        raise ValueError(f"{a.size} bytes are not whole {e}-byte elements")
    return a, 2 * (a.size // e)


class Rxb200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rxb200 {ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


class FmParamsC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "mode", "downsample", "downsample_passes", "comp_fir_size", "custom_atan", "output_scale",
        "post_downsample", "deemph", "deemph_a", "rate_out", "rate_out2", "squelch_level",
        "dc_block_audio", "adc_block_const", "dc_block_raw", "rdc_block_const", "offset_tuning", "report_levels")]


class FmCliC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "mode", "wbfm", "rate_s", "rate_r", "use_F", "comp_fir_size", "custom_atan", "post_downsample",
        "deemph", "time_constant_us", "offset_tuning", "squelch_level", "dc_block_audio", "dc_block_raw",
        "rdc_block_const")]


class FmDerivedC(C.Structure):
    _fields_ = [("params", FmParamsC), ("capture_rate", C.c_int), ("capture_freq_offset", C.c_int),
                ("output_rate", C.c_int)]


class FmStatsC(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("launches", "segments", "fixup_segments", "segment_len", "warmup_len", "kernel_kind")]


class PowerParamsC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "n_hops", "bin_e", "buf_len", "downsample", "downsample_passes", "comp_fir_size", "boxcar", "peak_hold")]


class PowerPathC(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("kernel", "bin_e", "threads", "nb", "tables_in_smem", "slices", "launches")]


POWER_PATHS = {0: "none", 1: "rms", 2: "fft8", 3: "generic", 4: "big_load", 5: "big_decim"}


class DdcC(C.Structure):
    _fields_ = [("decim", C.c_int), ("n_taps", C.c_int), ("taps", C.POINTER(C.c_int32)), ("shift", C.c_int)]


class FmCapturePlanC(C.Structure):
    _fields_ = [("centre_hz", C.c_int64), ("decim", C.c_int), ("capture_rate", C.c_int), ("n_taps", C.c_int)]


class FmTwoStagePlanC(C.Structure):
    _fields_ = [("centre_hz", C.c_int64), ("capture_rate", C.c_int), ("n_bins", C.c_int), ("coarse_decim", C.c_int),
                ("coarse_taps", C.c_int), ("coarse_shift", C.c_int), ("fine_decim", C.c_int), ("fine_taps", C.c_int),
                ("fine_shift", C.c_int)]


class FmRasterPlanC(C.Structure):
    _fields_ = [("centre_hz", C.c_int64), ("capture_rate", C.c_int), ("n_bins", C.c_int), ("decim", C.c_int),
                ("n_taps", C.c_int), ("shift", C.c_int)]


class ResamplerC(C.Structure):
    _fields_ = [("up", C.c_int), ("down", C.c_int), ("taps_per_phase", C.c_int), ("taps", C.POINTER(C.c_int32)),
                ("shift", C.c_int)]


class PowerPlanC(C.Structure):
    _fields_ = [("params", PowerParamsC), ("rate", C.c_int), ("crop", C.c_double),
                ("first_freq", C.c_int64), ("freq_step", C.c_int64), ("bin_size_hz", C.c_double)]


class PowerTilingC(C.Structure):
    _fields_ = [("n_tiles", C.c_int), ("hops_per_tile", C.c_int), ("decim", C.c_int), ("n_taps", C.c_int),
                ("capture_rate", C.c_int)]


# every symbol include/rxb200.h declares (tests/test_abi.py checks the header against this list)
SYMBOLS = [
    "rxb200_last_error", "rxb200_abi_version", "rxb200_device_count",
    "rxb200_fm_derive", "rxb200_fm_create", "rxb200_fm_destroy", "rxb200_fm_reset", "rxb200_fm_max_output",
    "rxb200_fm_process", "rxb200_fm_process_device", "rxb200_fm_process_read", "rxb200_fm_process_read_device",
    "rxb200_fm_squelch_hits", "rxb200_fm_levels", "rxb200_fm_stream",
    "rxb200_fm_last_stats", "rxb200_fm_tune", "rxb200_fm_kernel_ms", "rxb200_fm_disc_device",
    "rxb200_power_plan_range", "rxb200_window_table", "rxb200_sine_table", "rxb200_power_create",
    "rxb200_power_destroy", "rxb200_power_accumulate", "rxb200_power_accumulate_device", "rxb200_power_read",
    "rxb200_power_device_avg", "rxb200_power_reset", "rxb200_power_stream", "rxb200_power_last_launches",
    "rxb200_power_format_row", "rxb200_power_kernel_ms", "rxb200_power_row_len", "rxb200_power_read_db",
    "rxb200_power_format_db_row", "rxb200_power_last_path",
    "rxb200_comm_unique_id", "rxb200_comm_create", "rxb200_comm_create_all", "rxb200_comm_destroy", "rxb200_comm_size",
    "rxb200_comm_rank", "rxb200_power_shard", "rxb200_power_gather",
    "rxb200_power_group_create", "rxb200_power_group_destroy", "rxb200_power_group_size", "rxb200_power_group_member",
    "rxb200_power_group_accumulate", "rxb200_power_group_gather", "rxb200_power_group_reset",
    "rxb200_fm_group_create", "rxb200_fm_group_destroy", "rxb200_fm_group_size", "rxb200_fm_group_member",
    "rxb200_fm_group_process", "rxb200_fm_group_process_read", "rxb200_fm_group_squelch_hits", "rxb200_fm_group_levels",
    "rxb200_fm_group_reset",
    "rxb200_fm_mix_table", "rxb200_mix_device", "rxb200_fm_mix_create", "rxb200_fm_mix_destroy", "rxb200_fm_mix_reset",
    "rxb200_fm_mix_member", "rxb200_fm_mix_process", "rxb200_fm_mix_process_device", "rxb200_fm_mix_process_read",
    "rxb200_fm_mix_process_read_device", "rxb200_fm_mix_squelch_hits", "rxb200_fm_mix_levels", "rxb200_fm_mix_kernel_ms",
    "rxb200_fm_mix_group_create", "rxb200_fm_mix_group_destroy", "rxb200_fm_mix_group_size",
    "rxb200_fm_mix_group_member", "rxb200_fm_mix_group_process", "rxb200_fm_mix_group_process_read",
    "rxb200_fm_mix_group_squelch_hits", "rxb200_fm_mix_group_levels", "rxb200_fm_mix_group_reset",
    "rxb200_fm_mix_create_ddc", "rxb200_fm_mix_decimated_len", "rxb200_fm_mix_max_output", "rxb200_ddc_device",
    "rxb200_fm_mix_group_create_ddc", "rxb200_fm_mix_create_raster", "rxb200_raster_device",
    "rxb200_fm_plan_capture", "rxb200_fm_mix_create_two_stage", "rxb200_two_stage_word", "rxb200_two_stage_device",
    "rxb200_fm_plan_capture_two_stage", "rxb200_fm_plan_capture_raster",
    "rxb200_power_mix_create", "rxb200_power_mix_destroy", "rxb200_power_mix_member", "rxb200_power_mix_reset",
    "rxb200_power_mix_accumulate", "rxb200_power_mix_accumulate_device", "rxb200_power_mix_kernel_ms",
    "rxb200_nco_table", "rxb200_power_ddc_device", "rxb200_ddc_lowpass",
    "rxb200_power_plan_tiles", "rxb200_power_tile", "rxb200_power_mix_lead", "rxb200_power_mix_accumulate_burst",
    "rxb200_power_mix_accumulate_burst_device",
    "rxb200_sdr_convert", "rxb200_sdr_convert_device",
    "rxb200_sdr_mix_create", "rxb200_sdr_mix_create_two_stage", "rxb200_sdr_mix_create_raster",
    "rxb200_sdr_mix_destroy", "rxb200_sdr_mix_reset",
    "rxb200_sdr_mix_decimated_len", "rxb200_sdr_mix_process", "rxb200_sdr_mix_process_device",
    "rxb200_sdr_mix_kernel_ms", "rxb200_sdr_mix_stream", "rxb200_sdr_plan_capture",
    "rxb200_resample_lowpass", "rxb200_plan_resample", "rxb200_resample_create", "rxb200_resample_destroy",
    "rxb200_resample_reset", "rxb200_resample_out_len", "rxb200_resample_process", "rxb200_resample_process_device",
    "rxb200_resample_stream", "rxb200_resample_kernel_ms", "rxb200_resample_device",
    "rxb200_resample_in_len", "rxb200_fm_plan_capture_at", "rxb200_fm_plan_capture_two_stage_at",
    "rxb200_fm_plan_capture_raster_at", "rxb200_sdr_plan_capture_at",
    "rxb200_fm_mix_set_device_rate", "rxb200_sdr_mix_set_device_rate", "rxb200_power_mix_set_device_rate",
    "rxb200_power_plan_capture", "rxb200_power_plan_capture_at", "rxb200_power_plan_tiles_at",
    "rxb200_power_mix_set_burst_device_rate", "rxb200_power_mix_burst_in_len",
    "rxb200_fm_mix_set_input_format", "rxb200_sdr_mix_set_input_format", "rxb200_power_mix_set_input_format",
]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(librxb200 has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    p16, pint, pi64, sz = C.POINTER(C.c_int16), C.POINTER(C.c_int), C.POINTER(C.c_int64), C.c_size_t
    L.rxb200_last_error.restype = C.c_char_p
    L.rxb200_fm_derive.argtypes = [C.POINTER(FmCliC), C.POINTER(FmDerivedC)]
    L.rxb200_fm_create.argtypes = [C.POINTER(FmParamsC), C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_fm_destroy.argtypes = [C.c_void_p]
    L.rxb200_fm_destroy.restype = None
    L.rxb200_fm_reset.argtypes = [C.c_void_p]
    L.rxb200_fm_max_output.restype = sz
    L.rxb200_fm_max_output.argtypes = [C.c_void_p, sz, sz]
    L.rxb200_fm_process.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), pint]
    L.rxb200_fm_process_device.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), C.c_int]
    L.rxb200_fm_process_read.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_fm_process_read_device.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz), C.c_int]
    L.rxb200_fm_squelch_hits.argtypes = [C.c_void_p, pint]
    L.rxb200_fm_levels.argtypes = [C.c_void_p, pint, C.c_size_t, C.POINTER(C.c_size_t)]
    L.rxb200_fm_stream.restype = C.c_void_p
    L.rxb200_fm_stream.argtypes = [C.c_void_p]
    L.rxb200_fm_last_stats.argtypes = [C.c_void_p, C.POINTER(FmStatsC)]
    L.rxb200_fm_tune.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.rxb200_fm_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_fm_disc_device.argtypes = [C.c_int, C.c_void_p, sz, C.c_void_p, C.c_void_p]
    L.rxb200_power_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_power_plan_range.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(PowerPlanC)]
    L.rxb200_window_table.argtypes = [C.c_int, C.c_int, pint]
    L.rxb200_sine_table.argtypes = [C.c_int, p16]
    L.rxb200_power_create.argtypes = [C.POINTER(PowerParamsC), pint, p16, C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_power_destroy.argtypes = [C.c_void_p]
    L.rxb200_power_destroy.restype = None
    L.rxb200_power_accumulate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.rxb200_power_accumulate_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.rxb200_power_read.argtypes = [C.c_void_p, pi64, pint]
    L.rxb200_power_device_avg.restype = C.c_void_p
    L.rxb200_power_device_avg.argtypes = [C.c_void_p]
    L.rxb200_power_reset.argtypes = [C.c_void_p]
    L.rxb200_power_stream.restype = C.c_void_p
    L.rxb200_power_stream.argtypes = [C.c_void_p]
    L.rxb200_power_last_launches.argtypes = [C.c_void_p]
    L.rxb200_power_last_path.argtypes = [C.c_void_p, C.POINTER(PowerPathC)]
    L.rxb200_power_format_row.argtypes = [pi64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_double, C.c_int,
                                          C.c_char_p, sz]
    L.rxb200_power_row_len.argtypes = [C.c_int, C.c_double]
    L.rxb200_power_read_db.argtypes = [C.c_void_p, C.c_int, C.c_double, C.POINTER(C.c_double), sz, pint]
    L.rxb200_power_format_db_row.argtypes = [C.POINTER(C.c_double), C.c_int, C.c_int64, C.c_int, C.c_int, C.c_double,
                                             C.c_int, C.c_char_p, sz]
    L.rxb200_comm_unique_id.argtypes = [C.c_void_p]
    L.rxb200_comm_create.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_comm_create_all.argtypes = [C.c_int, pint, C.POINTER(C.c_void_p)]
    L.rxb200_comm_destroy.argtypes = [C.c_void_p]
    L.rxb200_comm_destroy.restype = None
    L.rxb200_comm_size.argtypes = [C.c_void_p]
    L.rxb200_comm_rank.argtypes = [C.c_void_p]
    L.rxb200_power_shard.argtypes = [C.c_int, C.c_int, C.c_int, pint, pint]
    L.rxb200_power_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.rxb200_power_group_create.argtypes = [C.POINTER(PowerParamsC), pint, p16, C.c_int, pint, C.POINTER(C.c_void_p)]
    L.rxb200_power_group_destroy.argtypes = [C.c_void_p]
    L.rxb200_power_group_destroy.restype = None
    L.rxb200_power_group_size.argtypes = [C.c_void_p]
    L.rxb200_power_group_member.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_power_group_member.restype = C.c_void_p
    L.rxb200_power_group_accumulate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.rxb200_power_group_gather.argtypes = [C.c_void_p]
    L.rxb200_power_group_reset.argtypes = [C.c_void_p]
    L.rxb200_fm_group_create.argtypes = [C.POINTER(FmParamsC), C.c_int, C.c_int, pint, C.POINTER(C.c_void_p)]
    L.rxb200_fm_group_destroy.argtypes = [C.c_void_p]
    L.rxb200_fm_group_destroy.restype = None
    L.rxb200_fm_group_size.argtypes = [C.c_void_p]
    L.rxb200_fm_group_member.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_fm_group_member.restype = C.c_void_p
    L.rxb200_fm_group_process.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), pint]
    L.rxb200_fm_group_process_read.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_fm_group_squelch_hits.argtypes = [C.c_void_p, pint]
    L.rxb200_fm_group_levels.argtypes = [C.c_void_p, pint, sz, C.POINTER(sz)]
    L.rxb200_fm_group_reset.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_table.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int32), sz, C.POINTER(sz)]
    L.rxb200_mix_device.argtypes = [C.c_int, C.c_int, C.c_longlong, C.c_void_p, sz, C.c_void_p, C.c_void_p]
    L.rxb200_fm_mix_create.argtypes = [C.POINTER(FmParamsC), C.c_int, pint, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_fm_mix_destroy.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_destroy.restype = None
    L.rxb200_fm_mix_reset.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_member.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_member.restype = C.c_void_p
    L.rxb200_fm_mix_process.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), pint]
    L.rxb200_fm_mix_process_device.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), C.c_int]
    L.rxb200_fm_mix_process_read.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_fm_mix_process_read_device.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz), C.c_int]
    L.rxb200_fm_mix_squelch_hits.argtypes = [C.c_void_p, pint]
    L.rxb200_fm_mix_levels.argtypes = [C.c_void_p, pint, sz, C.POINTER(sz)]
    L.rxb200_fm_mix_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_fm_mix_group_create.argtypes = [C.POINTER(FmParamsC), C.c_int, pint, C.c_int, C.c_int, pint,
                                             C.POINTER(C.c_void_p)]
    L.rxb200_fm_mix_group_destroy.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_group_destroy.restype = None
    L.rxb200_fm_mix_group_size.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_group_member.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_fm_mix_group_member.restype = C.c_void_p
    L.rxb200_fm_mix_group_process.argtypes = [C.c_void_p, C.c_void_p, sz, sz, C.c_void_p, sz, C.POINTER(sz), pint]
    L.rxb200_fm_mix_group_process_read.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_fm_mix_group_squelch_hits.argtypes = [C.c_void_p, pint]
    L.rxb200_fm_mix_group_levels.argtypes = [C.c_void_p, pint, sz, C.POINTER(sz)]
    L.rxb200_fm_mix_group_reset.argtypes = [C.c_void_p]
    L.rxb200_fm_mix_create_ddc.argtypes = [C.POINTER(FmParamsC), C.c_int, pint, C.c_int, C.POINTER(DdcC), C.c_int,
                                           C.POINTER(C.c_void_p)]
    L.rxb200_fm_mix_decimated_len.argtypes = [C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_fm_mix_max_output.argtypes = [C.c_void_p, sz, sz]
    L.rxb200_fm_mix_max_output.restype = sz
    L.rxb200_ddc_device.argtypes = [C.c_int, C.c_int, C.c_longlong, C.POINTER(DdcC), C.c_void_p, sz, C.c_void_p,
                                    C.c_void_p]
    L.rxb200_fm_mix_group_create_ddc.argtypes = [C.POINTER(FmParamsC), C.c_int, pint, C.c_int, C.POINTER(DdcC),
                                                 C.c_int, pint, C.POINTER(C.c_void_p)]
    L.rxb200_fm_mix_create_raster.argtypes = [C.POINTER(FmParamsC), C.c_int, pint, C.c_int, C.POINTER(DdcC), C.c_int,
                                              C.POINTER(C.c_void_p)]
    L.rxb200_raster_device.argtypes = [C.c_int, pint, C.c_int, C.c_ulonglong, C.POINTER(DdcC), C.c_void_p, sz,
                                       C.c_void_p, C.c_void_p]
    L.rxb200_fm_plan_capture.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.POINTER(FmCapturePlanC), pint]
    L.rxb200_fm_mix_create_two_stage.argtypes = [C.POINTER(FmParamsC), C.c_int, C.c_int, pint, C.c_int, C.POINTER(DdcC),
                                                 C.POINTER(DdcC), C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_two_stage_word.argtypes = [C.c_int, C.c_int, C.c_int, pint, C.c_int, pint, C.POINTER(C.c_uint32)]
    L.rxb200_two_stage_device.argtypes = [C.c_int, C.c_int, pint, C.c_int, C.c_ulonglong, C.POINTER(DdcC),
                                          C.POINTER(DdcC), C.c_void_p, sz, C.c_void_p, C.c_void_p]
    L.rxb200_fm_plan_capture_two_stage.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.POINTER(FmTwoStagePlanC),
                                                   pint]
    L.rxb200_fm_plan_capture_raster.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.POINTER(FmRasterPlanC), pint]
    L.rxb200_power_mix_create.argtypes = [C.POINTER(PowerParamsC), pint, p16, C.c_int, pint, C.POINTER(DdcC), C.c_int,
                                          C.POINTER(C.c_void_p)]
    L.rxb200_power_mix_destroy.argtypes = [C.c_void_p]
    L.rxb200_power_mix_destroy.restype = None
    L.rxb200_power_mix_member.argtypes = [C.c_void_p]
    L.rxb200_power_mix_member.restype = C.c_void_p
    L.rxb200_power_mix_reset.argtypes = [C.c_void_p]
    L.rxb200_power_mix_accumulate.argtypes = [C.c_void_p, C.c_void_p, sz]
    L.rxb200_power_mix_accumulate_device.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_int]
    L.rxb200_power_mix_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_nco_table.argtypes = [C.POINTER(C.c_int32)]
    L.rxb200_power_ddc_device.argtypes = [C.c_int, C.c_int, C.c_ulonglong, C.POINTER(DdcC), C.c_void_p, sz, C.c_void_p,
                                          C.c_void_p]
    L.rxb200_ddc_lowpass.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32)]
    L.rxb200_power_plan_tiles.argtypes = [C.POINTER(PowerPlanC), C.c_longlong, C.POINTER(PowerTilingC), pint]
    L.rxb200_power_tile.argtypes = [C.POINTER(PowerPlanC), C.POINTER(PowerTilingC), C.c_int, pint, pint,
                                    C.POINTER(C.c_int64)]
    L.rxb200_power_mix_lead.argtypes = [C.c_void_p]
    L.rxb200_power_mix_accumulate_burst.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, sz]
    L.rxb200_power_mix_accumulate_burst_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, sz, C.c_int]
    L.rxb200_sdr_convert.argtypes = [C.c_int, C.c_void_p, sz, C.c_void_p, C.c_int]
    L.rxb200_sdr_convert_device.argtypes = [C.c_int, C.c_void_p, sz, C.c_void_p, C.c_void_p]
    L.rxb200_sdr_mix_create.argtypes = [C.c_int, pint, C.c_int, C.POINTER(DdcC), C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_sdr_mix_create_two_stage.argtypes = [C.c_int, C.c_int, pint, C.c_int, C.POINTER(DdcC), C.POINTER(DdcC),
                                                  C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_sdr_mix_create_raster.argtypes = [C.c_int, pint, C.c_int, C.POINTER(DdcC), C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_sdr_mix_destroy.argtypes = [C.c_void_p]
    L.rxb200_sdr_mix_destroy.restype = None
    L.rxb200_sdr_mix_reset.argtypes = [C.c_void_p]
    L.rxb200_sdr_mix_decimated_len.argtypes = [C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_sdr_mix_process.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_int, C.c_void_p, sz, sz, C.POINTER(sz)]
    L.rxb200_sdr_mix_process_device.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_int, C.c_void_p, sz, sz, C.POINTER(sz),
                                                C.c_int]
    L.rxb200_sdr_mix_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_sdr_mix_stream.argtypes = [C.c_void_p]
    L.rxb200_sdr_mix_stream.restype = C.c_void_p
    L.rxb200_sdr_plan_capture.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.POINTER(FmCapturePlanC), pint]
    pr = C.POINTER(ResamplerC)
    L.rxb200_resample_lowpass.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32)]
    L.rxb200_plan_resample.argtypes = [C.c_longlong, C.c_longlong, C.c_longlong, pr]
    L.rxb200_resample_create.argtypes = [pr, C.c_int, C.POINTER(C.c_void_p)]
    L.rxb200_resample_destroy.argtypes = [C.c_void_p]
    L.rxb200_resample_destroy.restype = None
    L.rxb200_resample_reset.argtypes = [C.c_void_p]
    L.rxb200_resample_out_len.argtypes = [C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_resample_process.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz)]
    L.rxb200_resample_process_device.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz), C.c_int]
    L.rxb200_resample_stream.argtypes = [C.c_void_p]
    L.rxb200_resample_stream.restype = C.c_void_p
    L.rxb200_resample_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.rxb200_resample_device.argtypes = [pr, C.c_ulonglong, C.c_void_p, sz, C.c_void_p, C.c_void_p]
    L.rxb200_resample_in_len.argtypes = [C.c_int, C.c_int, C.c_ulonglong, sz, C.POINTER(sz)]
    L.rxb200_fm_plan_capture_at.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                            C.POINTER(FmCapturePlanC), pint]
    L.rxb200_fm_plan_capture_two_stage_at.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                                      C.POINTER(FmTwoStagePlanC), pint]
    L.rxb200_fm_plan_capture_raster_at.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                                   C.POINTER(FmRasterPlanC), pint]
    L.rxb200_sdr_plan_capture_at.argtypes = [pi64, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                             C.POINTER(FmCapturePlanC), pint]
    L.rxb200_fm_mix_set_device_rate.argtypes = [C.c_void_p, pr]
    L.rxb200_sdr_mix_set_device_rate.argtypes = [C.c_void_p, pr]
    L.rxb200_power_mix_set_device_rate.argtypes = [C.c_void_p, pr]
    L.rxb200_fm_mix_set_input_format.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_sdr_mix_set_input_format.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_power_mix_set_input_format.argtypes = [C.c_void_p, C.c_int]
    L.rxb200_power_plan_capture.argtypes = [C.POINTER(PowerPlanC), C.c_longlong, C.POINTER(FmCapturePlanC), pint]
    L.rxb200_power_plan_capture_at.argtypes = [C.POINTER(PowerPlanC), C.c_longlong, C.c_longlong,
                                               C.POINTER(FmCapturePlanC), pint]
    L.rxb200_power_plan_tiles_at.argtypes = [C.POINTER(PowerPlanC), C.c_longlong, C.c_longlong,
                                             C.POINTER(PowerTilingC), pint]
    L.rxb200_power_mix_set_burst_device_rate.argtypes = [C.c_void_p, pr]
    L.rxb200_power_mix_burst_in_len.argtypes = [C.c_void_p, C.c_int, C.POINTER(sz)]
    _lib = L
    return L


def check(rc: int) -> int:
    if rc < 0:
        raise Rxb200Error(rc, lib().rxb200_last_error().decode(errors="replace"))
    return rc
