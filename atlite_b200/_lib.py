"""ctypes binding of ``libatlite_b200.so`` (C ABI in ``include/atlite_b200.h``).

There is no CPU fallback: if the shared library is missing or a compute entry
point fails (e.g. no CUDA device) an exception is raised.
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libatlite_b200.so")

ATL_OK = 0

# enums (mirror include/atlite_b200.h)
TRACKING = {None: 0, "horizontal": 1, "tilted_horizontal": 2, "vertical": 3, "dual": 4}
TRIGON_SIMPLE, TRIGON_HAY_DAVIES = 0, 1
CLEARSKY = {"simple": 0, "enhanced": 1}
IRR_DIRECT_DIFFUSE, IRR_INFLUX, IRR_ERA5_RAW = 0, 1, 2
ALBEDO_VAR, ALBEDO_OUTFLUX = 0, 1
SOLAR_COMPUTED, SOLAR_STORED_F32, SOLAR_STORED_F64 = 0, 1, 2
PANEL = {"huld": 0, "bofinger": 1}
OUTPUT = {"panel": 0, "total": 1, "direct": 2, "diffuse": 3, "ground": 4, "solar_thermal": 5}
WIND_NONE, WIND_LOG, WIND_POWER = 0, 1, 2
CSP_TECH = {"parabolic trough": 0, "solar tower": 1}
# atl_plan_export array ids
PLAN_ARRAYS = ("tile_slot_ptr", "slot_row", "slot_w4", "slot_rec", "pairs", "active", "slot_ident", "row_slot_ptr",
               "row_slots", "indptr", "indices", "vals")


class AtlError(RuntimeError):
    pass


class PlanInfo(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("n_bus", C.c_int32),
        ("nnz", C.c_int64),
        ("n_tiles", C.c_int32),
        ("n_active_tiles", C.c_int32),
        ("n_slots", C.c_int64),
        ("slots_per_active_tile", C.c_double),
        ("fused", C.c_int32),
        ("pitch", C.c_int32),
        ("vec", C.c_int32),
        ("n_pairs", C.c_int64),
    ]


class PvConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("nt", C.c_int64),
        ("time_ns", C.c_void_p),
        ("time_shift_ns", C.c_int64),
        ("lon_deg", C.c_void_p),
        ("lat_deg", C.c_void_p),
        ("slope_rad", C.c_void_p),
        ("azimuth_rad", C.c_void_p),
        ("tracking", C.c_int32),
        ("trigon_model", C.c_int32),
        ("clearsky_model", C.c_int32),
        ("irr_branch", C.c_int32),
        ("albedo_src", C.c_int32),
        ("solar_src", C.c_int32),
        ("panel_model", C.c_int32),
        ("altitude_threshold_deg", C.c_double),
        ("panel", C.c_double * 16),
        ("output", C.c_int32),
        ("thermal", C.c_double * 3),
        ("pitch", C.c_int32),
        ("orientation_2d", C.c_int32),
    ]


class PvFields(C.Structure):
    _fields_ = [
        (n, C.c_void_p)
        for n in (
            "influx_toa",
            "influx_direct",
            "influx_diffuse",
            "influx",
            "albedo",
            "outflux",
            "temperature",
            "humidity",
            "solar_altitude",
            "solar_azimuth",
        )
    ]


class WindConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("method", C.c_int32),
        ("from_height", C.c_double),
        ("to_height", C.c_double),
        ("n_knots", C.c_int32),
        ("V", C.c_void_p),
        ("POW_norm", C.c_void_p),
        ("pitch", C.c_int32),
    ]


class WindFields(C.Structure):
    _fields_ = [("wnd", C.c_void_p), ("aux", C.c_void_p)]


class WindRawFields(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("u100", "v100", "u10", "v10", "fsr")]


class HeatConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("threshold_c", C.c_double),
        ("a", C.c_double),
        ("constant", C.c_double),
        ("cooling", C.c_int32),
        ("pitch", C.c_int32),
    ]


class PointwiseConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("shift", C.c_double),
        ("nan_to_zero", C.c_int32),
        ("poly", C.c_int32),
        ("sink", C.c_double),
        ("c0", C.c_double),
        ("c1", C.c_double),
        ("c2", C.c_double),
        ("cell_scale", C.c_void_p),
        ("pitch", C.c_int32),
    ]


class PointwiseConfigEx(C.Structure):
    _fields_ = [("base", PointwiseConfig), ("clip_min_zero", C.c_int32)]


class CspConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("nt", C.c_int64),
        ("time_ns", C.c_void_p),
        ("time_shift_ns", C.c_int64),
        ("lon_deg", C.c_void_p),
        ("lat_deg", C.c_void_p),
        ("solar_src", C.c_int32),
        ("technology", C.c_int32),
        ("r_irradiance", C.c_double),
        ("dni_altitude_threshold_deg", C.c_double),
        ("n_alt", C.c_int32),
        ("n_az", C.c_int32),
        ("altitude_rad", C.c_void_p),
        ("azimuth_rad", C.c_void_p),
        ("efficiency", C.c_void_p),
        ("pitch", C.c_int32),
    ]


class ChunkSpec(C.Structure):
    _fields_ = [("ny", C.c_int32), ("nx", C.c_int32), ("elem_bytes", C.c_int32), ("shuffle", C.c_int32),
                ("deflate", C.c_int32), ("chunk", C.c_int64 * 3)]


RAW_FLOAT, RAW_INT, RAW_UINT = 0, 1, 2  # ATL_RAW_* element kinds


class ChunkConvert(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "big_endian", "convert", "has_fill", "has_scale", "has_offset",
                                         "fill_as_int", "reserved")] + [
        ("fill_int", C.c_int64), ("fill", C.c_double), ("scale", C.c_float), ("offset", C.c_float)]


class CspFields(C.Structure):
    _fields_ = [("influx_direct", C.c_void_p), ("solar_altitude", C.c_void_p), ("solar_azimuth", C.c_void_p)]


# atl_reduce_host_many: kind of each job (ATL_JOB_*)
JOB = {"pv": 0, "wind": 1, "wind_raw": 2, "csp": 3, "pointwise": 4, "heat": 5}


class StreamJob(C.Structure):
    _fields_ = [("kind", C.c_int32), ("op", C.c_void_p), ("plan", C.c_void_p), ("fields", C.c_void_p),
                ("t0", C.c_int64), ("day_start", C.c_void_p), ("n_days", C.c_int64), ("chunk", C.c_int64),
                ("out_host", C.c_void_p)]


class StreamStats(C.Structure):
    _fields_ = [("h2d_bytes", C.c_int64), ("n_slabs", C.c_int64)]


class LineRatingConfig(C.Structure):
    _fields_ = [
        ("ny", C.c_int32),
        ("nx", C.c_int32),
        ("pitch", C.c_int32),
        ("nt", C.c_int64),
        ("time_ns", C.c_void_p),
        ("time_shift_ns", C.c_int64),
        ("lon_deg", C.c_void_p),
        ("lat_deg", C.c_void_p),
        ("solar_src", C.c_int32),
        ("n_lines", C.c_int32),
    ] + [(n, C.c_void_p) for n in ("psi", "R", "D", "Ts", "epsilon", "alpha")]


LINE_RATING_FIELDS = ("temperature", "wnd100m", "wnd_azimuth", "influx_direct", "height",
                      "solar_altitude", "solar_azimuth")
LINE_PARAMS = ("psi", "R", "D", "Ts", "epsilon", "alpha")


class LineRatingFields(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in LINE_RATING_FIELDS]


LINE_RATING_RAW_FIELDS = ("t2m", "u100", "v100", "fdir", "height", "solar_altitude", "solar_azimuth")


class LineRatingRawFields(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in LINE_RATING_RAW_FIELDS]


class LineRatingFlat(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in LINE_RATING_FIELDS + LINE_PARAMS]


class Lattice(C.Structure):
    _fields_ = [("c", C.c_double), ("a", C.c_double), ("f", C.c_double), ("e", C.c_double),
                ("nx", C.c_int64), ("ny", C.c_int64)]


class Laea(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("e2", "e", "qp", "rq", "sin_b0", "cos_b0", "d", "lam0", "fe", "fn",
                                          "s1", "s2", "s3")] + [("newton", C.c_int32)]


CRS_LONLAT, CRS_LAEA, CRS_MERCATOR, CRS_MOLLWEIDE = 0, 1, 2, 3


class Crs(C.Structure):
    _fields_ = [("kind", C.c_int32), ("newton", C.c_int32), ("r", C.c_double)]


class Projection(C.Structure):  # AtlProjection: C's `from` is `from_` here
    _fields_ = [("from_", Crs), ("to", Crs), ("laea", Laea)]


MASK_EVEN_ODD, MASK_NONZERO = 0, 1
AVAIL_TILE = 16

REGRID_DTYPE = {"int16": 0, "float32": 1, "float64": 2}  # ATL_REGRID_I16 / _F32 / _F64
RESAMPLING_NEAREST, RESAMPLING_AVERAGE = 0, 5  # ATL_RESAMPLING_*
RESAMPLING_MODE, RESAMPLING_MAX, RESAMPLING_MIN, RESAMPLING_MED, RESAMPLING_Q1, RESAMPLING_Q3 = 6, 8, 9, 10, 11, 12
RESAMPLING_SUM, RESAMPLING_RMS = 13, 14


class Reproject(C.Structure):
    _fields_ = [("src", Lattice), ("dst", Lattice), ("proj", Projection), ("resampling", C.c_int32),
                ("has_nodata", C.c_int32), ("src_nodata", C.c_double), ("dst_nodata", C.c_double),
                ("tile_y", C.c_int32), ("tile_x", C.c_int32)]


class Span(C.Structure):  # AtlSpan
    _fields_ = [("lo", C.c_int32), ("hi", C.c_int32), ("w_lo", C.c_double), ("w_hi", C.c_double)]


class ReprojectOptions(C.Structure):  # AtlReprojectOptions
    _fields_ = [("row_spans", C.c_void_p), ("col_spans", C.c_void_p), ("scratch_bytes", C.c_int64),
                ("select_small", C.c_int32), ("reserved", C.c_int32)]


class RasterSample(C.Structure):
    _fields_ = [("win", Lattice), ("ras", Lattice), ("proj", Projection), ("idx", C.c_void_p),
                ("idx_bytes", C.c_int32), ("mask", C.c_void_p), ("mask_i0", C.c_int64), ("mask_j0", C.c_int64),
                ("mask_nx", C.c_int64), ("mask_ny", C.c_int64), ("lut", C.c_void_p), ("ex_nodata", C.c_int32),
                ("or_into", C.c_int32), ("out", C.c_void_p), ("win_row0", C.c_int64)]


class GeomExclusion(C.Structure):
    _fields_ = [("win", Lattice), ("segs", C.c_void_p), ("n_segs", C.c_int64), ("buffer", C.c_double),
                ("invert", C.c_int32), ("inside", C.c_void_p), ("tile_cnt", C.c_void_p),
                ("tile_cursor", C.c_void_p), ("tile_ptr", C.c_void_p), ("tile_list", C.c_void_p),
                ("excl", C.c_void_p)]


class AvailCount(C.Structure):
    _fields_ = [("win", Lattice), ("proj", Projection), ("excl", C.c_void_p),
                ("gx0", C.c_double), ("gdx", C.c_double), ("gy0", C.c_double), ("gdy", C.c_double),
                ("gnx", C.c_int64), ("gny", C.c_int64), ("counts", C.c_void_p), ("win_row0", C.c_int64)]


class AvailAverage(C.Structure):
    _fields_ = [("win", Lattice), ("dst", Lattice), ("proj", Projection), ("pad", C.c_int64)] + [
        (n, C.c_int32) for n in ("row0", "col0", "row1", "col1", "tile_y", "tile_x")]


TIFF_NONE, TIFF_LZW, TIFF_DEFLATE = 1, 5, 8  # ATL_TIFF_* compressions


class TiffLayout(C.Structure):
    _fields_ = [("compression", C.c_int32), ("predictor", C.c_int32), ("sample_bytes", C.c_int32),
                ("big_endian", C.c_int32), ("tiled", C.c_int32)] + [
        (n, C.c_int64) for n in ("width", "height", "seg_w", "seg_h", "win_r0", "win_c0", "win_ny", "win_nx")]


class TiffStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("segments", "stored_bytes", "xfer_bytes", "batches")]


# name -> (restype, argtypes); every symbol declared in include/atlite_b200.h
_P = C.c_void_p
_SIGNATURES = {
    "atl_abi_version": (C.c_int, []),
    "atl_hash128": (C.c_int, [_P, C.c_int64, C.c_uint64, _P]),
    "atl_last_error": (C.c_char_p, []),
    "atl_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "atl_launch_count": (C.c_int64, []),
    "atl_set_deterministic": (C.c_int, [C.c_int]),
    "atl_device_local_cpus": (C.c_int, [C.c_int, _P, C.c_int32, C.POINTER(C.c_int32)]),
    "atl_plan_create": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(_P)]),
    "atl_plan_create_pitched": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(_P)]),
    "atl_plan_info": (C.c_int, [_P, C.POINTER(PlanInfo)]),
    "atl_plan_create_device": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P,
                                         C.c_int, _P, C.POINTER(_P)]),
    "atl_plan_export": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "atl_plan_tiling_host": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(PlanInfo), _P, _P, _P, C.c_int64]),
    "atl_plan_pairs_host": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(C.c_int64), _P, _P, _P,
                                      C.c_int64, C.c_int64]),
    "atl_plan_create_entries": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(_P)]),
    "atl_plan_destroy": (None, [_P]),
    "atl_spmm": (C.c_int, [_P, _P, C.c_int64, _P, _P]),
    "atl_pv_create": (C.c_int, [C.c_int, C.POINTER(PvConfig), C.POINTER(_P)]),
    "atl_pv_destroy": (None, [_P]),
    "atl_pv_reduce": (C.c_int, [_P, _P, C.POINTER(PvFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_pv_cells": (C.c_int, [_P, C.POINTER(PvFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_pv_timesum": (C.c_int, [_P, C.POINTER(PvFields), C.c_int64, C.c_int64, _P, _P, _P]),
    "atl_pv_reduce_host": (C.c_int, [_P, _P, C.POINTER(PvFields), C.c_int64, C.c_int64, _P, C.c_int64]),
    "atl_pv_op_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 4),
    "atl_release_host_staging": (None, []),
    "atl_era5_wind": (C.c_int, [C.c_int, C.c_int64] + [_P] * 5 + [C.c_int32] + [_P] * 4 + [_P]),
    "atl_era5_influx": (C.c_int, [C.c_int, C.c_int64] + [_P] * 4 + [C.c_int32] + [_P] * 4 + [_P]),
    "atl_solar_position": (C.c_int, [C.c_int, _P, C.c_int64, C.c_int64, _P, C.c_int32, _P, C.c_int32, _P, _P, _P]),
    "atl_indicator_compute": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double,
                                        C.c_double, C.c_int32, _P, _P, _P, _P, C.POINTER(_P)]),
    "atl_intersection_compute": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double,
                                           C.c_double, _P, _P, _P, _P, C.c_int32, _P, _P, _P, _P, C.POINTER(_P)]),
    "atl_overlay_compute": (C.c_int, [C.c_int, C.c_int32, _P, _P, _P, _P, C.c_int32, _P, _P, _P, _P, C.POINTER(_P)]),
    "atl_intersects_compute": (C.c_int, [C.c_int, C.c_int32, _P, _P, _P, _P, C.c_int32, _P, _P, _P, _P,
                                         C.POINTER(_P)]),
    "atl_indicator_nnz": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "atl_indicator_export": (C.c_int, [_P, _P, _P, _P]),
    "atl_indicator_destroy": (None, [_P]),
    "atl_decode_chunks": (C.c_int, [C.c_char_p, C.POINTER(ChunkSpec), C.c_int64, _P, _P, _P, C.c_int64, C.c_int64, _P,
                                    C.c_int32]),
    "atl_decode_chunks_device": (C.c_int, [C.c_int, C.c_char_p, C.POINTER(ChunkSpec), C.c_int64, _P, _P, _P,
                                           C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                           C.POINTER(ChunkConvert), _P, C.c_int64, C.c_int64, C.c_int32, _P]),
    "atl_wind_create": (C.c_int, [C.c_int, C.POINTER(WindConfig), C.POINTER(_P)]),
    "atl_wind_curve_eval_host": (C.c_int, [_P, _P, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P]),
    "atl_wind_curve_info_host": (C.c_int, [_P, _P, C.c_int32, C.c_int32, _P]),
    "atl_wind_destroy": (None, [_P]),
    "atl_wind_reduce": (C.c_int, [_P, _P, C.POINTER(WindFields), C.c_int64, _P, _P]),
    "atl_wind_cells": (C.c_int, [_P, C.POINTER(WindFields), C.c_int64, _P, _P]),
    "atl_wind_timesum": (C.c_int, [_P, C.POINTER(WindFields), C.c_int64, _P, _P, _P]),
    "atl_wind_reduce_host": (C.c_int, [_P, _P, C.POINTER(WindFields), C.c_int64, _P, C.c_int64]),
    "atl_wind_op_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 3),
    "atl_wind_raw_reduce": (C.c_int, [_P, _P, C.POINTER(WindRawFields), C.c_int64, _P, _P]),
    "atl_wind_raw_cells": (C.c_int, [_P, C.POINTER(WindRawFields), C.c_int64, _P, _P]),
    "atl_wind_raw_timesum": (C.c_int, [_P, C.POINTER(WindRawFields), C.c_int64, _P, _P, _P]),
    "atl_wind_raw_reduce_host": (C.c_int, [_P, _P, C.POINTER(WindRawFields), C.c_int64, _P, C.c_int64]),
    "atl_heat_create": (C.c_int, [C.c_int, C.POINTER(HeatConfig), C.POINTER(_P)]),
    "atl_heat_destroy": (None, [_P]),
    "atl_heat_reduce": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, _P]),
    "atl_heat_cells": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P]),
    "atl_heat_timesum": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, _P]),
    "atl_heat_reduce_host": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, C.c_int64]),
    "atl_heat_op_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 3),
    "atl_reduce_host_many": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int64, _P, C.c_int32, C.c_int64,
                                       C.POINTER(StreamStats)]),
    "atl_pointwise_create": (C.c_int, [C.c_int, C.POINTER(PointwiseConfig), C.POINTER(_P)]),
    "atl_pointwise_destroy": (None, [_P]),
    "atl_pointwise_reduce": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P]),
    "atl_pointwise_cells": (C.c_int, [_P, _P, C.c_int64, _P, _P]),
    "atl_pointwise_timesum": (C.c_int, [_P, _P, C.c_int64, _P, _P, _P]),
    "atl_pointwise_reduce_host": (C.c_int, [_P, _P, _P, C.c_int64, _P, C.c_int64]),
    "atl_pointwise_op_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 3),
    "atl_pointwise_create_ex": (C.c_int, [C.c_int, C.POINTER(PointwiseConfigEx), C.POINTER(_P)]),
    "atl_csp_create": (C.c_int, [C.c_int, C.POINTER(CspConfig), C.POINTER(_P)]),
    "atl_csp_raw_create": (C.c_int, [C.c_int, C.POINTER(CspConfig), C.POINTER(_P)]),
    "atl_csp_destroy": (None, [_P]),
    "atl_csp_reduce": (C.c_int, [_P, _P, C.POINTER(CspFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_csp_cells": (C.c_int, [_P, C.POINTER(CspFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_csp_timesum": (C.c_int, [_P, C.POINTER(CspFields), C.c_int64, C.c_int64, _P, _P, _P]),
    "atl_csp_reduce_host": (C.c_int, [_P, _P, C.POINTER(CspFields), C.c_int64, C.c_int64, _P, C.c_int64]),
    "atl_csp_op_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 4),
    "atl_line_rating_create": (C.c_int, [C.c_int, C.POINTER(LineRatingConfig), C.POINTER(_P)]),
    "atl_line_rating_destroy": (None, [_P]),
    "atl_line_rating_reduce": (C.c_int, [_P, _P, C.POINTER(LineRatingFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_line_rating_raw_reduce": (C.c_int, [_P, _P, C.POINTER(LineRatingRawFields), C.c_int64, C.c_int64, _P, _P]),
    "atl_line_rating_eval": (C.c_int, [C.c_int, C.c_int64, C.POINTER(LineRatingFlat), _P, _P]),
    "atl_hydro_shift_sum": (C.c_int, [C.c_int, C.c_int32, C.c_int64, _P, C.c_int32, _P, _P, _P, _P, _P, _P]),
    "atl_avail_mask": (C.c_int, [C.c_int, C.POINTER(Lattice), C.c_int64, C.c_int64, _P, _P, _P, _P, _P, _P,
                                 C.c_int32, C.c_int32, _P]),
    "atl_avail_raster_sample": (C.c_int, [C.c_int, C.POINTER(RasterSample), _P]),
    "atl_avail_dilate": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, _P]),
    "atl_avail_geom_bin": (C.c_int, [C.c_int, C.POINTER(GeomExclusion), C.c_int64, C.c_int32, _P]),
    "atl_avail_geometry": (C.c_int, [C.c_int, C.POINTER(GeomExclusion), C.c_int64, _P]),
    "atl_avail_count": (C.c_int, [C.c_int, C.POINTER(AvailCount), _P]),
    "atl_avail_average_rect": (C.c_int, [C.c_int, C.POINTER(AvailAverage), _P, _P, _P]),
    "atl_avail_average_counts": (C.c_int, [C.c_int, C.POINTER(AvailAverage), _P, C.c_int64, C.c_int64, _P, _P]),
    "atl_avail_average_finalize": (C.c_int, [C.c_int, C.POINTER(AvailAverage), _P, _P, _P]),
    "atl_avail_average_corners": (C.c_int, [C.c_int, C.POINTER(AvailAverage), _P, _P]),
    "atl_regrid_create": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P,
                                    C.c_int32, _P, _P, _P, C.POINTER(_P)]),
    "atl_regrid_info": (C.c_int, [_P] + [C.POINTER(C.c_int32)] * 4),
    "atl_regrid_f32": (C.c_int, [_P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P]),
    "atl_regrid_f64": (C.c_int, [_P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P]),
    "atl_regrid_destroy": (None, [_P]),
    "atl_regrid_band_rows": (C.c_int, [_P, _P, _P]),
    "atl_regrid_window": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int64,
                                    C.c_int32, C.c_double, _P, _P]),
    "atl_regrid_nodata": (C.c_int, [_P, C.c_int32, C.c_int64, _P, C.c_int64, C.c_int64, C.c_int32, C.c_double,
                                    C.c_double, _P, _P]),
    "atl_reproject": (C.c_int, [C.c_int, C.POINTER(Reproject), C.c_int32, C.c_int64, _P, C.c_int64, C.c_int64, _P,
                                _P]),
    "atl_reproject_ex": (C.c_int, [C.c_int, C.POINTER(Reproject), C.POINTER(ReprojectOptions), C.c_int32, C.c_int64,
                                   _P, C.c_int64, C.c_int64, _P, _P]),
    "atl_sarah_fill": (C.c_int, [C.c_int, C.c_int32, C.c_int64, _P, _P, C.c_int32, _P, C.c_int32, C.c_int32, _P, _P,
                                 _P]),
    "atl_geotiff_read": (C.c_int, [C.c_int, C.c_char_p, C.POINTER(TiffLayout), C.c_int64, _P, _P, _P, C.c_int64,
                                   C.c_int32, _P, C.POINTER(C.c_int64), C.POINTER(TiffStats), _P]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib, LIB_PATH
    if _lib is not None:
        return _lib
    if os.environ.get("ATL_LIB_PATH"):  # another build of the same library, e.g. another commit's, for A/B timing
        LIB_PATH = os.path.abspath(os.environ["ATL_LIB_PATH"])
    if not os.path.exists(LIB_PATH):
        raise AtlError(
            f"{LIB_PATH} not found: build the CUDA library first "
            "(python -c 'import __graft_entry__ as g; g.build()' or make -C atlite_b200/csrc). "
            "atlite_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so is stale
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != ATL_OK:
        msg = load().atl_last_error()
        raise AtlError(f"libatlite_b200 error {rc}: {msg.decode() if msg else ''}")


def set_deterministic(on=True):
    """Bitwise-repeatable fused reductions (fixed summation order); returns the previous setting."""
    return bool(load().atl_set_deterministic(1 if on else 0))


def release_host_staging():
    """Free the pinned staging buffers the host-streaming calls keep between calls."""
    load().atl_release_host_staging()


def launch_count():
    return int(load().atl_launch_count())


def device_count():
    n = C.c_int(0)
    rc = load().atl_device_count(C.byref(n))
    return n.value if rc == ATL_OK else 0


def device_local_cpus(device):
    """CPU ids next to GPU `device` (its NUMA node), [] when the topology is unknown."""
    n = C.c_int32(0)
    buf = np.zeros(4096, dtype=np.int32)
    check(load().atl_device_local_cpus(int(device), buf.ctypes.data_as(C.c_void_p), len(buf), C.byref(n)))
    return [int(c) for c in buf[: min(n.value, len(buf))]]


def ptr(a):
    """Host pointer of a C-contiguous NumPy array (kept alive by the caller)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def as_f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))
