/*
 * atlite_b200.h -- C ABI of libatlite_b200.so
 *
 * H100-native (sm_90a) replacement for the conversion-and-aggregation hot
 * path of PyPSA/atlite.  Plain C: pointers, sizes, opaque handles; no torch
 * or C++ types cross this boundary.  The reference is pure Python, so the
 * "FFI a maintainer would bind" is a ctypes stub (see INTEGRATION.md); the
 * entry points below are cut exactly where the reference hands work to
 * NumPy/dask/scipy:
 *
 *   reference (paths relative to atlite/)      entry point
 *   ---------------------------------------------------------  ------------------------
 *   aggregate.py:16-35  aggregate_matrix (dense x CSR^T)        atl_plan_create + *_reduce, atl_spmm
 *   convert.py:840-854  convert_pv  (+ pv/*.py)                 atl_pv_create, atl_pv_reduce/cells/timesum
 *   convert.py:634-662  convert_wind (+ wind.py:24-128)         atl_wind_create, atl_wind_*
 *   convert.py:405-418  convert_heat_demand                     atl_heat_create, atl_heat_*
 *   convert.py:475-491  convert_cooling_demand                  atl_heat_* with AtlHeatConfig.cooling = 1
 *   convert.py:748-767  convert_irradiation                     atl_pv_* with AtlPvConfig.output = ATL_OUT_TOTAL..GROUND
 *   convert.py:550-573  convert_solar_thermal                   atl_pv_* with AtlPvConfig.output = ATL_OUT_SOLAR_THERMAL
 *   convert.py:292-366  temperature / soil / dewpoint / COP     atl_pointwise_*
 *   convert.py:1028-1034 convert_runoff                         atl_pointwise_* with cell_scale = height
 *   datasets/era5.py:104-256 (raw ERA5 variables, no prepare)   atl_pv_* with irr_branch = ATL_IRR_ERA5_RAW,
 *                                                               atl_wind_raw_*, atl_csp_raw_create,
 *                                                               atl_line_rating_raw_reduce,
 *                                                               atl_pointwise_create_ex (runoff from ro);
 *                                                               derivations fused in-kernel
 *   convert.py:940-972  convert_csp (+ csp.py:18-58)            atl_csp_*
 *   hydro.py:81-104     shift_and_aggregate_runoff_for_plants   atl_hydro_shift_sum
 *   gis.py:263-325      shape_availability (+ availabilitymatrix) atl_avail_mask, _raster_sample, _dilate,
 *                                                               _geom_bin, _geometry, _count
 *   gis.py:328-373      shape_availability_reprojected          atl_avail_average_rect, _counts, _finalize
 *   gis.py:791-871      regrid (average / nearest, one CRS)     atl_regrid_create, atl_regrid_f32 / _f64
 *   datasets/gebco.py:23-44 get_data_gebco_height (average)     atl_regrid_band_rows, atl_regrid_window
 *   rasterio.warp.reproject (gis.reproject)                     atl_reproject(_ex); atl_regrid_nodata (one CRS)
 *   datasets/sarah.py:91-159 interpolate / fillna / hourly_mean atl_sarah_fill
 *   convert.py:200-211  no-matrix branch (_aggregate_time)      *_cells, *_timesum
 *   convert.py:257-271  reduce + time aggregation               *_reduce (+ host finalisation in Python)
 *
 * Conventions
 *   - All weather fields are C-contiguous (time, y, x) float32 slabs, x fastest
 *     (the cutout's NetCDF layout; SURVEY.md section 8).  A "slab" covers time
 *     steps [t0, t0+nt) of the operator's time axis and its pointers address
 *     the slab's first step.
 *   - `pitch` (0 = nx): elements per stored row of the DEVICE input fields.  A
 *     device-resident cutout whose width is not a multiple of 4 may be stored
 *     row-padded (pitch = round_up(nx, 4), padding contents arbitrary) so that
 *     the 128-bit kernels apply; operator and plan must be created with the same
 *     pitch.  Host entry points (*_reduce_host) always take unpadded arrays
 *     (pitch = nx operators); per-cell OUTPUTS are never padded.
 *   - Pointers named *_dev are device pointers on the operator's device, those
 *     named *_host are host pointers.  Small tables (coordinates, time axis,
 *     power curve) are always host pointers and are copied at create time.
 *   - The aggregated output is (nt, n_bus) float32, time-major -- the dim
 *     order of the reference's dask branch (aggregate.py:24-32) -- and is
 *     OVERWRITTEN (zero-filled, then accumulated) by each *_reduce call.
 *   - Every function returns ATL_OK (0) or a negative error code;
 *     atl_last_error() returns a thread-local message.  Nothing here falls
 *     back to a CPU implementation: without a CUDA device every compute entry
 *     point fails with ATL_ERR_CUDA.
 *   - stream: a cudaStream_t passed as void* (NULL = default stream).  Calls
 *     are asynchronous w.r.t. the host unless stated otherwise.
 */
#ifndef ATLITE_B200_H
#define ATLITE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ATL_OK 0
#define ATL_ERR_INVALID (-1) /* bad argument / unsupported combination */
#define ATL_ERR_CUDA (-2)    /* CUDA runtime error (see atl_last_error) */
#define ATL_ERR_NOMEM (-3)

#define ATL_ABI_VERSION 6

int atl_abi_version(void);
const char* atl_last_error(void);
int atl_device_count(int* count_out);
/* Host-only: 128-bit content hash of a byte range (MurmurHash3-style mixing, ~5 GB/s).  The
 * Python layer keys its plan cache on it: the reference rebuilds nothing per call, here a
 * matrix that is already planned must be recognised faster than it could be re-planned
 * (convert.py:213-249 hands over a fresh scipy matrix every call). */
int atl_hash128(const void* data, int64_t nbytes, uint64_t seed, uint64_t out[2]);
/* Deterministic reduce mode (default off, or env ATL_DETERMINISTIC=1): the fused
 * kernels accumulate every (tile, bus) partial in a private slot and a second
 * kernel sums each bus's slots in a fixed order -> bitwise-repeatable results at
 * ~2 % extra traffic.  Returns the previous setting. */
int atl_set_deterministic(int on);
/* CPUs the kernel lists as local to the GPU's PCI device (its NUMA node): host-streaming
 * calls bind their staging threads there for the duration of the call (ATL_NUMA_BIND=0
 * disables).  Fills up to `capacity` CPU ids, *n_out = how many there are (0 = unknown). */
int atl_device_local_cpus(int device, int32_t* cpus_out, int32_t capacity, int32_t* n_out);

/* ------------------------------------------------------------------ */
/* Aggregation plan: the (n_bus x S) CSR indicator/layout matrix       */
/* (convert.py:213-254) pre-tiled for the fused reduce kernels.        */
/* ------------------------------------------------------------------ */
typedef struct AtlPlan AtlPlan;

typedef struct {
  int32_t ny, nx, n_bus;
  int64_t nnz;            /* stored entries after merging duplicates   */
  int32_t n_tiles;        /* 32x4-cell warp tiles covering the grid     */
  int32_t n_active_tiles; /* tiles touched by at least one entry        */
  int64_t n_slots;        /* distinct (tile, bus) pairs                 */
  double slots_per_active_tile;
  int32_t fused;          /* 1: fused tile path, 0: two-pass CSR fallback */
  int32_t pitch;          /* row pitch of the input fields (elements), >= nx */
  int32_t vec;            /* 1: 128-bit lane layout (pitch % 4 == 0), 0: scalar */
  int64_t n_pairs;        /* stored (slot, cell) entries the staged reduce walks     */
} AtlPlanInfo;

/* indptr/indices/data: host CSR arrays (scipy layout), column index
 * s = iy*nx + ix (cutout.grid order, cutout.py:355-376). */
int atl_plan_create(int device, int32_t ny, int32_t nx, int32_t n_bus,
                    const int64_t* indptr_host, const int32_t* indices_host,
                    const double* data_host, AtlPlan** plan_out);
int atl_plan_create_pitched(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus,
                            const int64_t* indptr_host, const int32_t* indices_host,
                            const double* data_host, AtlPlan** plan_out);
int atl_plan_info(const AtlPlan* plan, AtlPlanInfo* info_out);
/* The same plan from a CSR matrix that already lives on `device`: indptr_dev (n_bus + 1, int64,
 * starting at 0 and ending at nnz), indices_dev (nnz, int32), data_dev (nnz, float64).  Duplicates
 * of one (bus, cell) are summed in CSR order, as by the host-array entry points, which upload their
 * arrays and call this builder.  entries != 0: as atl_plan_create_entries.  The build runs on
 * `stream` (a cudaStream_t, NULL = the legacy default stream); it reads one small block of counts
 * back to size the plan, and the plan is complete when the call returns. */
int atl_plan_create_device(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus, int64_t nnz,
                           const int64_t* indptr_dev, const int32_t* indices_dev, const double* data_dev,
                           int entries, void* stream, AtlPlan** plan_out);
/* Test hook: copies one device array of a plan to the host.  *bytes_out = its size in bytes (0 for
 * an array the plan does not have, e.g. the weight vectors of a plan that does not tile); the copy
 * is made when dst_host is given and capacity_bytes >= that size. */
#define ATL_PLAN_TILE_SLOT_PTR 0 /* int32 [n_tiles + 1]                                     */
#define ATL_PLAN_SLOT_ROW 1      /* int32 [n_slots]                                         */
#define ATL_PLAN_SLOT_W4 2       /* float [(n_slots + 3) * 128], lane order, 3 zero slots   */
#define ATL_PLAN_SLOT_REC 3      /* int32 pairs [n_slots] {first entry, entries / 8}        */
#define ATL_PLAN_PAIRS 4         /* {uint32 byte offset, float weight}, padded to 8 / slot */
#define ATL_PLAN_ACTIVE 5        /* int32 [n_active_tiles]                                  */
#define ATL_PLAN_SLOT_IDENT 6    /* int32 [n_slots] (deterministic mode)                    */
#define ATL_PLAN_ROW_SLOT_PTR 7  /* int32 [n_bus + 1] (deterministic mode)                  */
#define ATL_PLAN_ROW_SLOTS 8     /* int32 [n_slots] (deterministic mode)                    */
#define ATL_PLAN_INDPTR 9        /* int64 [n_bus + 1]                                       */
#define ATL_PLAN_INDICES 10      /* int32 [nnz]                                             */
#define ATL_PLAN_VALS 11         /* float [nnz]                                             */
int atl_plan_export(const AtlPlan* plan, int32_t array_id, void* dst_host, int64_t capacity_bytes,
                    int64_t* bytes_out);
/* Host-only view of the tiling (no CUDA needed; used by the CPU tests and for
 * inspection): fills *info_out; when the three output arrays are given
 * (slot_capacity >= n_slots) also tile_slot_ptr[n_tiles+1], slot_row[n_slots] and
 * slot_w[n_slots*128] (weights in lane order; VEC layout iff nx % 4 == 0:
 * cell (iy, ix) of a tile sits at ((iy%4)*8 + (ix%32)/4)*4 + ix%4, else at
 * (ix%32)*4 + iy%4). */
int atl_plan_tiling_host(int32_t ny, int32_t nx, int32_t n_bus, const int64_t* indptr_host,
                         const int32_t* indices_host, const double* data_host,
                         AtlPlanInfo* info_out, int32_t* tile_slot_ptr_out,
                         int32_t* slot_row_out, float* slot_w_out, int64_t slot_capacity);
/* Host-only view of the entry lists heat demand's staged reduce walks (CPU tests): for slot s
 * (same numbering as atl_plan_tiling_host) the entries slot_pair_ptr[s] .. slot_pair_ptr[s+1],
 * each {pair_cell = position 32*i + lane of the cell in the warp's staging row, pair_w}.
 * Duplicates of one (bus, cell) are summed, explicit zeros kept (scipy CSR semantics:
 * aggregate.py:25 multiplies exactly the stored entries).  Always fills *n_pairs_out; the
 * arrays only when all three are given. */
int atl_plan_pairs_host(int32_t ny, int32_t nx, int32_t n_bus, const int64_t* indptr_host,
                        const int32_t* indices_host, const double* data_host,
                        int64_t* n_pairs_out, int32_t* slot_pair_ptr_out, int32_t* pair_cell_out,
                        float* pair_w_out, int64_t slot_capacity, int64_t pair_capacity);
void atl_plan_destroy(AtlPlan* plan);

/* Generic (time, S) dense  x  CSR^T  ->  (time, n_bus)  (aggregate.py:24-32):
 * the path for unknown convert_func results. */
int atl_spmm(const AtlPlan* plan, const float* dense_dev, int64_t nt,
             float* out_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Cutout ingest: parallel decode of compressed (time, y, x) chunks      */
/* (the storage format of data.py:139,245-248: zlib + byte shuffle; the  */
/* read path of cutout.py:142-154)                                       */
/* ------------------------------------------------------------------ */
typedef struct {
  int32_t ny, nx;       /* grid of the variable                                   */
  int32_t elem_bytes;   /* 2, 4 or 8                                              */
  int32_t shuffle;      /* 1: HDF5 byte-shuffle filter was applied before deflate */
  int32_t deflate;      /* 1: chunks are zlib streams; 0: stored raw              */
  int64_t chunk[3];     /* chunk shape (time, y, x); edge chunks are stored whole */
} AtlChunkSpec;
/* Decode the listed chunks of one variable into dst_host, a C-contiguous (nt, ny, nx) slab
 * holding steps [t0, t0 + nt): every chunk is pread from `path` at file_offset[c]
 * (stored_bytes[c] bytes), inflated, un-shuffled and its part inside the slab copied to its
 * place; chunk_origin[3c..3c+2] = (t, y, x) of the chunk's first element.  Chunks run in
 * parallel on n_threads host threads (0 = all cores, at most 64).  Bytes are copied as
 * stored (the caller converts endianness / packing).  No GPU involved. */
int atl_decode_chunks(const char* path, const AtlChunkSpec* spec, int64_t n_chunks,
                      const int64_t* file_offset, const int64_t* stored_bytes,
                      const int64_t* chunk_origin, int64_t t0, int64_t nt, void* dst_host,
                      int32_t n_threads);

/* Per-stream status of the GPU zlib decoder (k_inflate, csrc/inflate.cu). */
#define ATL_INFLATE_OK 0
#define ATL_INFLATE_BAD_HEADER 1      /* not CM 8 with CINFO <= 7, or FCHECK wrong */
#define ATL_INFLATE_DICTIONARY 2      /* FDICT set: preset dictionaries are not supported */
#define ATL_INFLATE_BAD_BLOCK_TYPE 3  /* BTYPE 3 */
#define ATL_INFLATE_STORED_LENGTH 4   /* stored block with LEN != ~NLEN */
#define ATL_INFLATE_BAD_CODELEN_SET 5 /* invalid code-length code or code-length sequence */
#define ATL_INFLATE_BAD_LITLEN_SET 6  /* invalid literal/length code set */
#define ATL_INFLATE_BAD_DIST_SET 7    /* invalid distance code set */
#define ATL_INFLATE_BAD_SYMBOL 8      /* literal/length 286/287, distance 30/31, or no code */
#define ATL_INFLATE_TOO_FAR 9         /* distance before the start of the output */
#define ATL_INFLATE_LONG 10           /* more output than the span holds */
#define ATL_INFLATE_TRUNCATED 11      /* the input ends before the stream does */
#define ATL_INFLATE_SHORT 12          /* the stream ends before the span is full */
#define ATL_INFLATE_ADLER 13          /* Adler-32 trailer mismatch */
/* How raw chunk elements become float32, as ChunkedVariable.load does on the host: swap
 * big-endian elements, cast to float32 (round to nearest), a raw value equal to the fill value ->
 * NaN, then *= scale and += offset, each rounded on its own.  NaN operands propagate as x86 SSE
 * propagates them (quietened, payload kept), so results match the host bit for bit. */
#define ATL_RAW_FLOAT 0
#define ATL_RAW_INT 1
#define ATL_RAW_UINT 2
typedef struct {
  int32_t kind;        /* ATL_RAW_FLOAT / _INT / _UINT; the size is the spec's elem_bytes */
  int32_t big_endian;  /* elements are stored big-endian */
  int32_t convert;     /* 0: copy the bits (float32 without packing), 1: convert as above */
  int32_t has_fill, has_scale, has_offset;
  int32_t fill_as_int; /* compare raw == fill_int (integer kinds), else (double)raw == fill */
  int32_t reserved;
  int64_t fill_int;
  double fill;
  float scale, offset;
} AtlChunkConvert;
/* The device path of the same chunks: steps [t0, t0 + nt) x rows [y0, y0 + wy) x columns
 * [x0, x0 + wx) of the variable, as float32, into dst_dev, a (nt, wy, pitch) device array
 * (pitch >= wx elements; columns [wx, pitch) are zeroed).  Only the chunks that meet the window
 * are read; they cross PCIe compressed, in batches of at most batch_bytes compressed and decoded
 * bytes (one chunk at least), are inflated on the GPU (k_inflate) when spec->deflate, and a second
 * kernel un-shuffles, swaps, converts (*conv) and scatters the window's elements.  Chunks missing
 * from the index read as raw zeros.  Read with n_threads host threads (0: one per CPU, at most
 * 64).  Synchronous.  A corrupt chunk returns ATL_ERR_INVALID, the message starting "zlib:" and
 * naming the chunk's origin and the reason. */
int atl_decode_chunks_device(int device, const char* path, const AtlChunkSpec* spec, int64_t n_chunks,
                             const int64_t* file_offset, const int64_t* stored_bytes,
                             const int64_t* chunk_origin, int64_t t0, int64_t nt, int64_t y0, int64_t wy,
                             int64_t x0, int64_t wx, const AtlChunkConvert* conv, float* dst_dev,
                             int64_t pitch, int64_t batch_bytes, int32_t n_threads, void* stream);

/* ------------------------------------------------------------------ */
/* PV: SolarPosition -> SurfaceOrientation -> TiltedIrradiation ->     */
/* SolarPanelModel (convert.py:840-854)                                */
/* ------------------------------------------------------------------ */
enum { ATL_TRACK_NONE = 0, ATL_TRACK_HORIZONTAL = 1, ATL_TRACK_TILTED_HORIZONTAL = 2,
       ATL_TRACK_VERTICAL = 3, ATL_TRACK_DUAL = 4 };       /* pv/orientation.py:114-176 */
enum { ATL_TRIGON_SIMPLE = 0, ATL_TRIGON_HAY_DAVIES = 1 };  /* pv/irradiation.py:214-236 */
enum { ATL_CLEARSKY_SIMPLE = 0, ATL_CLEARSKY_ENHANCED = 1 };/* pv/irradiation.py:33-65  */
enum { ATL_IRR_DIRECT_DIFFUSE = 0, ATL_IRR_INFLUX = 1,    /* pv/irradiation.py:202-208 */
       /* raw ERA5 variables, derived in-kernel as datasets/era5.py:163-175 + 195-201 (sanitized)
        * do; AtlPvFields slots: influx <- ssrd, outflux <- ssr, influx_toa <- tisr,
        * influx_direct <- fdir (hourly J m-2 accumulations), temperature <- t2m; albedo_src is
        * ignored.  Pair it with time_shift_ns = -30 min to match a cutout whose stored solar
        * position era5.py:182-188 computed. */
       ATL_IRR_ERA5_RAW = 2 };
enum { ATL_ALBEDO_VAR = 0, ATL_ALBEDO_OUTFLUX = 1 };        /* pv/irradiation.py:128-139 */
enum { ATL_SOLAR_COMPUTED = 0, ATL_SOLAR_STORED_F32 = 1, ATL_SOLAR_STORED_F64 = 2 }; /* pv/solar_position.py:54-60 vs 69-116 */
enum { ATL_PANEL_HULD = 0, ATL_PANEL_BOFINGER = 1 };        /* pv/solar_panel_model.py:12-74 */
/* what the PV operator emits: panel power (convert_pv), one tilted-irradiation
 * component (convert_irradiation, pv/irradiation.py:238-245), or solar-thermal
 * collector output (convert_solar_thermal, convert.py:565-573) */
enum { ATL_OUT_PANEL = 0, ATL_OUT_TOTAL = 1, ATL_OUT_DIRECT = 2, ATL_OUT_DIFFUSE = 3,
       ATL_OUT_GROUND = 4, ATL_OUT_SOLAR_THERMAL = 5 };

typedef struct {
  int32_t ny, nx;
  int64_t nt;                 /* length of the time axis                        */
  const int64_t* time_ns;     /* host, nt: datetime64[ns] UTC                   */
  int64_t time_shift_ns;      /* SolarPosition(time_shift=...), default 0       */
  const double* lon_deg;      /* host, nx   (ds["lon"])                          */
  const double* lat_deg;      /* host, ny   (ds["lat"])                          */
  const double* slope_rad;    /* host, ny (ny*nx if orientation_2d)  orientation(lon,lat,sp)["slope"]   */
  const double* azimuth_rad;  /* host, ny (ny*nx if orientation_2d)  orientation(...)["azimuth"]        */
  int32_t tracking, trigon_model, clearsky_model, irr_branch, albedo_src,
      solar_src, panel_model;
  double altitude_threshold_deg; /* pv/irradiation.py:155, default 1.0         */
  /* Huld: c_temp_amb, c_temp_irrad, r_tmod, r_irradiance, k_1..k_6, inverter_efficiency
   * Bofinger: A, B, C, D, NOCT, Tamb, Intc, Tstd, ta, threshold, inverter_efficiency */
  double panel[16];
  int32_t output;             /* ATL_OUT_*; panel[] is ignored unless ATL_OUT_PANEL */
  double thermal[3];          /* ATL_OUT_SOLAR_THERMAL: c0, c1, t_store in deg C  */
  int32_t pitch;              /* row pitch of the device fields, 0 = nx            */
  int32_t orientation_2d;     /* 1: slope_rad / azimuth_rad vary per cell, (ny, nx) row-major:
                                 an orientation callback (pv/orientation.py:107) that returns
                                 (y, x) arrays */
} AtlPvConfig;

typedef struct { /* device pointers to (nt_slab, ny, nx) slabs; unused = NULL */
  const float* influx_toa;
  const float* influx_direct;
  const float* influx_diffuse;
  const float* influx;
  const float* albedo;
  const float* outflux;
  const float* temperature;
  const float* humidity;
  const void* solar_altitude; /* float or double per solar_src */
  const void* solar_azimuth;
} AtlPvFields;

typedef struct AtlPvOp AtlPvOp;
int atl_pv_create(int device, const AtlPvConfig* cfg, AtlPvOp** op_out);
void atl_pv_destroy(AtlPvOp* op);
/* fused convert + aggregate of slab [t0, t0+nt): out_dev (nt, n_bus) */
int atl_pv_reduce(const AtlPvOp* op, const AtlPlan* plan, const AtlPvFields* f,
                  int64_t t0, int64_t nt, float* out_dev, void* stream);
/* per-cell result (aggregate_time=None, no matrix): out_dev (nt, ny, nx) */
int atl_pv_cells(const AtlPvOp* op, const AtlPvFields* f, int64_t t0, int64_t nt,
                 float* out_dev, void* stream);
/* per-cell NaN-skipping time sum, ACCUMULATED into out_dev (ny, nx) (caller zero-fills);
 * count_dev (ny, nx, may be NULL) accumulates the number of non-NaN steps per cell: the
 * reference's `da.mean("time")` divides by it (convert.py:51-56).  Same for every *_timesum. */
int atl_pv_timesum(const AtlPvOp* op, const AtlPvFields* f, int64_t t0, int64_t nt,
                   float* out_dev, float* count_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Wind: extrapolate_wind_speed + np.interp power curve                */
/* (wind.py:24-128, convert.py:634-662)                                */
/* ------------------------------------------------------------------ */
enum { ATL_WIND_NONE = 0 /* wnd{hub}m present, wind.py:75-78 */,
       ATL_WIND_LOG = 1 /* wind.py:91-102 */, ATL_WIND_POWER = 2 /* wind.py:103-112 */ };

typedef struct {
  int32_t ny, nx;
  int32_t method;
  double from_height, to_height;
  int32_t n_knots;         /* <= 255 */
  const double* V;         /* host, n_knots, non-decreasing (resource.py:346-355) */
  const double* POW_norm;  /* host, n_knots: POW / P  (convert.py:649)            */
  int32_t pitch;           /* row pitch of the device fields, 0 = nx              */
} AtlWindConfig;

typedef struct {
  const float* wnd; /* wnd{from}m, (nt, ny, nx)                           */
  const float* aux; /* roughness (LOG) or wnd_shear_exp (POWER) or NULL   */
} AtlWindFields;

typedef struct AtlWindOp AtlWindOp;
int atl_wind_create(int device, const AtlWindConfig* cfg, AtlWindOp** op_out);
void atl_wind_destroy(AtlWindOp* op);
int atl_wind_reduce(const AtlWindOp* op, const AtlPlan* plan, const AtlWindFields* f,
                    int64_t nt, float* out_dev, void* stream);
int atl_wind_cells(const AtlWindOp* op, const AtlWindFields* f, int64_t nt,
                   float* out_dev, void* stream);
int atl_wind_timesum(const AtlWindOp* op, const AtlWindFields* f, int64_t nt,
                     float* out_dev, float* count_dev, void* stream);

/* The same operators on raw ERA5 variables (CDS short names; the download of
 * datasets/era5.py:104-137): wind speed |(u100, v100)|, roughness fsr (sanitized: < 0 or NaN ->
 * 2e-4) and shear exponent ln(|(u10, v10)| / |(u100, v100)|) / ln(10/100) are derived in-kernel
 * with atl_era5_wind's arithmetic, so the result equals the operator's on what era5.prepare
 * stores.  The operator comes from atl_wind_create: ATL_WIND_NONE reads u100, v100 (hub height
 * 100 m), ATL_WIND_LOG also fsr, ATL_WIND_POWER also u10, v10; LOG / POWER need from_height = 100.
 * Unused fields may be NULL. */
typedef struct {
  const float* u100;
  const float* v100;
  const float* u10;
  const float* v10;
  const float* fsr;
} AtlWindRawFields;

int atl_wind_raw_reduce(const AtlWindOp* op, const AtlPlan* plan, const AtlWindRawFields* f,
                        int64_t nt, float* out_dev, void* stream);
int atl_wind_raw_cells(const AtlWindOp* op, const AtlWindRawFields* f, int64_t nt,
                       float* out_dev, void* stream);
int atl_wind_raw_timesum(const AtlWindOp* op, const AtlWindRawFields* f, int64_t nt,
                         float* out_dev, float* count_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Heat demand: daily mean temperature -> degree days                  */
/* (convert.py:405-418)                                                */
/* ------------------------------------------------------------------ */
typedef struct {
  int32_t ny, nx;
  double threshold_c, a, constant; /* convert.py:413-418 (threshold in deg C) */
  int32_t cooling;                 /* 1: a * (Tmean - threshold), convert.py:475-491 */
  int32_t pitch;                   /* row pitch of the device field, 0 = nx            */
} AtlHeatConfig;

typedef struct AtlHeatOp AtlHeatOp;
int atl_heat_create(int device, const AtlHeatConfig* cfg, AtlHeatOp** op_out);
void atl_heat_destroy(AtlHeatOp* op);
/* day_start_host: n_days+1 offsets into the slab's time steps (calendar-day
 * bins of time+hour_shift, convert.py:408-412); out_dev (n_days, n_bus). */
int atl_heat_reduce(const AtlHeatOp* op, const AtlPlan* plan, const float* temperature_dev,
                    const int64_t* day_start_host, int64_t n_days, float* out_dev,
                    void* stream);
int atl_heat_cells(const AtlHeatOp* op, const float* temperature_dev,
                   const int64_t* day_start_host, int64_t n_days, float* out_dev,
                   void* stream);
int atl_heat_timesum(const AtlHeatOp* op, const float* temperature_dev,
                     const int64_t* day_start_host, int64_t n_days, float* out_dev,
                     float* count_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Pointwise conversions of ONE (time, y, x) field:                    */
/*   y = x + shift;  nan_to_zero: y = 0 where NaN;                     */
/*   poly: d = sink - y, out = c0 + c1 d + c2 d^2  else out = y;       */
/*   out *= cell_scale[y, x] (optional static (ny, nx) field)          */
/* temperature / dewpoint (shift = -273.15), soil temperature          */
/* (+ nan_to_zero), coefficient_of_performance (poly), runoff          */
/* (cell_scale = height): convert.py:292-366, 1028-1034.               */
/* ------------------------------------------------------------------ */
typedef struct {
  int32_t ny, nx;
  double shift;
  int32_t nan_to_zero;
  int32_t poly;
  double sink, c0, c1, c2;
  const float* cell_scale; /* host, ny*nx (unpadded), or NULL */
  int32_t pitch;           /* row pitch of the device field, 0 = nx */
} AtlPointwiseConfig;

typedef struct AtlPointwiseOp AtlPointwiseOp;
int atl_pointwise_create(int device, const AtlPointwiseConfig* cfg, AtlPointwiseOp** op_out);
void atl_pointwise_destroy(AtlPointwiseOp* op);
int atl_pointwise_reduce(const AtlPointwiseOp* op, const AtlPlan* plan, const float* field_dev,
                         int64_t nt, float* out_dev, void* stream);
int atl_pointwise_cells(const AtlPointwiseOp* op, const float* field_dev, int64_t nt,
                        float* out_dev, void* stream);
int atl_pointwise_timesum(const AtlPointwiseOp* op, const float* field_dev, int64_t nt,
                          float* out_dev, float* count_dev, void* stream);
int atl_pointwise_reduce_host(const AtlPointwiseOp* op, const AtlPlan* plan,
                              const float* field_host, int64_t nt, float* out_host,
                              int64_t chunk_steps);
/* atl_pointwise_create with options beyond AtlPointwiseConfig.  clip_min_zero != 0: the input
 * is first clipped at 0 (x < 0 -> 0, NaN stays), as sanitize_runoff (datasets/era5.py:241-246)
 * clips the raw ERA5 runoff `ro`; runoff from ro is then clip_min_zero = 1 with cell_scale =
 * height.  Every pointwise entry point (reduce, cells, timesum, reduce_host) honours it. */
typedef struct {
  AtlPointwiseConfig base;
  int32_t clip_min_zero;
} AtlPointwiseConfigEx;
int atl_pointwise_create_ex(int device, const AtlPointwiseConfigEx* cfg, AtlPointwiseOp** op_out);

/* ------------------------------------------------------------------ */
/* CSP: solar position -> direct irradiation (horizontal | DNI) x        */
/* efficiency(altitude, azimuth) table (convert.py:940-972, csp.py)     */
/* ------------------------------------------------------------------ */
enum { ATL_CSP_PARABOLIC_TROUGH = 0, ATL_CSP_SOLAR_TOWER = 1 };
typedef struct {
  int32_t ny, nx;
  int64_t nt;
  const int64_t* time_ns;      /* host, nt (needed unless the solar position is stored) */
  int64_t time_shift_ns;
  const double* lon_deg;       /* host, nx */
  const double* lat_deg;       /* host, ny */
  int32_t solar_src;           /* ATL_SOLAR_* */
  int32_t technology;          /* ATL_CSP_* */
  double r_irradiance;         /* W/m^2 */
  double dni_altitude_threshold_deg; /* csp.py:18, default 3.75 */
  int32_t n_alt, n_az;         /* efficiency table, each 2..128, product <= 8192 */
  const double* altitude_rad;  /* host, n_alt, increasing */
  const double* azimuth_rad;   /* host, n_az, increasing */
  const double* efficiency;    /* host, n_alt * n_az row-major, p.u. */
  int32_t pitch;               /* row pitch of the device fields, 0 = nx */
} AtlCspConfig;

typedef struct {
  const float* influx_direct;
  const void* solar_altitude; /* float or double per solar_src, or NULL */
  const void* solar_azimuth;
} AtlCspFields;

typedef struct AtlCspOp AtlCspOp;
int atl_csp_create(int device, const AtlCspConfig* cfg, AtlCspOp** op_out);
/* An operator on the raw ERA5 variable: every entry point (reduce, cells, timesum, reduce_host)
 * reads fdir (hourly J m-2 accumulation) in AtlCspFields.influx_direct and derives the direct
 * influx fdir / 3600 clipped at 0 in-kernel, with atl_era5_influx's arithmetic.  Pair a computed
 * solar position with time_shift_ns = -30 min to match the one era5.prepare stores. */
int atl_csp_raw_create(int device, const AtlCspConfig* cfg, AtlCspOp** op_out);
void atl_csp_destroy(AtlCspOp* op);
int atl_csp_reduce(const AtlCspOp* op, const AtlPlan* plan, const AtlCspFields* f, int64_t t0,
                   int64_t nt, float* out_dev, void* stream);
int atl_csp_cells(const AtlCspOp* op, const AtlCspFields* f, int64_t t0, int64_t nt,
                  float* out_dev, void* stream);
int atl_csp_timesum(const AtlCspOp* op, const AtlCspFields* f, int64_t t0, int64_t nt,
                    float* out_dev, float* count_dev, void* stream);
int atl_csp_reduce_host(const AtlCspOp* op, const AtlPlan* plan, const AtlCspFields* f_host,
                        int64_t t0, int64_t nt, float* out_host, int64_t chunk_steps);

/* ------------------------------------------------------------------ */
/* Host-buffer entry points: the call the reference-facing Python API  */
/* makes when the cutout lives in host memory (NumPy / NetCDF).  The   */
/* library streams time slabs through a pinned ring (H2D overlapped    */
/* with the kernels) and returns the (nt, n_bus) result in host memory.*/
/* Synchronous.  chunk_steps <= 0 picks a default.                     */
/* ------------------------------------------------------------------ */
int atl_pv_reduce_host(const AtlPvOp* op, const AtlPlan* plan, const AtlPvFields* f_host,
                       int64_t t0, int64_t nt, float* out_host, int64_t chunk_steps);
int atl_wind_reduce_host(const AtlWindOp* op, const AtlPlan* plan,
                         const AtlWindFields* f_host, int64_t nt, float* out_host,
                         int64_t chunk_steps);
int atl_wind_raw_reduce_host(const AtlWindOp* op, const AtlPlan* plan,
                             const AtlWindRawFields* f_host, int64_t nt, float* out_host,
                             int64_t chunk_steps);
int atl_heat_reduce_host(const AtlHeatOp* op, const AtlPlan* plan,
                         const float* temperature_host, const int64_t* day_start_host,
                         int64_t n_days, float* out_host, int64_t chunk_days);

/* Several reduces of one host-resident cutout from one pass of its time slabs through the ring.
 * The ring carries the union of the jobs' host fields, each array (by host pointer) copied host ->
 * device once per slab however many jobs read it.  Every job keeps the slabs its single-operator
 * call above would stream (`chunk` steps, or days for heat demand; <= 0: that call's default), so
 * its launches, and its result bits, are that call's: a job whose slabs are the ring's reduces the
 * ring slot in place, any other one assembles its slabs from the ring slots in a window of its own
 * (device -> device).  Each output is copied to out_host at the end.  The *_reduce_host calls above
 * are the one-job case of this call. */
enum {
  ATL_JOB_PV = 0,        /* op: AtlPvOp,        fields: AtlPvFields* (host)      */
  ATL_JOB_WIND = 1,      /* op: AtlWindOp,      fields: AtlWindFields*           */
  ATL_JOB_WIND_RAW = 2,  /* op: AtlWindOp,      fields: AtlWindRawFields*        */
  ATL_JOB_CSP = 3,       /* op: AtlCspOp,       fields: AtlCspFields*            */
  ATL_JOB_POINTWISE = 4, /* op: AtlPointwiseOp, fields: the float* field itself  */
  ATL_JOB_HEAT = 5       /* op: AtlHeatOp,      fields: the float* temperature   */
};
typedef struct {
  int32_t kind;              /* ATL_JOB_* */
  const void* op;
  const AtlPlan* plan;
  const void* fields;        /* host arrays of (nt, ny, nx), unpadded */
  int64_t t0;                /* pv, csp: step of the operator's time axis at host step 0 */
  const int64_t* day_start;  /* heat: n_days + 1 ascending step offsets, the last <= nt */
  int64_t n_days;
  int64_t chunk;             /* the job's slab length: steps, or days for heat; <= 0: default */
  float* out_host;           /* (rows, n_bus): one row per day for heat jobs, per step otherwise */
} AtlStreamJob;
typedef struct {
  int64_t h2d_bytes; /* bytes copied host -> device */
  int64_t n_slabs;   /* ring slabs */
} AtlStreamStats;
/* Every job's operator and plan must be on `device` with grid ny x nx (checked before anything is
 * allocated or launched; ATL_ERR_INVALID otherwise).  The ring covers the steps the jobs read, of
 * [0, nt), in slabs of chunk_steps (<= 0: ~192 MiB of the union's input per slab).  stats
 * (optional) reports the host -> device copies.  Synchronous. */
int atl_reduce_host_many(int32_t device, int32_t ny, int32_t nx, int64_t nt, const AtlStreamJob* jobs,
                         int32_t n_jobs, int64_t chunk_steps, AtlStreamStats* stats);

/* Introspection of operator handles (device, grid). */
int atl_pv_op_info(const AtlPvOp* op, int32_t* device, int32_t* ny, int32_t* nx,
                   int32_t* solar_src);
/* Host-only: evaluates the power-curve interpolation exactly as the kernels do
 * (same tables, same fp32 formula), no CUDA needed; the CPU tests compare it with
 * np.interp.  force_mode: -1 = the table atl_wind_create would pick, 0 = binary
 * search, 1 = general bucket LUT, 2 = lattice LUT (knots on a uniform lattice) with the
 * steps added back by compares, 3 = saturating lattice LUT (256 rows, steps folded into
 * the table, no clamps; what -1 picks when the curve qualifies);
 * *mode_out (optional) = the table actually built (a forced LUT mode the curve does
 * not qualify for falls back to 0). */
int atl_wind_curve_eval_host(const double* V, const double* POW_norm, int32_t n_knots,
                             int32_t force_mode, const float* x, int64_t n, float* y_out,
                             int32_t* mode_out);
/* Host-only: which table a power curve gets.  info[0] = table (0 binary search, 1 general
 * LUT, 2 lattice LUT, 3 saturating lattice LUT), info[1] = steps the kernel adds back by compares (0 when the curve has
 * none or they are folded into the lattice table), info[2] = steps in the curve (duplicate
 * knots with different powers), info[3] = bytes staged to shared memory. */
int atl_wind_curve_info_host(const double* V, const double* POW_norm, int32_t n_knots,
                             int32_t force_mode, int32_t info[4]);
int atl_wind_op_info(const AtlWindOp* op, int32_t* device, int32_t* ny, int32_t* nx);
int atl_heat_op_info(const AtlHeatOp* op, int32_t* device, int32_t* ny, int32_t* nx);
int atl_pointwise_op_info(const AtlPointwiseOp* op, int32_t* device, int32_t* ny, int32_t* nx);
int atl_csp_op_info(const AtlCspOp* op, int32_t* device, int32_t* ny, int32_t* nx,
                    int32_t* solar_src);

/* Number of kernel launches issued by this library since load (bench.py's
 * "gpu_launches" evidence). */
int64_t atl_launch_count(void);
/* The atl_*_reduce_host calls keep their pinned staging buffers (used for pageable
 * inputs) for the next call; this frees them. */
void atl_release_host_staging(void);

/* ------------------------------------------------------------------ */
/* Indicator matrix: shapes -> CSR (n_shapes, ny*nx) of covered cell   */
/* fractions (cutout.py:492-515 -> gis.py:104-145 on the regular grid  */
/* of cutout.py:355-376).  SURVEY section 8 f1.                        */
/* ------------------------------------------------------------------ */
typedef struct AtlIndicator AtlIndicator;
/* Grid: cell (iy, ix) is the box of half-width (dx/2, dy/2) about (x0 + ix*dx,
 * y0 + iy*dy); dx, dy > 0.  Shapes: shape s owns rings
 * shape_ring_ptr[s] .. shape_ring_ptr[s+1]-1; ring r owns the vertices
 * ring_ptr[r] .. ring_ptr[r+1]-1 of xy (x, y interleaved, float64, same CRS as the
 * grid; the closing vertex may be repeated or not); ring_is_hole[r] != 0 marks an
 * interior ring.  Ring orientation is free.  All pointers are HOST pointers; the
 * areas are computed on `device`.  Entries are kept when the covered fraction
 * exceeds 1e-10; columns are sorted (iy*nx + ix). */
int atl_indicator_compute(int device, int32_t ny, int32_t nx, double x0, double dx, double y0,
                          double dy, int32_t n_shapes, const int64_t* shape_ring_ptr,
                          const int64_t* ring_ptr, const int8_t* ring_is_hole, const double* xy,
                          AtlIndicator** out);
int atl_indicator_nnz(const AtlIndicator* ind, int64_t* nnz_out);
/* indptr_out[n_shapes+1], indices_out[nnz], data_out[nnz] (host, caller-owned) */
int atl_indicator_export(const AtlIndicator* ind, int64_t* indptr_out, int32_t* indices_out,
                         double* data_out);
void atl_indicator_destroy(AtlIndicator* ind);

/* Overlay: the general form of gis.py:104-145, two polygon collections.  Entry [i, j] of the
 * (n_dest, n_orig) CSR is area(dest_i ∩ orig_j) / area(orig_j), planar, in the units of xy.
 * Both sides use atl_indicator_compute's shape layout (shape_ring_ptr, ring_ptr, ring_is_hole,
 * xy; ring orientation free, closing vertex optional) and the same CRS.  Rings are taken as
 * valid OGC polygons; parts of one shape that overlap count twice.  Pairs that only touch give
 * no entry: shared boundary pieces, vertices on edges and collinear overlaps are decided exactly.
 * Entries are kept when the fraction exceeds 1e-10; columns are sorted; the result is bitwise
 * repeatable.  An orig shape with a ring but no positive area (exteriors minus holes) is refused
 * with ATL_ERR_INVALID before any device work; an orig shape without rings is an empty column.  All
 * pointers are HOST pointers; the work runs on `device`.  The handle is read and freed with
 * atl_indicator_nnz / _export / _destroy. */
int atl_overlay_compute(int device, int32_t n_orig, const int64_t* orig_shape_ring_ptr,
                        const int64_t* orig_ring_ptr, const int8_t* orig_ring_is_hole,
                        const double* orig_xy, int32_t n_dest, const int64_t* dest_shape_ring_ptr,
                        const int64_t* dest_ring_ptr, const int8_t* dest_ring_is_hole,
                        const double* dest_xy, AtlIndicator** out);

/* ------------------------------------------------------------------ */
/* Intersection matrix: shapes -> CSR (n_shapes, ny*nx) with 1.0 where */
/* the shape and the closed cell box intersect (cutout.py:517-537 ->   */
/* gis.py:148-183, shapely `intersects`).                              */
/* ------------------------------------------------------------------ */
#define ATL_PART_EXTERIOR 0 /* polygon exterior ring */
#define ATL_PART_HOLE 1     /* polygon interior ring of the preceding exterior */
#define ATL_PART_LINE 2     /* line path (a one-vertex path is a point) */
#define ATL_PART_POINTS 3   /* every vertex is a point */
/* Grid: the regular grid of atl_indicator_compute (x0, dx, y0, dy) and the boxes the
 * decision is taken against: cell (iy, ix) is [cell_x_lo[ix], cell_x_hi[ix]] x
 * [cell_y_lo[iy], cell_y_hi[iy]] (float64, closed; the reference builds them as
 * x[ix] -/+ (x[1] - x[0]) / 2).  The tables must be finite, ordered and within 1/8
 * cell of the regular grid's borders.  Shapes: shape s owns parts
 * shape_part_ptr[s] .. shape_part_ptr[s+1]-1; part p owns the vertices
 * part_ptr[p] .. part_ptr[p+1]-1 of xy (x, y interleaved) and is of kind
 * part_kind[p] (ATL_PART_*).  A shape is the union of its parts; ring orientation is
 * free and a ring's closing vertex may be repeated or not.  The predicates are exact:
 * points and segments are tested against the closed boxes with exact orientation
 * signs, and a cell no ring edge touches is kept when it lies inside a polygon.  All
 * pointers are HOST pointers; the work runs on `device`.  Columns are sorted
 * (iy*nx + ix).  The handle is read and freed with atl_indicator_nnz / _export /
 * _destroy. */
int atl_intersection_compute(int device, int32_t ny, int32_t nx, double x0, double dx, double y0,
                             double dy, const double* cell_x_lo, const double* cell_x_hi,
                             const double* cell_y_lo, const double* cell_y_hi, int32_t n_shapes,
                             const int64_t* shape_part_ptr, const int64_t* part_ptr,
                             const int8_t* part_kind, const double* xy, AtlIndicator** out);

/* Intersects: the general form of gis.py:148-183, two geometry collections.  Entry [i, j] of
 * the (n_dest, n_orig) CSR is 1.0 when dest_i and orig_j intersect as closed sets (shapely
 * `intersects`): a boundary contact counts.  Both sides use atl_intersection_compute's shape
 * layout (shape_part_ptr, part_ptr, part_kind, xy) and the same CRS.  The point set of a shape
 * is every segment of every part (ring edges including the closing edge, line segments, points
 * as zero-length segments) and the even-odd interior of each polygon, an exterior together with
 * the holes that follow it; a shape is the union of its polygons.  The predicates are exact.
 * Empty shapes give empty rows and columns; columns are sorted; the result is bitwise
 * repeatable.  Every pointer array, part kind and vertex is checked before any device work.  All
 * pointers are HOST pointers; the work runs on `device`.  The handle is read and freed with
 * atl_indicator_nnz / _export / _destroy. */
int atl_intersects_compute(int device, int32_t n_orig, const int64_t* orig_shape_part_ptr,
                           const int64_t* orig_part_ptr, const int8_t* orig_part_kind,
                           const double* orig_xy, int32_t n_dest, const int64_t* dest_shape_part_ptr,
                           const int64_t* dest_part_ptr, const int8_t* dest_part_kind,
                           const double* dest_xy, AtlIndicator** out);

/* ------------------------------------------------------------------ */
/* ERA5 prepare-time derivations (datasets/era5.py:120-201), SURVEY    */
/* section 8 f4.  All field pointers are DEVICE pointers to n float32  */
/* values (any shape); outputs may not alias inputs.                   */
/* ------------------------------------------------------------------ */
/* get_data_wind (era5.py:120-135) [+ sanitize_wind :141-146 if sanitize != 0]:
 * wnd100m = |(u100, v100)|, wnd_shear_exp = ln(|(u10, v10)| / wnd100m) / ln(10/100),
 * wnd_azimuth = atan2(u100, v100) mapped to [0, 2 pi), roughness = fsr (< 0 -> 2e-4). */
int atl_era5_wind(int device, int64_t n, const float* u100, const float* v100, const float* u10,
                  const float* v10, const float* fsr, int32_t sanitize, float* wnd100m,
                  float* wnd_shear_exp, float* wnd_azimuth, float* roughness, void* stream);
/* get_data_influx (era5.py:163-175) [+ sanitize_influx :195-201]: albedo =
 * ((ssrd - ssr) / ssrd, 0 where ssrd == 0 or NaN), influx_diffuse = ssrd - fdir, and
 * influx_{toa, direct, diffuse} converted J m-2 -> W m-2 (/ 3600) [clipped at 0]. */
int atl_era5_influx(int device, int64_t n, const float* ssrd, const float* ssr, const float* tisr,
                    const float* fdir, int32_t sanitize, float* influx_toa, float* influx_direct,
                    float* influx_diffuse, float* albedo, void* stream);
/* SolarPosition (pv/solar_position.py:69-116) materialised as the cutout variables
 * solar_altitude / solar_azimuth (era5.py:182-188 uses time_shift = -30 min):
 * (nt, ny, nx) float64 each, device; time / lon / lat are host arrays. */
int atl_solar_position(int device, const int64_t* time_ns_host, int64_t nt, int64_t time_shift_ns,
                       const double* lon_deg_host, int32_t nx, const double* lat_deg_host, int32_t ny,
                       double* altitude_dev, double* azimuth_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Dynamic line rating (convert.py:1152-1367): IEEE-738 maximal current */
/* per (line, cell, step), NaN-skipping min over each line's cells.    */
/* ------------------------------------------------------------------ */
/* A plan whose per-slot entry lists are on the device whatever its tiling: the
 * line-rating kernel walks them for every plan (fused or not).  Same arguments
 * as atl_plan_create_pitched. */
int atl_plan_create_entries(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus,
                            const int64_t* indptr_host, const int32_t* indices_host,
                            const double* data_host, AtlPlan** plan_out);

typedef struct AtlLineRatingOp AtlLineRatingOp;
typedef struct {
  int32_t ny, nx;
  int32_t pitch;             /* 0 = nx */
  int64_t nt;                /* time axis of the computed solar position */
  const int64_t* time_ns;    /* host, nt entries (solar_src == ATL_SOLAR_COMPUTED) */
  int64_t time_shift_ns;     /* line_rating computes the position at a 0 h shift */
  const double* lon_deg;     /* host, nx */
  const double* lat_deg;     /* host, ny */
  int32_t solar_src;         /* ATL_SOLAR_* as for PV */
  int32_t n_lines;
  /* host, n_lines each: the arguments of convert_line_rating per line.  psi is taken
   * through radians() as the reference does (line_rating passes its azimuth in radians
   * here, so it is converted twice; reproduced). */
  const double *psi, *R, *D, *Ts, *epsilon, *alpha;
} AtlLineRatingConfig;
/* Device fields of one slab: temperature, wnd100m, wnd_azimuth, influx_direct are
 * (nt, ny, pitch) float32, height is (ny, pitch) float32, the stored solar position
 * (nt, ny, pitch) float32 / float64 per solar_src (NULL when computed). */
typedef struct {
  const float *temperature, *wnd100m, *wnd_azimuth, *influx_direct, *height;
  const void *solar_altitude, *solar_azimuth;
} AtlLineRatingFields;
int atl_line_rating_create(int device, const AtlLineRatingConfig* cfg, AtlLineRatingOp** op_out);
void atl_line_rating_destroy(AtlLineRatingOp* op);
/* out_dev (nt, n_lines) float32: per step the min over the line's stored cells of
 * Imax, NaN cells skipped; NaN where no cell is valid or the line has none.  Steps
 * [t0, t0 + nt) of the operator's time axis.  The plan must come from
 * atl_plan_create_entries (one row per line, same grid and pitch).  Bitwise
 * repeatable: the min does not depend on the order of its operands. */
int atl_line_rating_reduce(const AtlLineRatingOp* op, const AtlPlan* plan, const AtlLineRatingFields* f,
                           int64_t t0, int64_t nt, float* out_dev, void* stream);
/* The same reduce on raw ERA5 variables (datasets/era5.py:104-188): t2m, u100, v100, fdir are
 * (nt, ny, pitch) float32 slabs (fdir an hourly J m-2 accumulation).  The wind speed |(u100, v100)|,
 * the wind azimuth atan2(u100, v100) in [0, 2 pi) and the direct influx fdir / 3600 clipped at 0
 * are derived in-kernel with atl_era5_wind / atl_era5_influx's arithmetic, so the result equals
 * atl_line_rating_reduce on what era5.prepare stores.  height and the stored solar position as for
 * AtlLineRatingFields; pair a computed position with time_shift_ns = -30 min to match the position
 * era5.prepare stores (era5.py:182-188). */
typedef struct {
  const float *t2m, *u100, *v100, *fdir, *height;
  const void *solar_altitude, *solar_azimuth;
} AtlLineRatingRawFields;
int atl_line_rating_raw_reduce(const AtlLineRatingOp* op, const AtlPlan* plan, const AtlLineRatingRawFields* f,
                               int64_t t0, int64_t nt, float* out_dev, void* stream);
/* Elementwise convert_line_rating on n values (the reference's dict inputs, broadcast by
 * the caller): every pointer is a DEVICE array of n values; solar altitude / azimuth in
 * radians, psi as for AtlLineRatingConfig. */
typedef struct {
  const float *temperature, *wnd100m, *wnd_azimuth, *influx_direct, *height, *solar_altitude,
      *solar_azimuth;
  const double *psi, *R, *D, *Ts, *epsilon, *alpha;
} AtlLineRatingFlat;
int atl_line_rating_eval(int device, int64_t n, const AtlLineRatingFlat* f, float* out_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Hydro inflow (hydro.py:81-104): basin runoff rolled by each basin's  */
/* travel time and summed per plant.                                    */
/* ------------------------------------------------------------------ */
/* out_dev (n_plants, nt) float64, plant-major:
 *   out[p, t] = sum over e in [entry_ptr[p], entry_ptr[p + 1]) of weights[e] * R[rows[e], (t - shifts[e]) mod nt]
 * with R = runoff_dev, (n_rows, nt) float64 row-major.  shifts may be negative or >= nt (the roll wraps).
 * Each product and sum is rounded separately, in entry order, so the result is that of adding the
 * rolled float64 rows one after another, and it is bitwise repeatable.  A plant with no entries gets
 * 0.  entry_ptr (n_plants + 1), rows (int32, each < n_rows), shifts (int64) and weights (float64) are
 * device arrays.  nt is at most 65535 * 256 steps. */
int atl_hydro_shift_sum(int device, int32_t n_rows, int64_t nt, const double* runoff_dev, int32_t n_plants,
                        const int64_t* entry_ptr_dev, const int32_t* rows_dev, const int64_t* shifts_dev,
                        const double* weights_dev, double* out_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Regridding (gis.py:791-871 regrid, Resampling.average / .nearest in  */
/* one CRS): (batch, ny_src, nx_src) -> (batch, ny_dst, nx_dst).        */
/* ------------------------------------------------------------------ */
/* Separable weights: destination cell (i, j) reads source rows yfirst[i] + k, k < ycount[i], with
 * weight yw[i * ky + k], and source columns xfirst[j] + k with weight xw[j * kx + k] (host tables,
 * copied at create time; indices inside the source grid, counts <= ky / kx).  atl_regrid_f32 / _f64
 * write
 *   out[b, i, j] = sum wy wx v / sum wy wx [v not NaN]   over the non-NaN source values v,
 * and NaN where that weight sum is 0.  Sums are float64 in a fixed order (bitwise repeatable); the
 * result is rounded once to the element type.  The source is row-strided: element (b, r, c) is at
 * src_dev[b * src_batch + r * src_row + c]; out_dev is contiguous.  batch may be 0. */
int atl_regrid_create(int device, int32_t ny_src, int32_t nx_src, int32_t ny_dst, int32_t nx_dst, int32_t ky,
                      const int32_t* yfirst, const int32_t* ycount, const double* yw, int32_t kx,
                      const int32_t* xfirst, const int32_t* xcount, const double* xw, void** out);
/* The launch shape create chose: row bands, column tiles, destination columns per tile and the
 * widest source span a tile reads (any pointer may be NULL). */
int atl_regrid_info(const void* plan, int32_t* n_bands, int32_t* n_ctiles, int32_t* tile_cols, int32_t* max_span);
int atl_regrid_f32(const void* plan, int64_t batch, const float* src_dev, int64_t src_row, int64_t src_batch,
                   float* out_dev, void* stream);
int atl_regrid_f64(const void* plan, int64_t batch, const double* src_dev, int64_t src_row, int64_t src_batch,
                   double* out_dev, void* stream);
/* Source rows [row_lo[b], row_hi[b]) that band b (RG_ROWS = 8 destination rows) reads, for every
 * band (n_bands of atl_regrid_info); 0, 0 for a band that reads none. */
int atl_regrid_band_rows(const void* plan, int32_t* row_lo, int32_t* row_hi);
/* One 2-D window (gebco.py: a terrain grid averaged onto a cutout), bands [band0, band0 + n_bands)
 * of the plan: src_dev holds source rows [row0, row0 + n_rows) (row r at src_dev + (r - row0) *
 * src_row elements, dtype ATL_REGRID_*), and every band must read rows inside it.  The same average
 * as atl_regrid_f32, except that with has_fill values equal to `fill` are skipped like NaN and a
 * cell without a valid value gets `fill` (without: NaN, or 0 for int16); int16 results are rounded
 * half away from zero.  out_dev is the whole (ny_dst, nx_dst) output, contiguous, in the source
 * dtype; only the rows of the given bands are written.  The int16 window is read as it is: no
 * wider copy is made. */
#define ATL_REGRID_I16 0
#define ATL_REGRID_F32 1
#define ATL_REGRID_F64 2
int atl_regrid_window(const void* plan, int32_t dtype, int32_t band0, int32_t n_bands, const void* src_dev,
                      int32_t row0, int32_t n_rows, int64_t src_row, int32_t has_fill, double fill, void* out_dev,
                      void* stream);
/* atl_regrid_f32 / _f64 with nodata (gis.reproject within one CRS), dtype ATL_REGRID_F32 or _F64:
 * with has_nodata, values equal to `nodata` are skipped like NaN, and a cell without a valid value
 * gets `empty` (which may be NaN). */
int atl_regrid_nodata(const void* plan, int32_t dtype, int64_t batch, const void* src_dev, int64_t src_row,
                      int64_t src_batch, int32_t has_nodata, double nodata, double empty, void* out_dev, void* stream);
void atl_regrid_destroy(void* plan);

/* ------------------------------------------------------------------ */
/* SARAH (datasets/sarah.py:91-159 interpolate / fillna(0) /            */
/* hourly_mean): gap filling per time block, then the pair mean.        */
/* ------------------------------------------------------------------ */
/* sis_dev / sid_dev: (nt, n_cells) float32, contiguous.  The steps are cut into n_blocks blocks,
 * block b = [block_start[b], block_start[b + 1]) with block_start[n_blocks] = nt implied
 * (block_start is a host array of n_blocks strictly ascending entries, the first 0).  Per cell and
 * block, with ATL_SARAH_FILL_INTERP: a NaN between the valid steps i0 and i1 becomes np.interp's
 * float64 (f1 - f0) / (i1 - i0) * (s - i0) + f0 rounded to float32, leading / trailing NaNs the first
 * / last valid value, an all-NaN block stays NaN; with ATL_SARAH_FILL_ZERO NaN becomes 0, with
 * ATL_SARAH_FILL_NONE it stays.  With pair_mean the output
 * is (nt / 2, n_cells): step k = (v[2k] + v[2k + 1]) / 2 in float32 (an odd last step is dropped);
 * else (nt, n_cells).  Results are NumPy's bit for bit, NaN payloads aside. */
#define ATL_SARAH_MAX_BLOCKS 512
#define ATL_SARAH_FILL_NONE 0
#define ATL_SARAH_FILL_ZERO 1
#define ATL_SARAH_FILL_INTERP 2
int atl_sarah_fill(int device, int32_t nt, int64_t n_cells, const float* sis_dev, const float* sid_dev, int32_t n_blocks,
                   const int32_t* block_start, int32_t fill, int32_t pair_mean, float* sis_out_dev,
                   float* sid_out_dev, void* stream);

/* ------------------------------------------------------------------ */
/* Land eligibility (gis.py:263-325 shape_availability and the          */
/* aggregation of availabilitymatrix): fine masks on a pixel lattice.   */
/* ------------------------------------------------------------------ */
/* Every pointer is a DEVICE pointer; masks are uint8 (0 / 1), row-major (ny, nx), row 0 at the
 * top.  Pixel (i, j) of a lattice has its centre at x = c + (i + 0.5) * a, y = f + (j + 0.5) * e,
 * each product and sum rounded separately. */
typedef struct {
  double c, a, f, e;
  int64_t nx, ny;
} AtlLattice;
/* EPSG:3035 (LAEA, EPSG method 9820) constants, as atlite_b200/proj.py computes them:
 * s1..s3 the series from authalic to geodetic latitude, newton the Newton steps after it. */
typedef struct {
  double e2, e, qp, rq, sin_b0, cos_b0, d, lam0, fe, fn, s1, s2, s3;
  int32_t newton;
} AtlLaea;
/* A CRS (atlite_b200/proj.py): EPSG:4326, EPSG:3035 (the AtlLaea constants), EPSG:3857 (spherical
 * Mercator) or ESRI:54009 (spherical Mollweide, `newton` Newton steps), the last two on a sphere of
 * radius r. */
#define ATL_CRS_LONLAT 0
#define ATL_CRS_LAEA 1
#define ATL_CRS_MERCATOR 2
#define ATL_CRS_MOLLWEIDE 3
typedef struct {
  int32_t kind;
  int32_t newton;
  double r;
} AtlCrs;
/* A lattice point taken from the lattice's CRS `from` into the CRS `to`: the inverse of `from` to
 * lon / lat, then the forward of `to` (atlite_b200/proj.py device_projection fills it).  A point
 * without an image becomes NaN: it is outside every raster and on no cutout cell. */
typedef struct {
  AtlCrs from, to;
  AtlLaea laea;
} AtlProjection;
#define ATL_MASK_EVEN_ODD 0
#define ATL_MASK_NONZERO 1

/* The lattices of the atl_avail_* entry points have a > 0 and e < 0.
 *
 * Polygon mask: out[j, i] = inside(centre) ^ flip on the rows lat_row0 .. lat_row0 + lat->ny - 1
 * of the lattice (c, a, f, e): pixel (i, j) of it has the centre of lattice row lat_row0 + j, and
 * edge rows (row0[e]) count from lat_row0 too.  edges (n_edges, 4) float64 x1, y1, x2, y2;
 * edge_w (n_edges) int32: 1 for even-odd, the ring's orientation sign (+1 exterior counter-
 * clockwise / hole clockwise, else -1) for nonzero winding.  An edge crosses row j when
 * (y1 > cy) != (y2 > cy); it counts for the centres strictly left of it (exact orient2d sign).
 * Edge e is tested on rows row0[e] .. row0[e] + (pair_ptr[e + 1] - pair_ptr[e]) - 1 (pair_ptr
 * int64, n_edges + 1, pair_ptr[0] = 0; a superset of the rows it crosses is fine).  cnt (ny * nx
 * int32) is scratch. */
int atl_avail_mask(int device, const AtlLattice* lat, int64_t lat_row0, int64_t n_edges, const double* edges,
                   const int32_t* edge_w, const int64_t* pair_ptr, const int32_t* row0, int32_t* cnt, uint8_t* out,
                   int32_t mode, int32_t flip, void* stream);

/* Raster sample (nearest): for each window pixel the raster pixel under its centre (projected by
 * `proj` first), read as nodata when it lies outside the raster or its own centre is outside the
 * shape (mask over the raster pixels [mask_i0, mask_i0 + mask_nx) x [mask_j0, ...), NULL: none is),
 * else lut[idx].  Result: ex_nodata or lut[idx] (0 / 1), written to out, or OR-ed into it.
 * Window row j has the centre of lattice row win_row0 + j (a band of rows of a larger window). */
typedef struct {
  AtlLattice win, ras;
  AtlProjection proj; /* win's CRS -> ras's CRS */
  const void* idx; /* (ras.ny, ras.nx) LUT indices, uint8 (idx_bytes 1) or int32 (4) */
  int32_t idx_bytes;
  const uint8_t* mask;
  int64_t mask_i0, mask_j0, mask_nx, mask_ny;
  const uint8_t* lut;
  int32_t ex_nodata;
  int32_t or_into;
  uint8_t* out;
  int64_t win_row0;
} AtlRasterSample;
int atl_avail_raster_sample(int device, const AtlRasterSample* s, void* stream);

/* excl |= (L1 distance to a pixel with src != 0, within the (ny, nx) window) <= k: src dilated
 * k times with the 4-connected cross, border 0.  rowdist (ny * nx int32) is scratch. */
int atl_avail_dilate(int device, int64_t ny, int64_t nx, int32_t k, const uint8_t* src, int32_t* rowdist,
                     uint8_t* excl, void* stream);

/* Geometry exclusion on a window: near = distance from the centre to a segment <= |buffer|,
 * in = inside (uint8 mask, NULL: nowhere).  buffer >= 0: ex = in | near; buffer < 0: ex = in & !near;
 * invert: ex = !ex.  excl |= ex.  Segments segs (n_segs, 4) float64 (a point is a zero-length one)
 * are binned to tiles of ATL_AVAIL_TILE x ATL_AVAIL_TILE pixels: phase 0 counts into tile_cnt
 * (n_tiles int32, zeroed by the caller), phase 1 fills tile_list from tile_cursor (n_tiles int64,
 * the exclusive prefix sum of the counts) and leaves tile_cursor[t] at the end of tile t's list;
 * atl_avail_geometry then reads tile t's segments from tile_ptr[t] (n_tiles + 1 int64). */
#define ATL_AVAIL_TILE 16
typedef struct {
  AtlLattice win;
  const double* segs;
  int64_t n_segs;
  double buffer;
  int32_t invert;
  const uint8_t* inside;
  int32_t* tile_cnt;
  int64_t* tile_cursor;
  const int64_t* tile_ptr;
  int32_t* tile_list;
  uint8_t* excl;
} AtlGeomExclusion;
/* Both work on rows win_row0 .. win_row0 + win.ny - 1 of the lattice win: pixel (i, j) has the
 * centre of lattice row win_row0 + j; tiles, inside and excl are relative to the band. */
int atl_avail_geom_bin(int device, const AtlGeomExclusion* g, int64_t win_row0, int32_t phase, void* stream);
int atl_avail_geometry(int device, const AtlGeomExclusion* g, int64_t win_row0, void* stream);

/* counts[iy * gnx + ix] += number of pixels with excl == 0 whose centre (projected by `proj`)
 * lies in cell ix = floor((x - gx0) / gdx), iy = floor((y - gy0) / gdy) of the (gny, gnx) grid;
 * centres off the grid are dropped.  Exact integer counts: bitwise repeatable.  Window row j has the
 * centre of lattice row win_row0 + j, as in AtlRasterSample. */
typedef struct {
  AtlLattice win;
  AtlProjection proj; /* win's CRS -> the cutout's CRS */
  const uint8_t* excl;
  double gx0, gdx, gy0, gdy;
  int64_t gnx, gny;
  unsigned long long* counts;
  int64_t win_row0;
} AtlAvailCount;
int atl_avail_count(int device, const AtlAvailCount* c, void* stream);

/* Reprojected availability (ExclusionContainer.compute_shape_availability with dst_*): the eligible
 * share of the cells of the grid dst, from a window win (its CRS; a > 0, e < 0) padded with `pad`
 * pixels of value 0 on every side.  Cell (i, j)'s box is gis.reproject's average footprint (dst's
 * corners (j, i) and (j + 1, i + 1), either sign of a and e, projected by `proj` and taken to window
 * pixel coordinates), clipped to [-pad, n + pad) along each axis.  Along an axis the box's pixels are
 * first (weight w_lo), interior (1) and last (w_hi); N_ab counts the eligible (excl == 0) window pixels
 * of row class a and column class b, and the value is
 *   (wy_f S_f + S_i + wy_l S_l) / (Wy Wx),  S_a = wx_f N_af + N_ai + wx_l N_al,
 *   Wx = w_lo + w_hi + (m - 2) for an m-pixel span (w_lo for m = 1),
 * in float64, left to right, each product and sum rounded.  An empty box, or a corner without an
 * image, gives 0.  Per shape: atl_avail_average_rect finds the rectangle of cells with a non-empty
 * box; atl_avail_average_counts adds each band's counts to those cells; atl_avail_average_finalize
 * writes their values.  Counts are exact integers, so the result does not depend on the bands. */
typedef struct {
  AtlLattice win, dst;
  AtlProjection proj;             /* dst's CRS -> win's CRS */
  int64_t pad;                    /* zero pixels around the window, >= 0 */
  int32_t row0, col0, row1, col1; /* the rectangle [row0, row1) x [col0, col1) of dst cells covered */
  int32_t tile_y, tile_x;         /* the counting kernel's CTA tile of cells (product in [1, 256]),
                                     a launch shape only */
} AtlAvailAverage;
/* rect_host[4] = (row0, col0, row1, col1) bounding the cells with a non-empty box, (0, 0, 0, 0)
 * when there is none; rect_dev is 4 int32 of device scratch.  Reads no pixels.  Synchronous. */
int atl_avail_average_rect(int device, const AtlAvailAverage* a, int32_t* rect_dev, int32_t* rect_host,
                           void* stream);
/* counts ((row1 - row0) * (col1 - col0) * 9 int64, cell-major, N_ab at 3 a + b; zeroed by the caller
 * before the first band) += the counts of the band excl (band_ny rows of win.nx pixels, window rows
 * band_row0 .. band_row0 + band_ny - 1, 0 / 1) for the cells of a's rectangle. */
int atl_avail_average_counts(int device, const AtlAvailAverage* a, const uint8_t* excl, int64_t band_row0,
                             int64_t band_ny, int64_t* counts, void* stream);
/* out ((row1 - row0) * (col1 - col0) float64, row-major) = the values of the rectangle's cells. */
int atl_avail_average_finalize(int device, const AtlAvailAverage* a, const int64_t* counts, double* out,
                               void* stream);
/* uv ((dst.ny + 1) * (dst.nx + 1) * 2 float64) = the window pixel coordinates (u, v) of dst's lattice
 * points (col, row), row-major, NaN without an image: the corners the three calls above use. */
int atl_avail_average_corners(int device, const AtlAvailAverage* a, double* uv, void* stream);

/* ------------------------------------------------------------------ */
/* Reprojection (gis.reproject, rasterio.warp.reproject with            */
/* Resampling.average / .nearest) across the CRSs above.                */
/* ------------------------------------------------------------------ */
/* (batch, src.ny, src.nx) -> (batch, dst.ny, dst.nx).  Axis-aligned lattices of either sign of a
 * and e: the corner (col, row) of a grid is at x = c + col * a, y = f + row * e.  Destination points
 * are projected into the source CRS by `proj`.
 * average: the cell's corners (j, i) and (j + 1, i + 1) span the source box whose pixels are
 * averaged with separable overlap weights (overlaps <= 1e-10 pixels left out, clipped to the source);
 * nearest: the pixel floor(u, v) under the projected centre (j + 1/2, i + 1/2).  NaN and, with
 * has_nodata, src_nodata are skipped; a cell without a valid pixel or without an image gets
 * dst_nodata (which may be NaN).  tile_y x tile_x (product in [1, 256]) is the average kernel's CTA
 * tile of destination cells, a launch shape only.  Sums are float64 in an order fixed by the geometry:
 * bitwise repeatable.  The source is row-strided (element (b, r, c) at src_dev[b * src_batch + r *
 * src_row + c]) and dtype ATL_REGRID_F32 or _F64; out_dev is contiguous.  batch may be 0.
 * The statistics take the average's box and pixel weights w = w_v * w_u (DESIGN.md section 1):
 * sum = sum w v; rms = sqrt(sum w v^2 / sum w); min / max = the smallest / largest valid value (-0.0
 * below +0.0), bit for bit; med, q1, q3 = the smallest valid x with 4 C(x) >= k W (k = 2, 1, 3) and
 * mode = the value of the largest W, ties to the smaller value, where q = llround(w 2^40), W = sum q,
 * C(x) = sum q of the valid values <= x and -0.0 counts as +0.0 (exact in any order); W = 0 gives
 * dst_nodata.  The selections (med, q1, q3, mode) allocate device scratch from the stream's pool. */
#define ATL_RESAMPLING_NEAREST 0
#define ATL_RESAMPLING_AVERAGE 5
#define ATL_RESAMPLING_MODE 6
#define ATL_RESAMPLING_MAX 8
#define ATL_RESAMPLING_MIN 9
#define ATL_RESAMPLING_MED 10
#define ATL_RESAMPLING_Q1 11
#define ATL_RESAMPLING_Q3 12
#define ATL_RESAMPLING_SUM 13
#define ATL_RESAMPLING_RMS 14
typedef struct {
  AtlLattice src, dst;
  AtlProjection proj; /* dst's CRS -> src's CRS */
  int32_t resampling;
  int32_t has_nodata;
  double src_nodata, dst_nodata;
  int32_t tile_y, tile_x;
} AtlReproject;
int atl_reproject(int device, const AtlReproject* r, int32_t dtype, int64_t batch, const void* src_dev,
                  int64_t src_row, int64_t src_batch, void* out_dev, void* stream);
/* One axis of a box: pixels [lo, hi) (empty: hi <= lo), the first weighted w_lo, the last w_hi and
 * every pixel between them 1. */
typedef struct {
  int32_t lo, hi;
  double w_lo, w_hi;
} AtlSpan;
/* atl_reproject with options for every resampling but nearest; b = NULL is atl_reproject.
 * row_spans / col_spans (host arrays of dst.ny / dst.nx, both or neither): cell (i, j) takes the box
 * row_spans[i] x col_spans[j] instead of its two-corner box (regrid's tables within one CRS; proj is
 * then unused), spans inside [0, src.ny) / [0, src.nx) with finite positive weights.  The selections
 * take boxes of at most select_small pixels (< 0: 32, at most 32) with the cell's own thread and
 * sort the larger ones in device scratch of about scratch_bytes (<= 0: 1 GiB; at least one cell's
 * box), in bands of destination cells and slabs of the batch. */
typedef struct {
  const AtlSpan* row_spans;
  const AtlSpan* col_spans;
  int64_t scratch_bytes;
  int32_t select_small;
  int32_t reserved;
} AtlReprojectOptions;
int atl_reproject_ex(int device, const AtlReproject* r, const AtlReprojectOptions* o, int32_t dtype, int64_t batch,
                     const void* src_dev, int64_t src_row, int64_t src_batch, void* out_dev, void* stream);

/* ------------------------------------------------------------------ */
/* GeoTIFF segments (atlite_b200/geotiff.py): one band decoded into a   */
/* device raster.                                                       */
/* ------------------------------------------------------------------ */
#define ATL_TIFF_NONE 1    /* Compression tag values */
#define ATL_TIFF_LZW 5
#define ATL_TIFF_DEFLATE 8 /* 8 and 32946 */
/* per-segment status of the LZW decode */
#define ATL_TIFF_OK 0
#define ATL_TIFF_LZW_TRUNCATED 1 /* the stream ends before the segment is complete */
#define ATL_TIFF_LZW_BAD_CODE 2  /* a code above the next free code */
#define ATL_TIFF_LZW_LONG 3      /* more output than the segment holds */
#define ATL_TIFF_LZW_SHORT 4     /* EOI before the segment is complete */
#define ATL_TIFF_LZW_OLD_STYLE 5 /* pre-6.0 LZW (first bytes 0x00, odd): refused as libtiff's check finds it */
typedef struct {
  int32_t compression;   /* ATL_TIFF_NONE / _LZW / _DEFLATE */
  int32_t predictor;     /* 1 none, 2 horizontal differencing, 3 floating point (libtiff's fpAcc) */
  int32_t sample_bytes;  /* 1, 2, 4 or 8 */
  int32_t big_endian;    /* the file is "MM" */
  int32_t tiled;         /* 1: tiles of seg_w x seg_h, 0: strips of seg_h rows (seg_w = width) */
  int64_t width, height; /* image */
  int64_t seg_w, seg_h;
  int64_t win_r0, win_c0, win_ny, win_nx; /* the window of the image the result holds */
} AtlTiffLayout;
typedef struct {
  int64_t segments;     /* segments decoded */
  int64_t stored_bytes; /* bytes read from the file */
  int64_t xfer_bytes;   /* bytes copied host -> device */
  int64_t batches;
} AtlTiffStats;
/* Decode segments seg_index[k] (row-major segment numbers of the file; file_offset[k] and
 * stored_bytes[k] from its StripOffsets / TileOffsets and byte counts) into out_dev, the (win_ny,
 * win_nx) window, row-major, of the image's native-endian samples.  Segments go to the device in
 * batches of at most batch_bytes transfer bytes (and decoded bytes, for LZW; one segment at least),
 * read with n_threads host threads (0: one per CPU, at most 64); the next batch is read and copied
 * while the current one decodes.  Device scratch: two batches of transfer bytes, two of decoded
 * bytes for LZW, and 4 bytes per segment.  Synchronous: returns when out_dev is complete.  A
 * corrupt segment returns ATL_ERR_INVALID with *bad_segment its segment number (else -1) and the
 * reason in atl_last_error(). */
int atl_geotiff_read(int device, const char* path, const AtlTiffLayout* layout, int64_t n_segs,
                     const int64_t* seg_index, const int64_t* file_offset, const int64_t* stored_bytes,
                     int64_t batch_bytes, int32_t n_threads, void* out_dev, int64_t* bad_segment,
                     AtlTiffStats* stats, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ATLITE_B200_H */
