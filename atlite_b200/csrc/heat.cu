// heat.cu -- degree-day heat demand fused with the shape reduce
// (convert.py:405-418): daily mean of `temperature` over calendar-day bins of
// (time + hour_shift), a * (threshold + 273.15 - Tmean), clip(min=0), + constant.
//
// Algorithmic traffic: 4 B per cell-timestep; output has one row per DAY.
#include <vector>

#include "kernels.cuh"

#ifndef ATL_HEAT_PREFETCH
#define ATL_HEAT_PREFETCH 0  // experiment knob (tools/build_variants.sh): L2 prefetch of the next day
#endif

namespace atl {

struct HeatParams {
  const float* temp;
  const int32_t* day_start;  // device, n_days + 1 step offsets
  int32_t base;              // subtracted from day_start[] -> offsets relative to `temp`
  int64_t S;
  int nx;
  float thr_k, a, constant;
  int cooling;  // 1: a * (Tmean - threshold)   (convert.py:475-491)
};

constexpr int HEAT_UNROLL = 6;
constexpr int HEAT_STAGE = 8;  // days a warp parks in shared memory before one reduce phase

// One chunk of up to HEAT_UNROLL consecutive time steps for the lane's 4 cells.
template <bool VEC>
__device__ __forceinline__ void heat_load_chunk(const HeatParams& hp, const TileGeomT<VEC>& g, int s,
                                                int s1, float (&x)[HEAT_UNROLL][4]) {
#pragma unroll
  for (int u = 0; u < HEAT_UNROLL; ++u) {
    if (s + u < s1) {
      load4(hp.temp, (int64_t)(s + u) * (hp.S * 4), g, x[u]);
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r) x[u][r] = __int_as_float(0x7fc00000);  // NaN: skipped
    }
  }
}

// daily mean + degree-day formula for the lane's 4 cells of day d.  The loads of
// chunk k+1 are issued before chunk k is accumulated (register double buffer).
// `s_last` = number of steps of the slab (L2 prefetch of the NEXT day's steps stops there).
template <bool VEC>
__device__ __forceinline__ void heat_day(const HeatParams& hp, const TileGeomT<VEC>& g, int d,
                                         float (&v)[4], int s_last) {
  const int s0 = __ldg(hp.day_start + d) - hp.base, s1 = __ldg(hp.day_start + d + 1) - hp.base;
  float sum[4] = {0.f, 0.f, 0.f, 0.f}, cnt[4] = {0.f, 0.f, 0.f, 0.f};
  float x[HEAT_UNROLL][4], y[HEAT_UNROLL][4];
  heat_load_chunk(hp, g, s0, s1, x);
#if ATL_HEAT_PREFETCH
  {  // the next day's slabs go to L2 while this day is summed (no registers: the kernel is latency-bound)
    const int e = min(s1 + (s1 - s0), s_last);
#pragma unroll 4
    for (int s = s1; s < e; ++s) prefetch4_l2(hp.temp, (int64_t)s * (hp.S * 4), g);
  }
#endif
#pragma unroll 1
  for (int s = s0; s < s1; s += HEAT_UNROLL) {
    const bool more = s + HEAT_UNROLL < s1;
    if (more) heat_load_chunk(hp, g, s + HEAT_UNROLL, s1, y);
#pragma unroll
    for (int u = 0; u < HEAT_UNROLL; ++u)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const bool ok = x[u][r] == x[u][r];  // resample(...).mean() skips NaN
        sum[r] += ok ? x[u][r] : 0.f;
        cnt[r] += ok ? 1.f : 0.f;
      }
    if (more) {
#pragma unroll
      for (int u = 0; u < HEAT_UNROLL; ++u)
#pragma unroll
        for (int r = 0; r < 4; ++r) x[u][r] = y[u][r];
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float mean = sum[r] / cnt[r];  // empty bin -> NaN, as xarray
    float h = hp.a * (hp.cooling ? (mean - hp.thr_k) : (hp.thr_k - mean));  // convert.py:413-414 / 484-485
    h = (h == h) ? fmaxf(h, 0.f) : h;    // .clip(min=0) keeps NaN  :416
    h = hp.constant + h;                 // :418
    v[r] = h;
  }
}

// MODE 0: fused reduce -> out (n_days, n_bus); 1: cells -> out (n_days, ny, nx);
// MODE 2: per-cell sum over days accumulated into out (ny, nx), and the number of non-NaN
// days into cnt_out (may be NULL)
template <int MODE, bool VEC>
__global__ void __launch_bounds__(CTA_THREADS, 6)  // latency-bound (ncu: long_scoreboard): 24 warps per SM
    k_heat(const HeatParams hp, const GridDev gd, const PlanDev plan, float* __restrict__ out,
           float* __restrict__ cnt_out, int n_days, int db) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ai = blockIdx.x * WARPS_PER_CTA + warp;
  int tile, s_beg = 0, s_end = 0;
  if (MODE == 0) {
    if (ai >= plan.n_active) return;
    tile = __ldg(plan.active_tiles + ai);
    s_beg = __ldg(plan.tile_slot_ptr + tile);
    s_end = __ldg(plan.tile_slot_ptr + tile + 1);
  } else {
    if (ai >= gd.n_tx * gd.n_ty) return;
    tile = ai;
  }
  const TileGeomT<VEC> g = make_geom<VEC>(tile, lane, gd);
  const int d0 = blockIdx.y * db, d1 = min(n_days, d0 + db);
  const int s_last = ATL_HEAT_PREFETCH ? __ldg(hp.day_start + n_days) - hp.base : 0;
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, cnt[4] = {0.f, 0.f, 0.f, 0.f};
  float v[4];
  if (MODE == 0) {
    // daily values of HEAT_STAGE days are parked in shared memory, then reduced with the lanes
    // along the days (kernels.cuh: staged_reduce); NaN days poison exactly the buses whose
    // stored entries meet them
    extern __shared__ __align__(16) float smem[];
    char* const stage = reinterpret_cast<char*>(smem) + warp * StageT<HEAT_STAGE>::kWarpBytes;
    stage_init<HEAT_STAGE>(stage, lane);
    const bool cached = tile_cache_load<HEAT_STAGE>(stage, plan, s_beg, s_end, lane);
    for (int dc = d0; dc < d1; dc += HEAT_STAGE) {
      const int n = min(HEAT_STAGE, d1 - dc);
      for (int k = 0; k < n; ++k) {
        heat_day(hp, g, dc + k, v, s_last);
        zero_invalid(g, v);
        stage_store1<HEAT_STAGE>(stage, lane, k, v);
      }
      __syncwarp();
      staged_reduce<HEAT_STAGE>(stage, plan, s_beg, s_end, out, dc, n, lane, cached);
      __syncwarp();
    }
    return;
  }
  for (int d = d0; d < d1; ++d) {
    heat_day(hp, g, d, v, s_last);
    if (MODE == 1) {
      store4(out + (int64_t)d * gd.S_out, gd, g, v);
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const bool ok = v[r] == v[r];
        acc[r] += ok ? v[r] : 0.f;
        cnt[r] += ok ? 1.f : 0.f;
      }
    }
  }
  if (MODE == 2) {
    atomic_add4(out, gd, g, acc);
    if (cnt_out) atomic_add4(cnt_out, gd, g, cnt);
  }
}

// Phys adaptor used only by the two-pass fallback (never on the fused path).
}  // namespace atl

using namespace atl;

struct AtlHeatOp {
  int device;
  GridDev grid;
  float thr_k, a, constant;
  int cooling;  // 1: a * (Tmean - threshold)   (convert.py:475-491)
};

static int upload_days(const int64_t* day_start, int64_t n_days, int32_t** d_out,
                       cudaStream_t st) {
  std::vector<int32_t> ds((size_t)n_days + 1);
  for (int64_t i = 0; i <= n_days; ++i) {
    ATL_REQUIRE(day_start[i] >= 0 && day_start[i] < (1LL << 31), "day offset out of range");
    ATL_REQUIRE(i == 0 || day_start[i] >= day_start[i - 1], "day offsets not monotone");
    ds[(size_t)i] = (int32_t)day_start[i];
  }
  ATL_CUDA(cudaMallocAsync((void**)d_out, ds.size() * 4, st));
  // pageable source: the copy is staged before the call returns
  ATL_CUDA(cudaMemcpyAsync(*d_out, ds.data(), ds.size() * 4, cudaMemcpyHostToDevice, st));
  ATL_CUDA(cudaStreamSynchronize(st));
  return ATL_OK;
}

namespace atl {
// Core launcher: `d_days` is a DEVICE table of n_days+1 step offsets, `base` is
// subtracted from every entry (so a slab can index into a table uploaded once
// for the whole time axis; see host_stream.cu).
int heat_launch_core(int mode, const AtlHeatOp* op, const AtlPlan* plan, const float* temp,
                     const int32_t* d_days, int32_t base, const int64_t* day_start_host,
                     int64_t n_days, float* out, cudaStream_t st, float* cnt_out) {
  ATL_REQUIRE(op && temp && out, "NULL argument");
  ATL_REQUIRE(n_days >= 0 && n_days < (1LL << 31), "bad day count");
  if (n_days == 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(op->device));
  PlanDev pd{};
  int gx;
  float* det_acc = nullptr;
  if (mode == 0) {
    ATL_REQUIRE(plan, "NULL plan");
    ATL_REQUIRE(plan->grid.nx == op->grid.nx && plan->grid.ny == op->grid.ny &&
                    plan->grid.pitch == op->grid.pitch,
                "plan / operator grid (or pitch) mismatch");
    ATL_CUDA(cudaMemsetAsync(out, 0, (size_t)n_days * plan->n_bus * sizeof(float), st));
    if (plan->fused) {
      if (plan->n_active == 0) return ATL_OK;
      pd = plan->dev();
      gx = (plan->n_active + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
      if (deterministic()) {  // see launch_fused: one writer per (slot, day), fixed-order gather
        ATL_CUDA(cudaMallocAsync((void**)&det_acc, (size_t)n_days * plan->n_slots * sizeof(float), st));
        ATL_CUDA(cudaMemsetAsync(det_acc, 0, (size_t)n_days * plan->n_slots * sizeof(float), st));
        pd = plan->dev_partial();
      }
    } else {
      // two-pass fallback: per-cell daily values, then CSR gather
      ATL_REQUIRE(day_start_host, "two-pass fallback needs the host day table");
      float* scratch = nullptr;
      const int64_t S = op->grid.S_out;  // unpadded scratch cube
      int64_t blk = (256LL << 20) / (S * 4);
      blk = blk < 1 ? 1 : (blk > n_days ? n_days : blk);
      ATL_CUDA(cudaMallocAsync((void**)&scratch, (size_t)blk * S * 4, st));
      int rc = ATL_OK;
      for (int64_t d = 0; d < n_days && rc == ATL_OK; d += blk) {
        const int64_t n = n_days - d < blk ? n_days - d : blk;
        rc = heat_launch_core(1, op, nullptr, temp + (day_start_host[d] - base) * op->grid.S, d_days + d,
                              (int32_t)day_start_host[d], nullptr, n, scratch, st, nullptr);
        if (rc == ATL_OK)
          rc = launch_csr_spmm(plan, scratch, n, out + (size_t)d * plan->n_bus, st);
      }
      cudaFreeAsync(scratch, st);
      return rc;
    }
  } else {
    gx = (op->grid.n_tx * op->grid.n_ty + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
  }
  HeatParams hp;
  hp.temp = temp;
  hp.day_start = d_days;
  hp.base = base;
  hp.S = op->grid.S;
  hp.nx = op->grid.nx;
  hp.thr_k = op->thr_k;
  hp.a = op->a;
  hp.constant = op->constant;
  hp.cooling = op->cooling;
  const int64_t want = (int64_t)sm_count() * 4 * 8;
  int db = (int)((n_days * gx + want - 1) / want);
  db = db < 1 ? 1 : (db > 8 ? 8 : db);
  size_t smem = 0;
  if (mode == 0) {  // whole staging chunks per block
    db = HEAT_STAGE;
    smem = StageT<HEAT_STAGE>::kCtaBytes;
  }
  dim3 grid(gx, (unsigned)((n_days + db - 1) / db));
  // lane layout: the plan's for the fused reduce, else by grid width / alignment
  const bool al = aligned16(temp);
  GridDev gdo = op->grid;
  gdo.out_vec = (mode == 1 && gdo.nx % 4 == 0 && aligned16(out)) ? 1 : 0;
  bool vec = op->grid.pitch % 4 == 0 && al;
  if (mode == 0) {
    vec = plan->vec;
    ATL_REQUIRE(!vec || al,
                "field pointers must be 16-byte aligned (pitch % 4 == 0 uses 128-bit loads)");
  }
  if (vec) {
    if (mode == 0)
      k_heat<0, true><<<grid, CTA_THREADS, smem, st>>>(hp, gdo, pd, det_acc ? det_acc : out, nullptr, (int)n_days, db);
    else if (mode == 1)
      k_heat<1, true><<<grid, CTA_THREADS, 0, st>>>(hp, gdo, pd, out, nullptr, (int)n_days, db);
    else
      k_heat<2, true><<<grid, CTA_THREADS, 0, st>>>(hp, gdo, pd, out, cnt_out, (int)n_days, db);
  } else {
    if (mode == 0)
      k_heat<0, false><<<grid, CTA_THREADS, smem, st>>>(hp, gdo, pd, det_acc ? det_acc : out, nullptr, (int)n_days, db);
    else if (mode == 1)
      k_heat<1, false><<<grid, CTA_THREADS, 0, st>>>(hp, gdo, pd, out, nullptr, (int)n_days, db);
    else
      k_heat<2, false><<<grid, CTA_THREADS, 0, st>>>(hp, gdo, pd, out, cnt_out, (int)n_days, db);
  }
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  if (det_acc) {
    int rc = launch_gather_slots(plan, det_acc, n_days, out, st);
    cudaFreeAsync(det_acc, st);
    return rc;
  }
  return ATL_OK;
}

int heat_upload_days(const int64_t* day_start, int64_t n_days, int32_t** d_out,
                     cudaStream_t st) {
  return upload_days(day_start, n_days, d_out, st);
}
}  // namespace atl

static int heat_launch(int mode, const AtlHeatOp* op, const AtlPlan* plan, const float* temp,
                       const int64_t* day_start, int64_t n_days, float* out, cudaStream_t st,
                       float* cnt_out = nullptr) {
  ATL_REQUIRE(op && temp && day_start && out, "NULL argument");
  if (n_days <= 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(op->device));
  int32_t* d_days = nullptr;
  int rc = upload_days(day_start, n_days, &d_days, st);
  if (rc) return rc;
  rc = heat_launch_core(mode, op, plan, temp, d_days, 0, day_start, n_days, out, st, cnt_out);
  cudaFreeAsync(d_days, st);
  return rc;
}

extern "C" {

int atl_heat_create(int device, const AtlHeatConfig* cfg, AtlHeatOp** op_out) {
  ATL_REQUIRE(cfg && op_out, "NULL argument");
  *op_out = nullptr;
  ATL_REQUIRE(cfg->ny > 0 && cfg->nx > 0, "bad grid");
  AtlHeatOp* op = new AtlHeatOp();
  op->device = device;
  ATL_REQUIRE(cfg->pitch == 0 || cfg->pitch >= cfg->nx, "pitch must be >= nx");
  op->grid = make_grid(cfg->ny, cfg->nx, cfg->pitch);
  // the reference adds 273.15 in float64 and then meets the float32 field
  // (weak python scalar -> float32): convert.py:413-414
  op->thr_k = (float)(cfg->threshold_c + 273.15);
  op->a = (float)cfg->a;
  op->constant = (float)cfg->constant;
  op->cooling = cfg->cooling ? 1 : 0;
  *op_out = op;
  return ATL_OK;
}

void atl_heat_destroy(AtlHeatOp* op) { delete op; }

int atl_heat_op_info(const AtlHeatOp* op, int32_t* device, int32_t* ny, int32_t* nx) {
  ATL_REQUIRE(op, "NULL argument");
  if (device) *device = op->device;
  if (ny) *ny = op->grid.ny;
  if (nx) *nx = op->grid.nx;
  return ATL_OK;
}

int atl_heat_reduce(const AtlHeatOp* op, const AtlPlan* plan, const float* temperature_dev,
                    const int64_t* day_start_host, int64_t n_days, float* out_dev,
                    void* stream) {
  return heat_launch(0, op, plan, temperature_dev, day_start_host, n_days, out_dev,
                     (cudaStream_t)stream);
}
int atl_heat_cells(const AtlHeatOp* op, const float* temperature_dev,
                   const int64_t* day_start_host, int64_t n_days, float* out_dev, void* stream) {
  return heat_launch(1, op, nullptr, temperature_dev, day_start_host, n_days, out_dev,
                     (cudaStream_t)stream);
}
int atl_heat_timesum(const AtlHeatOp* op, const float* temperature_dev,
                     const int64_t* day_start_host, int64_t n_days, float* out_dev,
                     float* count_dev, void* stream) {
  return heat_launch(2, op, nullptr, temperature_dev, day_start_host, n_days, out_dev,
                     (cudaStream_t)stream, count_dev);
}

}  // extern "C"
