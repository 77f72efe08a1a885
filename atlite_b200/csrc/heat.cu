// heat.cu -- degree-day heat demand fused with the shape reduce
// (convert.py:405-418): daily mean of `temperature` over calendar-day bins of
// (time + hour_shift), a * (threshold + 273.15 - Tmean), clip(min=0), + constant.
//
// Algorithmic traffic: 4 B per cell-timestep; output has one row per DAY.
#include <vector>

#include "kernels.cuh"

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

// ---------------------------------------------------------------- staged reduce
// A warp owns one 32x4 tile and walks its days, but it does not reduce every day with warp
// shuffles against DENSE 128-float weight vectors (4 FMAs + ~1.1 shuffles per slot and step
// whatever the slot's fill: 70 of wind's 213 warp-instructions per step).  Instead the per-cell
// values of HEAT_STAGE days are parked in shared memory, and the reduce runs with the lanes
// spanning TIME: lane (q, r) owns the day pair r of the chunk and walks a q-th of the slot's
// STORED matrix entries {cell, weight}; per entry it costs one broadcast 8-byte load of the entry,
// one conflict-light 8-byte shared load of the cell's two days and two FMAs -- work proportional
// to the entries of the tile (~1.2 per cell for NUTS-like shapes), independent of how many buses
// touch the tile, ~12 instructions per step instead of ~70.  Entries a CSR matrix does not store are
// never multiplied, so NaN/Inf cells poison exactly the buses that contain them (scipy semantics)
// with no special path.  The per-step operators (PV, wind, ...) use the shuffle reduce instead:
// alternating a compute phase and a latency-bound reduce phase inside one warp needs more resident
// warps than the staging area's shared-memory footprint allows.
//
// Staging area of one warp: R = HEAT_STAGE/2 rows (one per PAIR of consecutive days); a row holds
// the tile's 128 cells as float2 {even day, odd day} in stage_index order, then 8 * 16/R bytes that
// stay 0.0f (the target of the plan's padding entries) and shift consecutive rows by 16/R
// eight-byte bank pairs.  In the reduce phase the R lanes of a group read R different rows at the
// same cell (bank pairs 16/R apart) and the 16/R groups that share a shared-memory pass read
// CONSECUTIVE entries of the slot's list, which is sorted by stage index -- neighbouring cells,
// i.e. the bank pairs in between: conflict-free for the usual contiguous slot, never worse than
// 2-way.
constexpr int ENT_CAP = 256;  // entries of the warp's tile kept in shared memory (8 B each)
constexpr int SLOT_CAP = 24;  // slot records of the warp's tile kept in shared memory (16 B each)
struct Stage {
  static constexpr int kRows = HEAT_STAGE / 2;
  static constexpr int kShift = 16 / kRows > 0 ? 16 / kRows : 1;
  static constexpr int kRowBytes = TILE_CELLS * 8 + 8 * kShift;
  static constexpr int kEntOff = kRows * kRowBytes;          // entry cache (16-byte aligned)
  static constexpr int kSlotOff = kEntOff + ENT_CAP * 8;     // slot-record cache
  static constexpr int kWarpBytes = kSlotOff + SLOT_CAP * 16;
  static constexpr int kCtaBytes = WARPS_PER_CTA * kWarpBytes;
  static_assert(kEntOff % 16 == 0, "entry cache must be 16-byte aligned");
};

// The bytes behind the 128 cells of every staging row hold 0.0f (the padding entries of the
// plan point there).
__device__ __forceinline__ void stage_init(char* stage, int lane) {
  if (lane < Stage::kRows) {
#pragma unroll
    for (int k = 0; k < Stage::kShift; ++k)
      *reinterpret_cast<float2*>(stage + lane * Stage::kRowBytes + PAD_OFF + 8 * k) = make_float2(0.f, 0.f);
  }
}

// Park the lane's 4 values of day k of the chunk (row = day pair, half = parity).
__device__ __forceinline__ void stage_store1(char* stage, int lane, int k, const float (&v)[4]) {
  char* const w = stage + lane * 8 + (k >> 1) * Stage::kRowBytes + (k & 1) * 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) *reinterpret_cast<float*>(w + 256 * i) = v[i];
}

// A warp keeps its tile for many chunks, so the tile's slot records {first entry, entry count /
// PAIR_PAD, bus} and entry lists are copied into shared memory once (they are contiguous in the
// plan): the reduce phase then depends on shared-memory latency only, not on whether L1 / L2
// still hold the lists.  Tiles with more than SLOT_CAP slots or ENT_CAP entries (rare: the
// average is 4 slots / 160 entries) keep reading the plan from global memory.
__device__ __forceinline__ bool tile_cache_load(char* stage, const PlanDev& plan, int s_beg, int s_end,
                                                int lane) {
  const int K = s_end - s_beg;
  if (K <= 0 || K > SLOT_CAP) return false;
  const int base = __ldg(plan.slot_rec + s_beg).x;
  const int2 last = __ldg(plan.slot_rec + s_end - 1);
  const int total = last.x + last.y * PAIR_PAD - base;
  if (total > ENT_CAP) return false;
  int4* const slots = reinterpret_cast<int4*>(stage + Stage::kSlotOff);
  uint2* const ent = reinterpret_cast<uint2*>(stage + Stage::kEntOff);
  if (lane < K) {
    const int2 r = __ldg(plan.slot_rec + s_beg + lane);
    slots[lane] = make_int4(r.x - base, r.y, __ldg(plan.slot_row + s_beg + lane), 0);
  }
  const uint2* const src = reinterpret_cast<const uint2*>(plan.pairs) + base;
  for (int i = lane; i < total; i += 32) ent[i] = __ldg(src + i);
  return true;
}

// The reduce phase of one chunk: rows [row0, row0 + nvalid) of `out` receive the sums of the
// staged days.  Lane = group * R + row: lane (q, r) owns the day pair r and walks the
// entries q, q + NQ, q + 2 NQ, ... of every slot's list; one butterfly over the groups, then
// group 0 adds the even day and group 1 the odd one in ONE atomic instruction.
// (__syncwarp() before -- the stores of all lanes must be visible -- and after.)
__device__ __forceinline__ void staged_reduce(const char* stage, const PlanDev& plan, int s_beg, int s_end,
                                              float* __restrict__ out, int row0, int nvalid, int lane,
                                              bool cached) {
  constexpr int R = Stage::kRows;  // rows = lanes along time
  static_assert(32 % R == 0, "the rows must divide the warp");
  constexpr int NQ = 32 / R;  // lanes sharing a row split a slot's entries NQ ways
  constexpr int U = PAIR_PAD / NQ;  // entries per group and padding unit
  static_assert(U >= 1 && U * NQ == PAIR_PAD, "PAIR_PAD must be a multiple of the group count");
  const int rp = lane & (R - 1), q = lane / R;
  const char* const rd_row = stage + rp * Stage::kRowBytes;
  const int nb = plan.n_bus;
  const int odd = lane >= R ? 1 : 0;
  float* const o_mine = out + (size_t)(row0 + 2 * rp + odd) * nb;
  const bool w_mine = lane < 2 * R && 2 * rp + odd < nvalid;
  auto finish = [&](float a0, float a1, int row) {
#pragma unroll
    for (int o = R; o < 32; o <<= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (w_mine) atomicAdd(o_mine + row, odd ? a1 : a0);
  };
  if (cached) {
    const int4* const slots = reinterpret_cast<const int4*>(stage + Stage::kSlotOff);
    const uint2* const ent_q = reinterpret_cast<const uint2*>(stage + Stage::kEntOff) + q;
    const int K = s_end - s_beg;
    // two slots at a time: their load -> load -> FMA chains are independent, which halves the
    // latency a warp spends in this phase (the phase is latency-, not issue-bound)
    int k = 0;
#pragma unroll 1
    for (; k + 1 < K; k += 2) {
      const int4 sa = slots[k], sb = slots[k + 1];
      const uint2 *pa = ent_q + sa.x, *pb = ent_q + sb.x;
      float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
      const int nmin = min(sa.y, sb.y);
      int it = 0;
#pragma unroll 2
      for (; it < nmin; ++it, pa += PAIR_PAD, pb += PAIR_PAD) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint2 wa = pa[u * NQ], wb = pb[u * NQ];
          const float2 xa = *reinterpret_cast<const float2*>(rd_row + wa.x);
          const float2 xb = *reinterpret_cast<const float2*>(rd_row + wb.x);
          a0 = fmaf(__uint_as_float(wa.y), xa.x, a0);
          a1 = fmaf(__uint_as_float(wa.y), xa.y, a1);
          b0 = fmaf(__uint_as_float(wb.y), xb.x, b0);
          b1 = fmaf(__uint_as_float(wb.y), xb.y, b1);
        }
      }
#pragma unroll 2
      for (int ia = it; ia < sa.y; ++ia, pa += PAIR_PAD) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint2 wa = pa[u * NQ];
          const float2 xa = *reinterpret_cast<const float2*>(rd_row + wa.x);
          a0 = fmaf(__uint_as_float(wa.y), xa.x, a0);
          a1 = fmaf(__uint_as_float(wa.y), xa.y, a1);
        }
      }
#pragma unroll 2
      for (int ib = it; ib < sb.y; ++ib, pb += PAIR_PAD) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint2 wb = pb[u * NQ];
          const float2 xb = *reinterpret_cast<const float2*>(rd_row + wb.x);
          b0 = fmaf(__uint_as_float(wb.y), xb.x, b0);
          b1 = fmaf(__uint_as_float(wb.y), xb.y, b1);
        }
      }
#pragma unroll
      for (int o = R; o < 32; o <<= 1) {  // both butterflies interleaved
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        b0 += __shfl_xor_sync(0xffffffffu, b0, o);
        b1 += __shfl_xor_sync(0xffffffffu, b1, o);
      }
      if (w_mine) {
        atomicAdd(o_mine + sa.z, odd ? a1 : a0);
        atomicAdd(o_mine + sb.z, odd ? b1 : b0);
      }
    }
    if (k < K) {
      const int4 sr = slots[k];
      const uint2* p = ent_q + sr.x;
      float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
      for (int it = 0; it < sr.y; ++it, p += PAIR_PAD) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint2 pw = p[u * NQ];
          const float2 x = *reinterpret_cast<const float2*>(rd_row + pw.x);
          const float w = __uint_as_float(pw.y);
          a0 = fmaf(w, x.x, a0);
          a1 = fmaf(w, x.y, a1);
        }
      }
      finish(a0, a1, sr.z);
    }
    return;
  }
  const uint2* const pairs_q = reinterpret_cast<const uint2*>(plan.pairs) + q;
#pragma unroll 1
  for (int s = s_beg; s < s_end; ++s) {
    const int2 rec = __ldg(plan.slot_rec + s);
    const uint2* p = pairs_q + rec.x;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll 2
    for (int it = 0; it < rec.y; ++it, p += PAIR_PAD) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint2 pw = __ldg(p + u * NQ);
        const float2 x = *reinterpret_cast<const float2*>(rd_row + pw.x);
        const float w = __uint_as_float(pw.y);
        a0 = fmaf(w, x.x, a0);
        a1 = fmaf(w, x.y, a1);
      }
    }
    finish(a0, a1, __ldg(plan.slot_row + s));
  }
}

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
template <bool VEC>
__device__ __forceinline__ void heat_day(const HeatParams& hp, const TileGeomT<VEC>& g, int d,
                                         float (&v)[4]) {
  const int s0 = __ldg(hp.day_start + d) - hp.base, s1 = __ldg(hp.day_start + d + 1) - hp.base;
  float sum[4] = {0.f, 0.f, 0.f, 0.f}, cnt[4] = {0.f, 0.f, 0.f, 0.f};
  float x[HEAT_UNROLL][4], y[HEAT_UNROLL][4];
  heat_load_chunk(hp, g, s0, s1, x);
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
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, cnt[4] = {0.f, 0.f, 0.f, 0.f};
  float v[4];
  if (MODE == 0) {
    // daily values of HEAT_STAGE days are parked in shared memory, then reduced with the lanes
    // along the days (staged_reduce); NaN days poison exactly the buses whose
    // stored entries meet them
    extern __shared__ __align__(16) float smem[];
    char* const stage = reinterpret_cast<char*>(smem) + warp * Stage::kWarpBytes;
    stage_init(stage, lane);
    const bool cached = tile_cache_load(stage, plan, s_beg, s_end, lane);
    for (int dc = d0; dc < d1; dc += HEAT_STAGE) {
      const int n = min(HEAT_STAGE, d1 - dc);
      for (int k = 0; k < n; ++k) {
        heat_day(hp, g, dc + k, v);
        zero_invalid(g, v);
        stage_store1(stage, lane, k, v);
      }
      __syncwarp();
      staged_reduce(stage, plan, s_beg, s_end, out, dc, n, lane, cached);
      __syncwarp();
    }
    return;
  }
  for (int d = d0; d < d1; ++d) {
    heat_day(hp, g, d, v);
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
    smem = Stage::kCtaBytes;
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
