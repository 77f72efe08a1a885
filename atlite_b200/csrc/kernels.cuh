// kernels.cuh -- generic "per-cell physics -> {shape reduce | per-cell store |
// per-cell time sum}" kernels, templated on a physics functor.
//
// A physics functor `Phys` provides
//   static constexpr bool kVec;   lane layout (see common.cuh: TileGeomT<VEC>)
//   struct Cell;   per-thread constants (geometry of the lane's 4 cells)
//   struct Raw;    the raw field values of one time step (4 cells)
//   static constexpr int kSmemFloats;        CTA-shared lookup tables
//   static constexpr int kBatch, kMinBlocks; time steps per batch / CTAs per SM
//   __device__ void stage(float* smem) const;            (whole CTA, before use)
//   __device__ void init(Cell&, const Geom&, const float* smem) const;
//   __device__ void load(const Cell&, const Geom&, int64_t tb, Raw&) const;
//        tb = byte offset of the time slab (t * S * 4), maintained by the caller
//   __device__ void compute(const Cell&, const Geom&, int t, const Raw&,
//                           float (&v)[4], const float* smem) const;
//        values of out-of-grid lanes are unspecified (finite border copies): they
//        carry zero weight in every slot and are never stored
//   static constexpr bool kHasExact;  if true, compute() may differ from the reference
//        when an INPUT is NaN/Inf but then always yields a non-finite value, and
//        compute_exact(...) (same signature) reproduces the reference's NaN rules; the
//        kernels call it only for steps whose fast result came out non-finite
//   static constexpr bool kSunGate (optional, default false): if true,
//   __device__ bool lit(const Cell&, int t) const;
//        false only if compute() yields exactly 0 for all 4 cells of the lane at step t WHATEVER
//        the raw values (finite or not); the shuffle-reduce walk and k_cells then skip the loads
//        of such lane-steps (and the shuffle-reduce walk whole batches no lane of the warp needs)
// `t` is relative to the slab the functor's field pointers address.
//
// Loop structure: a warp owns one 32x4 tile and walks a block of `tb`
// consecutive time steps.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace atl {

// Physics that are issue-bound rather than HBM-bound opt into two copies of the time walk
// (`static constexpr bool kSplitMask = true`), see fused_walk.
template <class P, class = void>
struct resident_weights : std::false_type {};
template <class P>
struct resident_weights<P, std::void_t<decltype(P::kResidentWeights)>> : std::bool_constant<P::kResidentWeights> {};
template <class P, class = void>
struct l2_prefetch : std::integral_constant<int, 0> {};
template <class P>
struct l2_prefetch<P, std::void_t<decltype(P::kL2Prefetch)>> : std::integral_constant<int, P::kL2Prefetch> {};
template <class P, class = void>
struct split_mask : std::false_type {};
template <class P>
struct split_mask<P, std::void_t<decltype(P::kSplitMask)>> : std::bool_constant<P::kSplitMask> {};
template <class P, class = void>
struct sun_gate : std::false_type {};
template <class P>
struct sun_gate<P, std::void_t<decltype(P::kSunGate)>> : std::bool_constant<P::kSunGate> {};

// kSunGate: bit j = phys.lit(c, t + j), j < N
template <int N, class Phys>
__device__ __forceinline__ unsigned lit_bits(const Phys& phys, const typename Phys::Cell& c, int t) {
  unsigned m = 0;
#pragma unroll
  for (int j = 0; j < N; ++j) m |= phys.lit(c, t + j) ? 1u << j : 0u;
  return m;
}

// The time walk of one warp tile.  MASK = the tile overhangs the grid (row padding / last tile
// column): only then are the values of out-of-grid lanes zeroed; interior tiles (the vast
// majority) run the copy of the loop without the selects (about one instruction in eight of
// the wind kernel).  The choice is warp-uniform, made once per tile.
template <class Phys, int B, bool MASK, class Geom>
__device__ __forceinline__ void fused_walk(const Phys& phys, const GridDev& gd, const PlanDev& plan,
                                           float* __restrict__ out, int nt, int tb, const Geom& g,
                                           int s_beg, int s_end, int lane, const float* smem) {
  const int t0 = blockIdx.y * tb;
  const int t1 = min(nt, t0 + tb);
  const int nb = plan.n_bus;

  typename Phys::Cell c;
  phys.init(c, g, smem);
  typename Phys::Raw r[B];
  float v[B][4];
  const int64_t S4 = gd.S * 4;
  int64_t sb = (int64_t)t0 * S4;  // byte offset of the next slab to LOAD
  const int nfull = (t1 - t0) / B;
  int t = t0;
  constexpr bool RES = resident_weights<Phys>::value && (B % 2 == 0);
  float4 wres[RES ? 4 : 1];
  int row_res = -1;
  if constexpr (RES) load_group_weights(wres, row_res, s_beg, s_end, plan, lane);
  // kSunGate: a lane loads step t only if phys.lit(c, t).  A skipped load leaves that step's raw
  // registers as they were (zero, or an earlier step of the same 4 cells): by the lit() contract
  // compute() still yields exactly 0 from them -- finite, so neither the NaN probe nor the exact
  // paths can be triggered by stale values.  A batch no lane of the warp needs is skipped whole (no
  // physics, no reduce, no atomics): its output rows keep the zeros of launch_fused's memset (the
  // per-slot partials in deterministic mode), which is what the reduce of all-zero values adds.
  // Batches keep their alignment (t0 + kB ..) and the reduce pairs the same steps as without the
  // gate, so a batch that does run (the exact path included) computes what it computed before.
  constexpr bool GATE = sun_gate<Phys>::value;
  unsigned lit = ~0u;  // bit j: this lane loads step j of the current batch
  bool run = true;     // some lane of the warp loads a step of the current batch
  if constexpr (GATE) {
#pragma unroll
    for (int j = 0; j < B; ++j) r[j] = typename Phys::Raw{};
  }
  if (nfull > 0) {
    if constexpr (GATE) {
      lit = lit_bits<B>(phys, c, t0);
      run = __any_sync(0xffffffffu, lit != 0);
    }
#pragma unroll
    for (int j = 0; j < B; ++j)
      if (!GATE || ((lit >> j) & 1u)) phys.load(c, g, sb + j * S4, r[j]);
    sb += B * S4;
#pragma unroll 1
    for (int k = 0; k < nfull; ++k, t += B) {
      bool bad = false;  // kHasExact: one probe serves the physics' NaN rules AND the reduce
      if (!GATE || run) {
#pragma unroll
        for (int j = 0; j < B; ++j) {
          phys.compute(c, g, t + j, r[j], v[j], smem);
          if (MASK) zero_invalid(g, v[j]);
        }
        if constexpr (Phys::kHasExact) {
          float chk = 0.f;
#pragma unroll
          for (int j = 0; j < B; ++j) chk += (v[j][0] + v[j][1]) + (v[j][2] + v[j][3]);
          bad = __any_sync(0xffffffffu, !(fabsf(chk) <= 3.0e38f));
          if (bad) {  // cold: a NaN/Inf reached a result -> the reference's NaN rules
#pragma unroll
            for (int j = 0; j < B; ++j) {
              phys.compute_exact(c, g, t + j, r[j], v[j], smem);
              if (MASK) zero_invalid(g, v[j]);
            }
          }
        }
      }
      unsigned lit_next = ~0u;
      bool run_next = true;
      if (k + 1 < nfull) {
        if constexpr (GATE) {
          lit_next = lit_bits<B>(phys, c, t + B);
          run_next = __any_sync(0xffffffffu, lit_next != 0);
        }
#pragma unroll
        for (int j = 0; j < B; ++j)
          if (!GATE || ((lit_next >> j) & 1u)) phys.load(c, g, sb + j * S4, r[j]);
        sb += B * S4;
        // kL2Prefetch = D > 0: the batch D batches past the one just requested goes to L2 now
        if constexpr (l2_prefetch<Phys>::value > 0) {
          constexpr int D = l2_prefetch<Phys>::value;
          if (k + 1 + D < nfull) {
#pragma unroll
            for (int j = 0; j < B; ++j) phys.prefetch(c, g, sb + ((D - 1) * B + j) * S4);
          }
        }
      }
      const bool dark = GATE && !run;  // nothing to add
      if constexpr (GATE) {
        lit = lit_next;
        run = run_next;
      }
      if (dark) continue;
#pragma unroll
      for (int j = 0; j + 1 < B; j += 2) {
        float* const o = out + (size_t)(t + j) * nb;
        if constexpr (Phys::kHasExact) {
          if (bad) {  // cold: what is left non-finite is meant to be; stored entries only
            reduce_slots_exact(v[j][0], v[j][1], v[j][2], v[j][3], s_beg, s_end, plan, o, lane);
            reduce_slots_exact(v[j + 1][0], v[j + 1][1], v[j + 1][2], v[j + 1][3], s_beg, s_end, plan, o + nb, lane);
          } else if constexpr (RES) {
            reduce_slots2g_res<false>(v[j], v[j + 1], wres, row_res, s_beg, s_end, plan, o, lane);
          } else {
            reduce_slots2g<false>(v[j], v[j + 1], s_beg, s_end, plan, o, lane);
          }
        } else if constexpr (RES) {
          reduce_slots2g_res(v[j], v[j + 1], wres, row_res, s_beg, s_end, plan, o, lane);
        } else {  // slots in groups of four (transposed butterfly)
          reduce_slots2g(v[j], v[j + 1], s_beg, s_end, plan, o, lane);
        }
      }
      if (B & 1) reduce_slots(v[B - 1], s_beg, s_end, plan, out + (size_t)(t + B - 1) * nb, lane);
    }
  }
  // tail: fewer than B steps left
#pragma unroll 1
  for (; t < t1; ++t, sb += S4) {
    if constexpr (GATE) {
      const bool l = phys.lit(c, t);
      if (!__any_sync(0xffffffffu, l)) continue;
      if (l) phys.load(c, g, sb, r[0]);
    } else {
      phys.load(c, g, sb, r[0]);
    }
    phys.compute(c, g, t, r[0], v[0], smem);
    if (MASK) zero_invalid(g, v[0]);
    if constexpr (Phys::kHasExact) {
      if (__any_sync(0xffffffffu, !(fabsf((v[0][0] + v[0][1]) + (v[0][2] + v[0][3])) <= 3.0e38f))) {
        phys.compute_exact(c, g, t, r[0], v[0], smem);
        if (MASK) zero_invalid(g, v[0]);
      }
    }
    reduce_slots(v[0], s_beg, s_end, plan, out + (size_t)t * nb, lane);
  }
}

// A warp owns one 32x4 tile and walks `tb` consecutive time steps in batches of
// B.  Per batch: the arithmetic of the B resident steps runs first, then the
// loads of the NEXT batch are issued into the now-dead raw registers, and only
// then the shuffle-reduce + atomics of the current batch execute -- so B steps of
// loads are in flight across the whole reduce phase at no extra register cost.
// Steps are reduced two at a time, slots four at a time, in one transposed
// butterfly (reduce_slots2g).  B is chosen per physics so that B x (#fields) 16-byte
// loads per lane cover the HBM latency (PV: 2 x 5, wind: 4 x 2, SpMM: 4 x 1).
// MINB = CTAs/SM the register allocator must allow.
template <class Phys, int B, int MINB>
__global__ void __launch_bounds__(CTA_THREADS, MINB)
    k_fused_reduce(const Phys phys, const GridDev gd, const PlanDev plan,
                   float* __restrict__ out, int nt, int tb) {
  extern __shared__ float smem[];
  phys.stage(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ai = blockIdx.x * WARPS_PER_CTA + warp;
  if (ai >= plan.n_active) return;
  const int tile = __ldg(plan.active_tiles + ai);
  const auto g = make_geom<Phys::kVec>(tile, lane, gd);
  const int s_beg = __ldg(plan.tile_slot_ptr + tile);
  const int s_end = __ldg(plan.tile_slot_ptr + tile + 1);
  if constexpr (split_mask<Phys>::value) {
    if (__any_sync(0xffffffffu, g.valid != 0xFu))
      fused_walk<Phys, B, true>(phys, gd, plan, out, nt, tb, g, s_beg, s_end, lane, smem);
    else
      fused_walk<Phys, B, false>(phys, gd, plan, out, nt, tb, g, s_beg, s_end, lane, smem);
  } else {
    fused_walk<Phys, B, true>(phys, gd, plan, out, nt, tb, g, s_beg, s_end, lane, smem);
  }
}

// MODE 0: store per-cell values out[(t - t_begin), y, x]
// MODE 1: accumulate the (NaN-skipping) time sum into out[y, x]
// Rolling software pipeline over B register sets: as soon as step t has been
// evaluated from set j its registers are reloaded with step t + B, so B - 1 steps
// of arithmetic (and the other warps) cover every load.  Load indices are clamped
// to the block's last step instead of predicated (at most B - 1 redundant loads
// and evaluations per time block, their results discarded).
// MODE 1 also counts the valid (non-NaN) steps per cell into `cnt_out` (may be NULL): the
// reference's per-cell mean skips NaN steps (convert.py:51-56).
template <class Phys, int MODE, int B, int MINB>
__global__ void __launch_bounds__(CTA_THREADS, MINB)
    k_cells(const Phys phys, const GridDev gd, float* __restrict__ out,
            float* __restrict__ cnt_out, int t_begin, int t_end, int tb) {
  extern __shared__ float smem[];
  phys.stage(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x * WARPS_PER_CTA + warp;
  if (tile >= gd.n_tx * gd.n_ty) return;
  const auto g = make_geom<Phys::kVec>(tile, lane, gd);
  const int t0 = t_begin + blockIdx.y * tb;
  const int t1 = min(t_end, t0 + tb);
  if (t0 >= t1) return;

  typename Phys::Cell c;
  phys.init(c, g, smem);
  typename Phys::Raw r[B];
  float v[4];
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  int n_nan[4] = {0, 0, 0, 0};
  const int64_t S4 = gd.S * 4;
  const int tl = t1 - 1;
  // kSunGate: lane-predicated loads only (see fused_walk for why stale raw registers are
  // harmless); a skipped step still yields exactly 0 and counts as a valid step of the mean
  constexpr bool GATE = sun_gate<Phys>::value;
  if constexpr (GATE) {
#pragma unroll
    for (int j = 0; j < B; ++j) r[j] = typename Phys::Raw{};
  }
  auto load_step = [&](int tn, typename Phys::Raw& rr) {
    if constexpr (GATE) {
      if (!phys.lit(c, tn)) return;
    }
    phys.load(c, g, (int64_t)tn * S4, rr);
  };
#pragma unroll
  for (int j = 0; j < B; ++j) load_step(min(t0 + j, tl), r[j]);
#pragma unroll 1
  for (int t = t0; t < t1; t += B) {
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const bool live = t + j < t1;
      phys.compute(c, g, min(t + j, tl), r[j], v, smem);
      if constexpr (Phys::kHasExact) {  // cold, warp-uniform: a NaN/Inf reached a result
        if (__any_sync(0xffffffffu, !(fabsf((v[0] + v[1]) + (v[2] + v[3])) <= 3.0e38f)))
          phys.compute_exact(c, g, min(t + j, tl), r[j], v, smem);
      }
      load_step(min(t + j + B, tl), r[j]);
      if (MODE == 0) {
        if (live) store4(out + (int64_t)(t + j - t_begin) * gd.S_out, gd, g, v);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {  // NaN steps are skipped and counted (one predicated add)
          const bool ok = v[q] == v[q];
          acc[q] += (live && ok) ? v[q] : 0.f;
          if (live && !ok) ++n_nan[q];
        }
      }
    }
  }
  if (MODE == 1) {
    atomic_add4(out, gd, g, acc);
    if (cnt_out) {  // valid steps of this block = its steps minus the NaN ones
      float cnt[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) cnt[q] = (float)(t1 - t0 - n_nan[q]);
      atomic_add4(cnt_out, gd, g, cnt);
    }
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Deterministic reduce mode (atl_set_deterministic): bitwise-repeatable results.
bool deterministic();

// Generic CSR gather SpMM: out[t, row] = sum_k val[k] * dense[t, col[k]]
// (aggregate.py:24-32 on an already materialised field).  One warp per
// (row, t); used for plans that do not tile well and as second pass of the
// two-pass fallback.
__global__ void k_csr_spmm(const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx,
                           const float* __restrict__ val, const float* __restrict__ dense,
                           int64_t S, float* __restrict__ out, int n_bus, int nt);

// Time steps per CTA of the fused reduce from the environment (ATL_TB, for time-block sweeps);
// 0 = chosen by pick_tb.
int tb_override();

__global__ void k_gather_slots(const float* __restrict__ partial, const int32_t* __restrict__ row_slot_ptr,
                               const int32_t* __restrict__ row_slots, float* __restrict__ out,
                               int n_bus, int64_t n_slots, int nt);
int launch_gather_slots(const AtlPlan* plan, const float* partial, int64_t nt, float* out,
                        cudaStream_t st);

inline int pick_tb(int n_cta_x, int64_t nt) {
  // time steps per CTA: aim for ~24 CTAs per resident slot (SMs x 5 CTAs) so
  // the tail wave is small, but keep the per-CTA prologue (geometry, slot setup)
  // amortised over >= 16 steps.
  const int64_t want = (int64_t)sm_count() * 5 * 24;
  int64_t tb = (nt * n_cta_x + want - 1) / want;
  if (tb < 16) tb = 16;
  if (tb > 128) tb = 128;
  tb += tb & 1;
  if (tb > nt) tb = nt > 0 ? nt : 1;
  return (int)tb;
}

template <class Phys>
int launch_cells(const Phys& phys, const GridDev& gd, float* out, int64_t t_begin,
                 int64_t t_end, bool timesum, cudaStream_t st, float* cnt_out = nullptr) {
  if (t_end <= t_begin) return ATL_OK;
  const int n_tiles = gd.n_tx * gd.n_ty;
  const int gx = (n_tiles + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
  // deterministic time sums: one time block, so every cell receives exactly one add
  const int tb = (timesum && deterministic()) ? (int)(t_end - t_begin) : pick_tb(gx, t_end - t_begin);
  const int gy = (int)((t_end - t_begin + tb - 1) / tb);
  dim3 grid(gx, gy);
  const size_t smem = Phys::kSmemFloats * sizeof(float);
  GridDev go = gd;
  go.out_vec = (gd.nx % 4 == 0 && aligned16(out)) ? 1 : 0;
  if (timesum)
    k_cells<Phys, 1, Phys::kBatch, Phys::kMinBlocks>
        <<<grid, CTA_THREADS, smem, st>>>(phys, go, out, cnt_out, (int)t_begin, (int)t_end, tb);
  else
    k_cells<Phys, 0, Phys::kBatch, Phys::kMinBlocks>
        <<<grid, CTA_THREADS, smem, st>>>(phys, go, out, nullptr, (int)t_begin, (int)t_end, tb);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int launch_csr_spmm(const AtlPlan* plan, const float* dense, int64_t nt, float* out,
                    cudaStream_t st);

// Fused path of one slab.  `Phys` must use the plan's lane layout.
template <class Phys>
int launch_fused(const Phys& phys, const AtlPlan* plan, float* out, int64_t nt, cudaStream_t st) {
  const bool det = deterministic() && plan->n_slots > 0;
  float* acc = out;  // where the per-(slot, step) partial sums are accumulated
  PlanDev pd = plan->dev();
  if (det) {
    ATL_CUDA(cudaMallocAsync((void**)&acc, (size_t)nt * plan->n_slots * sizeof(float), st));
    pd = plan->dev_partial();
  }
  ATL_CUDA(cudaMemsetAsync(acc, 0, (size_t)nt * pd.n_bus * sizeof(float), st));
  if (plan->n_active == 0) {
    if (det) ATL_CUDA(cudaFreeAsync(acc, st));
    if (det) ATL_CUDA(cudaMemsetAsync(out, 0, (size_t)nt * plan->n_bus * sizeof(float), st));
    return ATL_OK;
  }
  const int gx = (plan->n_active + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
  int tb = tb_override();
  if (tb <= 0) tb = pick_tb(gx, nt);
  dim3 grid(gx, (unsigned)((nt + tb - 1) / tb));
  k_fused_reduce<Phys, Phys::kBatch, Phys::kMinBlocks>
      <<<grid, CTA_THREADS, Phys::kSmemFloats * sizeof(float), st>>>(phys, plan->grid, pd, acc, (int)nt, tb);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  if (det) {
    int rc = launch_gather_slots(plan, acc, nt, out, st);
    cudaFreeAsync(acc, st);
    return rc;
  }
  return ATL_OK;
}

// Two-pass fallback for matrices that do not tile (e.g. one bus per cell):
// materialise a block of per-cell values, then CSR-gather it.
template <class Phys>
int launch_two_pass(const Phys& phys, const AtlPlan* plan, float* out, int64_t nt,
                    cudaStream_t st) {
  const int64_t S = plan->grid.S_out;  // the scratch cube is unpadded
  int64_t blk = (256LL << 20) / (S * 4);  // <= 256 MiB scratch
  if (blk < 1) blk = 1;
  if (blk > nt) blk = nt;
  float* scratch = nullptr;
  ATL_CUDA(cudaMallocAsync((void**)&scratch, (size_t)blk * S * sizeof(float), st));
  for (int64_t t = 0; t < nt; t += blk) {
    const int64_t n = (nt - t < blk) ? nt - t : blk;
    int rc = launch_cells(phys, plan->grid, scratch, t, t + n, false, st);
    if (rc == ATL_OK) rc = launch_csr_spmm(plan, scratch, n, out + (size_t)t * plan->n_bus, st);
    if (rc != ATL_OK) {
      cudaFreeAsync(scratch, st);
      return rc;
    }
  }
  ATL_CUDA(cudaFreeAsync(scratch, st));
  return ATL_OK;
}

// Dispatch on the lane layout.  `make(vec_tag)` builds the functor for a layout:
// make(std::true_type{}) -> Phys<VEC>, make(std::false_type{}) -> Phys<SCALAR>.
// `ptrs_aligned`: every field pointer is 16-byte aligned (needed for VEC).
template <class Make>
int dispatch_reduce(Make make, const AtlPlan* plan, bool ptrs_aligned, float* out, int64_t nt,
                    cudaStream_t st) {
  if (nt <= 0) return ATL_OK;
  ATL_REQUIRE(nt < (1LL << 31), "slab too long");
  if (plan->fused) {
    if (plan->vec) {
      ATL_REQUIRE(ptrs_aligned,
                  "field pointers must be 16-byte aligned (pitch % 4 == 0 uses 128-bit loads)");
      return launch_fused(make(std::true_type{}), plan, out, nt, st);
    }
    return launch_fused(make(std::false_type{}), plan, out, nt, st);
  }
  if (plan->vec && ptrs_aligned) return launch_two_pass(make(std::true_type{}), plan, out, nt, st);
  return launch_two_pass(make(std::false_type{}), plan, out, nt, st);
}

template <class Make>
int dispatch_cells(Make make, const GridDev& gd, bool ptrs_aligned, float* out, int64_t nt,
                   bool timesum, cudaStream_t st, float* cnt_out = nullptr) {
  if (gd.pitch % 4 == 0 && ptrs_aligned)
    return launch_cells(make(std::true_type{}), gd, out, 0, nt, timesum, st, cnt_out);
  return launch_cells(make(std::false_type{}), gd, out, 0, nt, timesum, st, cnt_out);
}

}  // namespace atl
