// plan.cu -- error plumbing, aggregation-plan construction and the generic SpMM.
//
// The reference turns `matrix | shapes | layout` into ONE scipy CSR matrix
// (convert.py:213-254) and multiplies every dense (time, spatial) block by its
// transpose (aggregate.py:24-32).  Here the CSR is re-tiled once into
// (tile, bus) "slots": for every 32x4-cell warp tile the distinct buses that
// touch it, each with a dense 128-entry weight vector.  The fused kernels then
// reduce the per-cell values of a tile into its slots with warp shuffles and
// one atomicAdd per (slot, time step) -- per-cell values never reach HBM.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "kernels.cuh"

namespace atl {

static thread_local std::string g_err;
int64_t g_launches = 0;

static bool g_deterministic = [] {
  const char* v = getenv("ATL_DETERMINISTIC");
  return v && atoi(v) != 0;
}();
bool deterministic() { return g_deterministic; }

// out[t, bus] = sum of the bus's slot partials, always in the same order.
__global__ void k_gather_slots(const float* __restrict__ partial, const int32_t* __restrict__ row_slot_ptr,
                               const int32_t* __restrict__ row_slots, float* __restrict__ out,
                               int n_bus, int64_t n_slots, int nt) {
  const int row = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.y * (blockDim.x >> 5) + warp;
  if (t >= nt) return;
  const int b = row_slot_ptr[row], e = row_slot_ptr[row + 1];
  const float* p = partial + (size_t)t * n_slots;
  float acc = 0.f;
  for (int k = b + lane; k < e; k += 32) acc += p[row_slots[k]];
  acc = warp_sum(acc);
  if (lane == 0) out[(size_t)t * n_bus + row] = acc;
}

int launch_gather_slots(const AtlPlan* plan, const float* partial, int64_t nt, float* out,
                        cudaStream_t st) {
  if (nt <= 0 || plan->n_bus == 0) return ATL_OK;
  const int wpb = 8;
  for (int64_t t = 0; t < nt; t += 65535LL * wpb) {
    const int64_t n = std::min<int64_t>(nt - t, 65535LL * wpb);
    dim3 grid(plan->n_bus, (unsigned)((n + wpb - 1) / wpb));
    k_gather_slots<<<grid, 32 * wpb, 0, st>>>(partial + (size_t)t * plan->n_slots,
                                              plan->d_row_slot_ptr, plan->d_row_slots,
                                              out + (size_t)t * plan->n_bus, plan->n_bus,
                                              plan->n_slots, (int)n);
    ++g_launches;
    ATL_CUDA(cudaGetLastError());
  }
  return ATL_OK;
}

int tb_override() {
  static const int tb = [] {
    const char* v = getenv("ATL_TB");
    return v ? atoi(v) : 0;
  }();
  return tb;
}

void set_error(const std::string& msg) { g_err = msg; }
int cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what;
  return ATL_ERR_CUDA;
}

__global__ void k_csr_spmm(const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx,
                           const float* __restrict__ val, const float* __restrict__ dense,
                           int64_t S, float* __restrict__ out, int n_bus, int nt) {
  const int row = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.y * (blockDim.x >> 5) + warp;
  if (t >= nt) return;
  const int64_t b = indptr[row], e = indptr[row + 1];
  const float* d = dense + (int64_t)t * S;
  float acc = 0.f;
  for (int64_t k = b + lane; k < e; k += 32) acc = fmaf(val[k], d[idx[k]], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[(size_t)t * n_bus + row] = acc;
}

int launch_csr_spmm(const AtlPlan* plan, const float* dense, int64_t nt, float* out,
                    cudaStream_t st) {
  if (nt <= 0 || plan->n_bus == 0) return ATL_OK;
  const int wpb = 8;
  for (int64_t t = 0; t < nt; t += 65535LL * wpb) {
    const int64_t n = std::min<int64_t>(nt - t, 65535LL * wpb);
    dim3 grid(plan->n_bus, (unsigned)((n + wpb - 1) / wpb));
    k_csr_spmm<<<grid, 32 * wpb, 0, st>>>(plan->d_indptr, plan->d_indices, plan->d_vals,
                                          dense + t * plan->grid.S_out, plan->grid.S_out,
                                          out + (size_t)t * plan->n_bus, plan->n_bus, (int)n);
    ++g_launches;
    ATL_CUDA(cudaGetLastError());
  }
  return ATL_OK;
}

// Identity physics: the "field" already is the per-cell value (unknown
// convert_func evaluated upstream) -> fused tile SpMM.
template <bool VEC>
struct IdentityPhys {
  static constexpr bool kVec = VEC;
  using Geom = TileGeomT<VEC>;
  const float* f;
  int64_t S;
  struct Cell {};
  struct Raw {
    float v[4];
  };
  static constexpr int kSmemFloats = 0;
  static constexpr int kBatch = 4, kMinBlocks = 6;
  static constexpr bool kHasExact = false;
  static constexpr bool kResidentWeights = VEC;  // first slot group's weights in registers for the whole tile walk
  __device__ void stage(float*) const {}
  __device__ void init(Cell&, const Geom&, const float*) const {}
  __device__ void load(const Cell&, const Geom& g, int64_t tb, Raw& r) const { load4(f, tb, g, r.v); }
  __device__ void compute(const Cell&, const Geom&, int, const Raw& r, float (&v)[4],
                          const float*) const {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = r.v[i];
  }
};

}  // namespace atl

using namespace atl;

extern "C" {

int atl_abi_version(void) { return ATL_ABI_VERSION; }

int atl_hash128(const void* data, int64_t nbytes, uint64_t seed, uint64_t out[2]) {
  ATL_REQUIRE(out && nbytes >= 0 && (data || nbytes == 0), "bad arguments");
  auto rotl = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
  auto fmix = [](uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdULL;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ULL;
    k ^= k >> 33;
    return k;
  };
  const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
  uint64_t h1 = seed, h2 = seed ^ 0x9e3779b97f4a7c15ULL;
  const unsigned char* p = static_cast<const unsigned char*>(data);
  const int64_t nblocks = nbytes / 16;
  for (int64_t i = 0; i < nblocks; ++i) {
    uint64_t k1, k2;
    std::memcpy(&k1, p + 16 * i, 8);
    std::memcpy(&k2, p + 16 * i + 8, 8);
    k1 *= c1; k1 = rotl(k1, 31); k1 *= c2; h1 ^= k1;
    h1 = rotl(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729ULL;
    k2 *= c2; k2 = rotl(k2, 33); k2 *= c1; h2 ^= k2;
    h2 = rotl(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5ULL;
  }
  unsigned char tail[16] = {0};
  const int64_t rest = nbytes - 16 * nblocks;
  if (rest > 0) {
    std::memcpy(tail, p + 16 * nblocks, (size_t)rest);
    uint64_t k1, k2;
    std::memcpy(&k1, tail, 8);
    std::memcpy(&k2, tail + 8, 8);
    k2 *= c2; k2 = rotl(k2, 33); k2 *= c1; h2 ^= k2;
    k1 *= c1; k1 = rotl(k1, 31); k1 *= c2; h1 ^= k1;
  }
  h1 ^= (uint64_t)nbytes; h2 ^= (uint64_t)nbytes;
  h1 += h2; h2 += h1;
  h1 = fmix(h1); h2 = fmix(h2);
  h1 += h2; h2 += h1;
  out[0] = h1;
  out[1] = h2;
  return ATL_OK;
}
int atl_set_deterministic(int on) {
  const int prev = g_deterministic ? 1 : 0;
  g_deterministic = on != 0;
  return prev;
}
const char* atl_last_error(void) { return g_err.c_str(); }
int64_t atl_launch_count(void) { return g_launches; }

int atl_device_count(int* count_out) {
  ATL_REQUIRE(count_out, "count_out is NULL");
  *count_out = 0;
  ATL_CUDA(cudaGetDeviceCount(count_out));
  return ATL_OK;
}

}  // extern "C"

namespace atl {

// Host-side tiling of the CSR matrix (no CUDA involved; also exported through
// atl_plan_tiling_host for CPU tests).
struct Tiling {
  GridDev gd;
  bool vec = false, fused = false;
  int64_t nnz = 0, n_slots = 0;
  int32_t n_tiles = 0, n_active = 0;
  std::vector<int32_t> tile_slot_ptr, slot_row, active;
  std::vector<float> w;  // n_slots * 128 weights in lane order (only if fused)
  // the stored entries of every slot for the staged reduce: {stage byte offset, weight},
  // sorted by stage index, duplicates of one (bus, cell) summed (csr_matrix semantics),
  // explicit zeros kept; slot s owns pairs[slot_pair_ptr[s] .. slot_pair_ptr[s+1]), the first
  // slot_pair_n[s] of which are real, the rest padding {PAD_OFF, 0} up to a multiple of PAIR_PAD
  std::vector<int32_t> slot_pair_ptr, slot_pair_n;
  std::vector<PairEnt> pairs;
  int64_t n_pairs = 0;  // real entries
};

static int build_tiling(int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus, const int64_t* indptr,
                        const int32_t* indices, const double* data, bool force_arrays,
                        Tiling& T) {
  ATL_REQUIRE(ny > 0 && nx > 0 && n_bus >= 0, "bad plan shape");
  if (pitch <= 0) pitch = nx;
  ATL_REQUIRE(pitch >= nx, "pitch must be >= nx");
  ATL_REQUIRE((int64_t)ny * pitch < (1LL << 29), "grid too large (ny*pitch must be < 2^29)");
  ATL_REQUIRE(indptr && (n_bus == 0 || indptr[n_bus] == 0 || (indices && data)),
              "CSR arrays missing");
  const GridDev gd = make_grid(ny, nx, pitch);
  const bool vec = (pitch % 4 == 0);  // lane layout of the weight vectors / kernels
  const int64_t nnz_in = n_bus ? indptr[n_bus] : 0;
  const int64_t n_tiles = (int64_t)gd.n_tx * gd.n_ty;

  struct Ent {
    int64_t key;    // tile * n_bus + bus
    int32_t local;  // position inside the tile's 128-entry weight vector
    float w;
  };
  // Entries in (tile, bus, stage position) order.  A layout changes the matrix values with every
  // call of a "many layouts" workflow, so the plan is rebuilt per call: a counting sort by tile
  // (entries keep their CSR order inside a tile) followed by independent small sorts per tile on a
  // few threads replaces one global sort of all entries (1.2 M at 1440 x 720 -> 3000 shapes:
  // 113 ms -> 34 ms per build on the 8-core build box, bit-identical plans).
  std::vector<Ent> raw((size_t)nnz_in);
  std::vector<int64_t> tile_ptr((size_t)n_tiles + 1, 0);
  {
    size_t q = 0;
    for (int32_t r = 0; r < n_bus; ++r) {
      ATL_REQUIRE(indptr[r + 1] >= indptr[r], "indptr not monotone");
      for (int64_t k = indptr[r]; k < indptr[r + 1]; ++k, ++q) {
        const int32_t c = indices[k];
        ATL_REQUIRE(c >= 0 && c < gd.S_out, "column index out of range");
        const int iy = c / nx, ix = c - iy * nx;
        const int64_t tile = (int64_t)(iy / TILE_Y) * gd.n_tx + ix / TILE_X;
        Ent& e = raw[q];
        e.key = tile * (int64_t)n_bus + r;
        e.local = tile_local_index(vec, iy, ix);
        e.w = (float)data[k];
        ++tile_ptr[(size_t)tile + 1];
      }
    }
  }
  for (int64_t t = 0; t < n_tiles; ++t) tile_ptr[(size_t)t + 1] += tile_ptr[(size_t)t];
  std::vector<Ent> ents((size_t)nnz_in);
  {
    std::vector<int64_t> fill(tile_ptr.begin(), tile_ptr.end() - 1);
    for (const Ent& e : raw) ents[(size_t)fill[(size_t)(e.key / n_bus)]++] = e;
  }
  std::vector<Ent>().swap(raw);
  {
    // inside a tile the entries already come bus by bus (CSR rows are walked in order): each run
    // of one bus -- at most 128 entries -- only needs ordering by stage position; a stable
    // insertion sort does that without allocating (duplicates keep their CSR order)
    auto sort_tiles = [&](int64_t t_lo, int64_t t_hi) {
      Ent* const base = ents.data();
      int64_t a = tile_ptr[(size_t)t_lo];
      const int64_t end = tile_ptr[(size_t)t_hi];
      while (a < end) {
        int64_t z = a + 1;
        while (z < end && base[z].key == base[a].key) ++z;
        // the usual case -- column indices ascending inside a CSR row, hence `local` ascending in
        // the run -- makes stage order (32 * (local & 3) + (local >> 2)) a stable 4-way
        // de-interleave by (local & 3): O(n); anything else takes the insertion sort
        bool ascending = z - a <= 256;
        for (int64_t i = a + 1; i < z && ascending; ++i) ascending = base[i - 1].local <= base[i].local;
        if (ascending) {
          Ent tmp[256];
          int n_in[5] = {0, 0, 0, 0, 0};
          for (int64_t i = a; i < z; ++i) ++n_in[(base[i].local & 3) + 1];
          for (int g = 0; g < 4; ++g) n_in[g + 1] += n_in[g];
          for (int64_t i = a; i < z; ++i) tmp[n_in[base[i].local & 3]++] = base[i];
          std::memcpy(base + a, tmp, (size_t)(z - a) * sizeof(Ent));
        } else {
          for (int64_t i = a + 1; i < z; ++i) {
            const Ent e = base[i];
            const int se = stage_index(e.local);
            int64_t j = i;
            while (j > a && stage_index(base[j - 1].local) > se) {
              base[j] = base[j - 1];
              --j;
            }
            base[j] = e;
          }
        }
        a = z;
      }
    };
    unsigned nthr = std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
    if (nnz_in < (1 << 16)) nthr = 1;
    std::vector<std::thread> pool;
    int64_t t_lo = 0;
    for (unsigned i = 0; i < nthr; ++i) {  // tile ranges with about the same number of entries
      int64_t t_hi = t_lo;
      const int64_t want = nnz_in * (int64_t)(i + 1) / nthr;
      while (t_hi < n_tiles && (tile_ptr[(size_t)t_hi + 1] <= want || i + 1 == nthr)) ++t_hi;
      if (i + 1 == nthr) t_hi = n_tiles;
      if (nthr == 1) sort_tiles(t_lo, t_hi);
      else pool.emplace_back(sort_tiles, t_lo, t_hi);
      t_lo = t_hi;
    }
    for (auto& th : pool) th.join();
  }

  int64_t n_slots = 0, n_active = 0;
  {
    int64_t prev = -1, prev_tile = -1;
    for (const Ent& e : ents) {
      if (e.key != prev) {
        prev = e.key;
        ++n_slots;
        const int64_t tile = e.key / n_bus;
        if (tile != prev_tile) {
          prev_tile = tile;
          ++n_active;
        }
      }
    }
  }
  ATL_REQUIRE(n_slots < (1LL << 31), "too many (tile,bus) slots");
  // A matrix "tiles well" when a tile is touched by few buses; otherwise (e.g.
  // one bus per cell) the padded slot work explodes: use the two-pass CSR path.
  const double spt = n_active ? (double)n_slots / (double)n_active : 0.0;
  T.gd = gd;
  T.vec = vec;
  T.fused = spt <= 24.0 && (double)n_slots * TILE_CELLS * 4.0 <= 4.0e9;
  T.nnz = nnz_in;
  T.n_slots = n_slots;
  T.n_tiles = (int32_t)n_tiles;
  T.n_active = (int32_t)n_active;
  if (!(T.fused || force_arrays)) return ATL_OK;

  T.tile_slot_ptr.assign((size_t)n_tiles + 1, 0);
  T.slot_row.resize((size_t)n_slots);
  T.w.assign((size_t)n_slots * TILE_CELLS, 0.f);
  T.active.clear();
  T.active.reserve((size_t)n_active);
  T.slot_pair_ptr.assign((size_t)n_slots + 1, 0);
  T.slot_pair_n.assign((size_t)n_slots, 0);
  T.pairs.clear();
  T.pairs.reserve(ents.size() + (size_t)n_slots * (PAIR_PAD / 2));
  T.n_pairs = 0;
  auto close_slot = [&](int64_t slot) {  // pad the finished slot's list
    if (slot < 0) return;
    T.slot_pair_n[(size_t)slot] = (int32_t)(T.pairs.size() - (size_t)T.slot_pair_ptr[(size_t)slot]);
    while ((T.pairs.size() - (size_t)T.slot_pair_ptr[(size_t)slot]) % PAIR_PAD) {
      PairEnt pad;
      pad.off = PAD_OFF;
      pad.w = 0.f;
      T.pairs.push_back(pad);
    }
    T.slot_pair_ptr[(size_t)slot + 1] = (int32_t)T.pairs.size();
  };
  int64_t s = -1, prev = -1, prev_tile = -1;
  int32_t prev_local = -1;
  for (const Ent& e : ents) {
    if (e.key != prev) {
      close_slot(s);
      prev = e.key;
      prev_local = -1;
      ++s;
      const int64_t tile = e.key / n_bus;
      T.slot_row[(size_t)s] = (int32_t)(e.key - tile * n_bus);
      T.tile_slot_ptr[(size_t)tile + 1]++;
      if (tile != prev_tile) {
        prev_tile = tile;
        T.active.push_back((int32_t)tile);
      }
    }
    T.w[(size_t)s * TILE_CELLS + e.local] += e.w;  // duplicates sum (csr_matrix semantics)
    if (e.local == prev_local) {
      T.pairs.back().w += e.w;
    } else {
      PairEnt pe;
      pe.off = (uint32_t)stage_index(e.local) * 8u;
      pe.w = e.w;
      T.pairs.push_back(pe);
      prev_local = e.local;
      ++T.n_pairs;
    }
  }
  close_slot(s);
  ATL_REQUIRE(T.pairs.size() < (1ull << 31), "too many matrix entries for one plan");
  for (int64_t t = 0; t < n_tiles; ++t) T.tile_slot_ptr[(size_t)t + 1] += T.tile_slot_ptr[(size_t)t];
  return ATL_OK;
}

}  // namespace atl

extern "C" {

int atl_plan_tiling_host(int32_t ny, int32_t nx, int32_t n_bus, const int64_t* indptr,
                         const int32_t* indices, const double* data, AtlPlanInfo* info,
                         int32_t* tile_slot_ptr_out, int32_t* slot_row_out, float* slot_w_out,
                         int64_t slot_capacity) {
  ATL_REQUIRE(info, "info is NULL");
  Tiling T;
  const bool want = tile_slot_ptr_out || slot_row_out || slot_w_out;
  int rc = build_tiling(ny, nx, 0, n_bus, indptr, indices, data, want, T);
  if (rc) return rc;
  info->ny = ny;
  info->nx = nx;
  info->n_bus = n_bus;
  info->nnz = T.nnz;
  info->n_tiles = T.n_tiles;
  info->n_active_tiles = T.n_active;
  info->n_slots = T.n_slots;
  info->slots_per_active_tile = T.n_active ? (double)T.n_slots / T.n_active : 0.0;
  info->fused = T.fused ? 1 : 0;
  info->pitch = nx;
  info->vec = T.vec ? 1 : 0;
  info->n_pairs = T.n_pairs;
  if (!want) return ATL_OK;
  ATL_REQUIRE(tile_slot_ptr_out && slot_row_out && slot_w_out, "all three output arrays are needed");
  ATL_REQUIRE(slot_capacity >= T.n_slots, "slot_capacity too small");
  std::memcpy(tile_slot_ptr_out, T.tile_slot_ptr.data(), T.tile_slot_ptr.size() * 4);
  std::memcpy(slot_row_out, T.slot_row.data(), T.slot_row.size() * 4);
  std::memcpy(slot_w_out, T.w.data(), T.w.size() * 4);
  return ATL_OK;
}

int atl_plan_pairs_host(int32_t ny, int32_t nx, int32_t n_bus, const int64_t* indptr,
                        const int32_t* indices, const double* data, int64_t* n_pairs_out,
                        int32_t* slot_pair_ptr_out, int32_t* pair_cell_out, float* pair_w_out,
                        int64_t slot_capacity, int64_t pair_capacity) {
  ATL_REQUIRE(n_pairs_out, "n_pairs_out is NULL");
  Tiling T;
  int rc = build_tiling(ny, nx, 0, n_bus, indptr, indices, data, true, T);
  if (rc) return rc;
  *n_pairs_out = T.n_pairs;
  if (!slot_pair_ptr_out && !pair_cell_out && !pair_w_out) return ATL_OK;
  ATL_REQUIRE(slot_pair_ptr_out && pair_cell_out && pair_w_out, "all three output arrays are needed");
  ATL_REQUIRE(slot_capacity >= T.n_slots && pair_capacity >= T.n_pairs, "output capacity too small");
  // compact (unpadded) view: the padding entries {PAD_OFF, 0} are skipped
  int64_t o = 0;
  for (int64_t k = 0; k < T.n_slots; ++k) {
    slot_pair_ptr_out[k] = (int32_t)o;
    const int32_t b = T.slot_pair_ptr[(size_t)k];
    ATL_REQUIRE((T.slot_pair_ptr[(size_t)k + 1] - b) % PAIR_PAD == 0, "internal: unpadded slot");
    for (int32_t i = 0; i < T.slot_pair_n[(size_t)k]; ++i, ++o) {
      pair_cell_out[o] = (int32_t)(T.pairs[(size_t)b + i].off / 8u);
      pair_w_out[o] = T.pairs[(size_t)b + i].w;
    }
    for (int32_t i = b + T.slot_pair_n[(size_t)k]; i < T.slot_pair_ptr[(size_t)k + 1]; ++i)
      ATL_REQUIRE(T.pairs[(size_t)i].off == PAD_OFF && T.pairs[(size_t)i].w == 0.f, "internal: bad padding");
  }
  slot_pair_ptr_out[T.n_slots] = (int32_t)o;
  return ATL_OK;
}

int atl_plan_create(int device, int32_t ny, int32_t nx, int32_t n_bus,
                    const int64_t* indptr, const int32_t* indices, const double* data,
                    AtlPlan** plan_out) {
  return atl_plan_create_pitched(device, ny, nx, 0, n_bus, indptr, indices, data, plan_out);
}

int atl_plan_create_pitched(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus,
                            const int64_t* indptr, const int32_t* indices, const double* data,
                            AtlPlan** plan_out) {
  ATL_REQUIRE(plan_out, "plan_out is NULL");
  *plan_out = nullptr;
  Tiling T;
  int rc0 = build_tiling(ny, nx, pitch, n_bus, indptr, indices, data, false, T);
  if (rc0) return rc0;
  const int64_t nnz_in = T.nnz;

  AtlPlan* p = new AtlPlan();
  p->device = device;
  p->grid = T.gd;
  p->n_bus = n_bus;
  p->nnz = nnz_in;
  p->n_tiles = T.n_tiles;
  p->n_active = T.n_active;
  p->n_slots = T.n_slots;
  p->fused = T.fused;
  p->vec = T.vec;

  auto fail = [&](int rc) {
    atl_plan_destroy(p);
    return rc;
  };
  cudaError_t ce = cudaSetDevice(device);
  if (ce != cudaSuccess) return fail(cuda_fail(ce, "cudaSetDevice"));

#define PLAN_CUDA(call)                                   \
  do {                                                    \
    cudaError_t _e = (call);                              \
    if (_e != cudaSuccess) return fail(cuda_fail(_e, #call)); \
  } while (0)

  if (T.fused) {
    PLAN_CUDA(cudaMalloc((void**)&p->d_tile_slot_ptr, T.tile_slot_ptr.size() * 4));
    PLAN_CUDA(cudaMemcpy(p->d_tile_slot_ptr, T.tile_slot_ptr.data(), T.tile_slot_ptr.size() * 4,
                         cudaMemcpyHostToDevice));
    PLAN_CUDA(cudaMalloc((void**)&p->d_slot_row, std::max<size_t>(T.slot_row.size(), 1) * 4));
    PLAN_CUDA(cudaMemcpy(p->d_slot_row, T.slot_row.data(), T.slot_row.size() * 4,
                         cudaMemcpyHostToDevice));
    // + 3 zero slots: the grouped reduce (reduce_slots2g) reads up to 3 weight
    // vectors past a tile's last slot (their sums are discarded)
    PLAN_CUDA(cudaMalloc((void**)&p->d_slot_w4, (T.w.size() + 3 * 128) * 4));
    PLAN_CUDA(cudaMemset(p->d_slot_w4, 0, (T.w.size() + 3 * 128) * 4));
    PLAN_CUDA(cudaMemcpy(p->d_slot_w4, T.w.data(), T.w.size() * 4, cudaMemcpyHostToDevice));
    p->n_pairs = T.n_pairs;
    {
      std::vector<int2> rec((size_t)T.n_slots);
      for (int64_t k = 0; k < T.n_slots; ++k)
        rec[(size_t)k] = make_int2(T.slot_pair_ptr[(size_t)k],
                                   (T.slot_pair_ptr[(size_t)k + 1] - T.slot_pair_ptr[(size_t)k]) / PAIR_PAD);
      PLAN_CUDA(cudaMalloc((void**)&p->d_slot_rec, std::max<size_t>(rec.size(), 1) * sizeof(int2)));
      PLAN_CUDA(cudaMemcpy(p->d_slot_rec, rec.data(), rec.size() * sizeof(int2), cudaMemcpyHostToDevice));
    }
    PLAN_CUDA(cudaMalloc((void**)&p->d_pairs, std::max<size_t>(T.pairs.size(), 1) * sizeof(PairEnt)));
    PLAN_CUDA(cudaMemcpy(p->d_pairs, T.pairs.data(), T.pairs.size() * sizeof(PairEnt),
                         cudaMemcpyHostToDevice));
    PLAN_CUDA(cudaMalloc((void**)&p->d_active, std::max<size_t>(T.active.size(), 1) * 4));
    PLAN_CUDA(cudaMemcpy(p->d_active, T.active.data(), T.active.size() * 4,
                         cudaMemcpyHostToDevice));
    // deterministic mode: identity slot index and the slots of every bus (ascending tile)
    std::vector<int32_t> ident((size_t)T.n_slots), rsp((size_t)n_bus + 1, 0), rs((size_t)T.n_slots);
    for (int64_t s = 0; s < T.n_slots; ++s) {
      ident[(size_t)s] = (int32_t)s;
      rsp[(size_t)T.slot_row[(size_t)s] + 1]++;
    }
    for (int32_t r = 0; r < n_bus; ++r) rsp[(size_t)r + 1] += rsp[(size_t)r];
    {
      std::vector<int32_t> cur(rsp.begin(), rsp.end() - 1);
      for (int64_t s = 0; s < T.n_slots; ++s) rs[(size_t)cur[(size_t)T.slot_row[(size_t)s]]++] = (int32_t)s;
    }
    PLAN_CUDA(cudaMalloc((void**)&p->d_slot_ident, std::max<size_t>(ident.size(), 1) * 4));
    PLAN_CUDA(cudaMemcpy(p->d_slot_ident, ident.data(), ident.size() * 4, cudaMemcpyHostToDevice));
    PLAN_CUDA(cudaMalloc((void**)&p->d_row_slot_ptr, rsp.size() * 4));
    PLAN_CUDA(cudaMemcpy(p->d_row_slot_ptr, rsp.data(), rsp.size() * 4, cudaMemcpyHostToDevice));
    PLAN_CUDA(cudaMalloc((void**)&p->d_row_slots, std::max<size_t>(rs.size(), 1) * 4));
    PLAN_CUDA(cudaMemcpy(p->d_row_slots, rs.data(), rs.size() * 4, cudaMemcpyHostToDevice));
  }
  {
    // CSR copy (float weights) for the gather SpMM
    std::vector<float> vals((size_t)nnz_in);
    for (int64_t k = 0; k < nnz_in; ++k) vals[(size_t)k] = (float)data[k];
    PLAN_CUDA(cudaMalloc((void**)&p->d_indptr, ((size_t)n_bus + 1) * 8));
    PLAN_CUDA(cudaMemcpy(p->d_indptr, indptr, ((size_t)n_bus + 1) * 8, cudaMemcpyHostToDevice));
    PLAN_CUDA(cudaMalloc((void**)&p->d_indices, std::max<size_t>((size_t)nnz_in, 1) * 4));
    PLAN_CUDA(cudaMalloc((void**)&p->d_vals, std::max<size_t>((size_t)nnz_in, 1) * 4));
    if (nnz_in) {
      PLAN_CUDA(cudaMemcpy(p->d_indices, indices, (size_t)nnz_in * 4, cudaMemcpyHostToDevice));
      PLAN_CUDA(cudaMemcpy(p->d_vals, vals.data(), (size_t)nnz_in * 4, cudaMemcpyHostToDevice));
    }
  }
#undef PLAN_CUDA
  *plan_out = p;
  return ATL_OK;
}

int atl_plan_info(const AtlPlan* plan, AtlPlanInfo* info) {
  ATL_REQUIRE(plan && info, "NULL argument");
  info->ny = plan->grid.ny;
  info->nx = plan->grid.nx;
  info->n_bus = plan->n_bus;
  info->nnz = plan->nnz;
  info->n_tiles = plan->n_tiles;
  info->n_active_tiles = plan->n_active;
  info->n_slots = plan->n_slots;
  info->slots_per_active_tile = plan->n_active ? (double)plan->n_slots / plan->n_active : 0.0;
  info->fused = plan->fused ? 1 : 0;
  info->pitch = plan->grid.pitch;
  info->vec = plan->vec ? 1 : 0;
  info->n_pairs = plan->n_pairs;
  return ATL_OK;
}

void atl_plan_destroy(AtlPlan* p) {
  if (!p) return;
  cudaSetDevice(p->device);
  cudaFree(p->d_tile_slot_ptr);
  cudaFree(p->d_slot_row);
  cudaFree(p->d_slot_w4);
  cudaFree(p->d_slot_rec);
  cudaFree(p->d_pairs);
  cudaFree(p->d_active);
  cudaFree(p->d_slot_ident);
  cudaFree(p->d_row_slot_ptr);
  cudaFree(p->d_row_slots);
  cudaFree(p->d_indptr);
  cudaFree(p->d_indices);
  cudaFree(p->d_vals);
  delete p;
}

int atl_spmm(const AtlPlan* plan, const float* dense_dev, int64_t nt, float* out_dev,
             void* stream) {
  ATL_REQUIRE(plan && dense_dev && out_dev, "NULL argument");
  ATL_CUDA(cudaSetDevice(plan->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (!plan->fused) {
    ATL_REQUIRE(plan->grid.pitch == plan->grid.nx, "atl_spmm on a non-tiling plan needs an unpadded field");
    return launch_csr_spmm(plan, dense_dev, nt, out_dev, st);
  }
  auto make = [&](auto vec) {
    IdentityPhys<decltype(vec)::value> ph;
    ph.f = dense_dev;
    ph.S = plan->grid.S;
    return ph;
  };
  return dispatch_reduce(make, plan, aligned16(dense_dev), out_dev, nt, st);
}

}  // extern "C"
