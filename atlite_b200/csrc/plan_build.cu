// plan_build.cu -- the aggregation plan (AtlPlan, see plan.cu) built on the device.
//
// Every stored entry k of the CSR matrix gets the key of the place it takes in the plan,
// ((tile * n_bus + bus) << 7) | stage index.  One stable radix sort by that key puts the entries
// in plan order: slots ascending by (tile, bus), the entries of a slot by stage index, and
// duplicates of one (bus, cell) next to each other in CSR order.  Every plan array then follows
// from the sorted keys by flag, scan and scatter passes.  The arrays are byte for byte those of the
// host tiling (build_tiling in plan.cu, which the tests compare against): weights are rounded and
// summed as the host does it, without flush-to-zero and with the NaN bits an x86 host produces.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace atl {
namespace {

constexpr int BUILD_THREADS = 256;
enum : int { ERR_MONOTONE = 1, ERR_COLUMN = 2, ERR_ENDS = 4 };

unsigned blocks_for(int64_t n) { return (unsigned)std::max<int64_t>((n + BUILD_THREADS - 1) / BUILD_THREADS, 1); }

// (float)x as the host computes it: round to nearest even and keep subnormals (the library is built
// with -ftz=true, which a plain cast in device code would follow); a NaN keeps its sign and top
// payload bits and is quieted, as x86 cvtsd2ss does.
__device__ __forceinline__ float host_f32(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  if ((b & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL)
    return __uint_as_float(((unsigned)(b >> 32) & 0x80000000u) | 0x7fc00000u | ((unsigned)(b >> 29) & 0x003fffffu));
  float r;
  asm("cvt.rn.f32.f64 %0, %1;" : "=f"(r) : "d"(x));
  return r;
}

// a += b as the host computes it (duplicates of one (bus, cell)): no flush-to-zero; a NaN operand
// is returned (the first one if both are), an invalid sum is x86's default NaN.
__device__ __forceinline__ float host_add(float a, float b) {
  if (isnan(a)) return a;
  if (isnan(b)) return b;
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return isnan(r) ? __uint_as_float(0xffc00000u) : r;
}

__global__ void k_check_indptr(const int64_t* __restrict__ indptr, int32_t n_bus, int64_t nnz, int* err) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_bus) return;
  if (r < n_bus && indptr[r + 1] < indptr[r]) atomicOr(err, ERR_MONOTONE);
  if ((r == 0 && indptr[0] != 0) || (r == n_bus && indptr[n_bus] != nnz)) atomicOr(err, ERR_ENDS);
}

// sort key and CSR position of every entry; the row is the last one starting at or before k
__global__ void k_entry_keys(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                             int32_t n_bus, int64_t nnz, int32_t nx, int64_t S_out, int32_t n_tx, bool vec,
                             unsigned long long* __restrict__ keys, int32_t* __restrict__ pos, int* err) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  int32_t lo = 0, hi = n_bus;
  while (hi - lo > 1) {
    const int32_t mid = (lo + hi) >> 1;
    if (indptr[mid] <= k) lo = mid;
    else hi = mid;
  }
  int32_t c = indices[k];
  if (c < 0 || c >= S_out) {
    atomicOr(err, ERR_COLUMN);
    c = 0;
  }
  const int iy = c / nx, ix = c - iy * nx;
  const int64_t tile = (int64_t)(iy / TILE_Y) * n_tx + ix / TILE_X;
  keys[k] = ((unsigned long long)(tile * n_bus + lo) << 7) | (unsigned)stage_index(tile_local_index(vec, iy, ix));
  pos[k] = (int32_t)k;
}

// first entry of a (slot, stage) pair / of a slot
__global__ void k_entry_heads(const unsigned long long* __restrict__ key, int64_t nnz, int32_t* __restrict__ pair_head,
                              int32_t* __restrict__ slot_head) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  const unsigned long long k = key[i], p = i ? key[i - 1] : ~0ULL;
  pair_head[i] = k != p;
  slot_head[i] = (k >> 7) != (p >> 7);
}

// per slot: its (tile * n_bus + bus) and the index of its first pair
__global__ void k_slot_starts(const unsigned long long* __restrict__ key, const int32_t* __restrict__ pair_id,
                              const int32_t* __restrict__ slot_id, int64_t nnz, int64_t* __restrict__ slot_key,
                              int32_t* __restrict__ slot_pair0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz || (i && slot_id[i] == slot_id[i - 1])) return;
  const int32_t s = slot_id[i] - 1;
  slot_key[s] = (int64_t)(key[i] >> 7);
  slot_pair0[s] = pair_id[i] - 1;
}

// per slot s < n_slots: its entry count padded to PAIR_PAD, and whether it opens a tile; 0 behind
// the last slot, so that the scans can run over nnz (an upper bound of n_slots) items
__global__ void k_slot_counts(const int64_t* __restrict__ slot_key, const int32_t* __restrict__ slot_pair0,
                              const int32_t* __restrict__ pair_id, const int32_t* __restrict__ slot_id, int64_t nnz,
                              int32_t n_bus, int64_t* __restrict__ padded, int32_t* __restrict__ tile_head) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nnz) return;
  const int32_t n_slots = slot_id[nnz - 1];
  if (s >= n_slots) {
    padded[s] = 0;
    tile_head[s] = 0;
    return;
  }
  const int32_t c = (s + 1 < n_slots ? slot_pair0[s + 1] : pair_id[nnz - 1]) - slot_pair0[s];
  padded[s] = (c + PAIR_PAD - 1) / PAIR_PAD * PAIR_PAD;
  tile_head[s] = s == 0 || slot_key[s] / n_bus != slot_key[s - 1] / n_bus;
}

struct Counts {
  int64_t n_padded;
  int32_t n_slots, n_pairs, n_active, err;
};

__global__ void k_counts(const int32_t* pair_id, const int32_t* slot_id, const int32_t* tile_scan,
                         const int64_t* pad_scan, int64_t nnz, const int* err, Counts* out) {
  Counts c{};
  if (nnz > 0) {
    c.n_padded = pad_scan[nnz - 1];
    c.n_slots = slot_id[nnz - 1];
    c.n_pairs = pair_id[nnz - 1];
    c.n_active = tile_scan[nnz - 1];
  }
  c.err = *err;
  *out = c;
}

// out[t] = the first s with v[s] >= t * scale, for t = 0 .. n_out - 1 (v ascending)
template <typename T>
__global__ void k_lower_bounds(const T* __restrict__ v, int64_t n, int64_t scale, int32_t* __restrict__ out,
                               int64_t n_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_out) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)v[mid] < t * scale) lo = mid + 1;
    else hi = mid;
  }
  out[t] = (int32_t)lo;
}

// the per-slot arrays, the padding of every entry list and the active-tile list
__global__ void k_slots(const int64_t* __restrict__ slot_key, const int32_t* __restrict__ slot_pair0,
                        const int64_t* __restrict__ padded, const int64_t* __restrict__ pad_scan,
                        const int32_t* __restrict__ tile_head, const int32_t* __restrict__ tile_scan, int32_t n_slots,
                        int32_t n_pairs, int32_t n_bus, int32_t* __restrict__ slot_row, int2* __restrict__ slot_rec,
                        PairEnt* __restrict__ pairs, int32_t* __restrict__ active, int32_t* __restrict__ ident) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const int64_t tile = slot_key[s] / n_bus;
  slot_row[s] = (int32_t)(slot_key[s] - tile * n_bus);
  const int64_t first = pad_scan[s] - padded[s];
  slot_rec[s] = make_int2((int)first, (int)(padded[s] / PAIR_PAD));
  const int32_t c = (s + 1 < n_slots ? slot_pair0[s + 1] : n_pairs) - slot_pair0[s];
  for (int64_t j = first + c; j < first + padded[s]; ++j) {
    PairEnt pad;
    pad.off = PAD_OFF;
    pad.w = 0.f;
    pairs[j] = pad;
  }
  if (tile_head[s]) active[tile_scan[s] - 1] = (int32_t)tile;
  if (ident) ident[s] = (int32_t)s;
}

// one thread per (slot, stage) pair: its weight (duplicates summed in CSR order), its entry and,
// for fused plans, its place in the slot's dense weight vector, where a stored entry whose float32
// weight is 0 becomes -0.0f (unstored cells stay +0.0f: the exact path multiplies stored entries)
__global__ void k_pairs(const unsigned long long* __restrict__ key, const int32_t* __restrict__ pos,
                        const double* __restrict__ data, const int32_t* __restrict__ pair_id,
                        const int32_t* __restrict__ slot_id, const int32_t* __restrict__ slot_pair0,
                        const int64_t* __restrict__ padded, const int64_t* __restrict__ pad_scan, int64_t nnz,
                        PairEnt* __restrict__ pairs, float* __restrict__ w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz || (i && key[i] == key[i - 1])) return;
  const int32_t s = slot_id[i] - 1;
  float wt = host_f32(data[pos[i]]);
  for (int64_t j = i + 1; j < nnz && key[j] == key[i]; ++j) wt = host_add(wt, host_f32(data[pos[j]]));
  const unsigned stage = (unsigned)(key[i] & 127u);
  PairEnt e;
  e.off = stage * 8u;
  e.w = wt;
  pairs[pad_scan[s] - padded[s] + (pair_id[i] - 1 - slot_pair0[s])] = e;
  if (w) {
    const int local = 4 * (stage & 31) + (stage >> 5);  // inverse of stage_index
    w[(size_t)s * TILE_CELLS + local] = (__float_as_uint(wt) & 0x7fffffffu) ? wt : __uint_as_float(0x80000000u);
  }
}

__global__ void k_vals(const double* __restrict__ data, int64_t nnz, float* __restrict__ vals) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < nnz) vals[k] = host_f32(data[k]);
}

// stream-ordered scratch, released on every return path
struct Scratch {
  cudaStream_t st;
  std::vector<void*> held;
  explicit Scratch(cudaStream_t s) : st(s) {}
  ~Scratch() {
    for (void* p : held) cudaFreeAsync(p, st);  // stream-ordered: after the kernels that use them
  }
  template <typename T>
  cudaError_t get(T** p, int64_t n) {
    *p = nullptr;
    cudaError_t e = cudaMallocAsync((void**)p, (size_t)std::max<int64_t>(n, 1) * sizeof(T), st);
    if (e == cudaSuccess) held.push_back(*p);
    return e;
  }
};

int bits_for(unsigned long long max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

}  // namespace

int check_plan_shape(int32_t ny, int32_t nx, int32_t& pitch, int32_t n_bus) {
  ATL_REQUIRE(ny > 0 && nx > 0 && n_bus >= 0, "bad plan shape");
  if (pitch <= 0) pitch = nx;
  ATL_REQUIRE(pitch >= nx, "pitch must be >= nx");
  ATL_REQUIRE((int64_t)ny * pitch < (1LL << 29), "grid too large (ny*pitch must be < 2^29)");
  return ATL_OK;
}

// The device plan builder behind atl_plan_create_device and the host-array entry points.
// `entries`: see plan_create in plan.cu.  Everything runs on `st`; the plan is complete on return.
int plan_build_device(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus, int64_t nnz,
                      const int64_t* indptr, const int32_t* indices, const double* data, bool entries,
                      cudaStream_t st, AtlPlan** plan_out) {
  ATL_REQUIRE(plan_out, "plan_out is NULL");
  *plan_out = nullptr;
  if (int rc = check_plan_shape(ny, nx, pitch, n_bus)) return rc;
  ATL_REQUIRE(nnz >= 0, "indptr not monotone");
  ATL_REQUIRE(indptr && (nnz == 0 || (indices && data)), "CSR arrays missing");
  // every entry is a pair of the plan, and the plan indexes pairs (and slots) with int32
  ATL_REQUIRE(nnz < (1LL << 31), "too many matrix entries for one plan");
  ATL_CUDA(cudaSetDevice(device));
  const GridDev gd = make_grid(ny, nx, pitch);
  const bool vec = (pitch % 4 == 0);
  const int64_t n_tiles = (int64_t)gd.n_tx * gd.n_ty;

  Scratch sc(st);
  int* d_err;
  Counts* d_counts;
  ATL_CUDA(sc.get(&d_err, 1));
  ATL_CUDA(sc.get(&d_counts, 1));
  ATL_CUDA(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  k_check_indptr<<<blocks_for((int64_t)n_bus + 1), BUILD_THREADS, 0, st>>>(indptr, n_bus, nnz, d_err);
  ++g_launches;

  // entry-level arrays (nnz items) and slot-level ones (n_slots <= nnz items)
  unsigned long long *key_in = nullptr, *key = nullptr;
  int32_t *pos_in = nullptr, *pos = nullptr, *pair_id = nullptr, *slot_id = nullptr, *slot_pair0 = nullptr,
          *tile_head = nullptr, *tile_scan = nullptr;
  int64_t *slot_key = nullptr, *padded = nullptr, *pad_scan = nullptr;
  char* temp = nullptr;
  size_t temp_bytes = 0;
  if (nnz > 0) {
    const int n = (int)nnz;
    ATL_CUDA(sc.get(&key_in, nnz));
    ATL_CUDA(sc.get(&key, nnz));
    ATL_CUDA(sc.get(&pos_in, nnz));
    ATL_CUDA(sc.get(&pos, nnz));
    ATL_CUDA(sc.get(&pair_id, nnz));
    ATL_CUDA(sc.get(&slot_id, nnz));
    ATL_CUDA(sc.get(&slot_pair0, nnz));
    ATL_CUDA(sc.get(&tile_head, nnz));
    ATL_CUDA(sc.get(&tile_scan, nnz));
    ATL_CUDA(sc.get(&slot_key, nnz));
    ATL_CUDA(sc.get(&padded, nnz));
    ATL_CUDA(sc.get(&pad_scan, nnz));
    size_t b = 0;
    ATL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, key_in, key, pos_in, pos, n, 0, 64, st));
    temp_bytes = std::max(temp_bytes, b);
    ATL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, pos_in, pos_in, pos, pos, n, 0, 32, st));
    temp_bytes = std::max(temp_bytes, b);
    ATL_CUDA(cub::DeviceScan::InclusiveSum(nullptr, b, pair_id, pair_id, n, st));
    temp_bytes = std::max(temp_bytes, b);
    ATL_CUDA(cub::DeviceScan::InclusiveSum(nullptr, b, padded, pad_scan, n, st));
    temp_bytes = std::max(temp_bytes, b);
    ATL_CUDA(sc.get(&temp, (int64_t)temp_bytes));

    const unsigned g = blocks_for(nnz);
    k_entry_keys<<<g, BUILD_THREADS, 0, st>>>(indptr, indices, n_bus, nnz, nx, gd.S_out, gd.n_tx, vec, key_in,
                                              pos_in, d_err);
    const int end_bit = bits_for(((unsigned long long)n_tiles * (unsigned long long)n_bus) << 7);
    size_t tb = temp_bytes;
    ATL_CUDA(cub::DeviceRadixSort::SortPairs(temp, tb, key_in, key, pos_in, pos, n, 0, end_bit, st));
    // the flags are scanned in place into running counts (1-based ids)
    k_entry_heads<<<g, BUILD_THREADS, 0, st>>>(key, nnz, pair_id, slot_id);
    tb = temp_bytes;
    ATL_CUDA(cub::DeviceScan::InclusiveSum(temp, tb, pair_id, pair_id, n, st));
    tb = temp_bytes;
    ATL_CUDA(cub::DeviceScan::InclusiveSum(temp, tb, slot_id, slot_id, n, st));
    k_slot_starts<<<g, BUILD_THREADS, 0, st>>>(key, pair_id, slot_id, nnz, slot_key, slot_pair0);
    k_slot_counts<<<g, BUILD_THREADS, 0, st>>>(slot_key, slot_pair0, pair_id, slot_id, nnz, n_bus, padded, tile_head);
    tb = temp_bytes;
    ATL_CUDA(cub::DeviceScan::InclusiveSum(temp, tb, padded, pad_scan, n, st));
    tb = temp_bytes;
    ATL_CUDA(cub::DeviceScan::InclusiveSum(temp, tb, tile_head, tile_scan, n, st));
    g_launches += 4;
  }
  k_counts<<<1, 1, 0, st>>>(pair_id, slot_id, tile_scan, pad_scan, nnz, d_err, d_counts);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  Counts cnt;
  ATL_CUDA(cudaMemcpyAsync(&cnt, d_counts, sizeof(Counts), cudaMemcpyDeviceToHost, st));
  ATL_CUDA(cudaStreamSynchronize(st));
  ATL_REQUIRE(!(cnt.err & ERR_MONOTONE), "indptr not monotone");
  ATL_REQUIRE(!(cnt.err & ERR_COLUMN), "column index out of range");
  ATL_REQUIRE(!(cnt.err & ERR_ENDS), "indptr must start at 0 and end at nnz");

  const int64_t n_slots = cnt.n_slots;
  // A matrix "tiles well" when a tile is touched by few buses (the same rule as build_tiling).
  const double spt = cnt.n_active ? (double)n_slots / (double)cnt.n_active : 0.0;
  const bool fused = spt <= 24.0 && (double)n_slots * TILE_CELLS * 4.0 <= 4.0e9;
  if (fused || entries) ATL_REQUIRE(cnt.n_padded < (1LL << 31), "too many matrix entries for one plan");

  AtlPlan* p = new AtlPlan();
  p->device = device;
  p->grid = gd;
  p->n_bus = n_bus;
  p->nnz = nnz;
  p->n_tiles = (int32_t)n_tiles;
  p->n_active = cnt.n_active;
  p->n_slots = n_slots;
  p->fused = fused;
  p->vec = vec;
  auto fail = [&](int rc) {
    cudaStreamSynchronize(st);
    atl_plan_destroy(p);
    return rc;
  };
#define PLAN_CUDA(call)                                       \
  do {                                                        \
    cudaError_t _e = (call);                                  \
    if (_e != cudaSuccess) return fail(cuda_fail(_e, #call)); \
  } while (0)
  auto alloc = [&](auto** ptr, int64_t n) {
    return cudaMalloc((void**)ptr, (size_t)std::max<int64_t>(n, 1) * sizeof(**ptr));
  };

  if (fused || entries) {
    p->n_pairs = cnt.n_pairs;
    p->n_pairs_padded = cnt.n_padded;
    PLAN_CUDA(alloc(&p->d_tile_slot_ptr, n_tiles + 1));
    PLAN_CUDA(alloc(&p->d_slot_row, n_slots));
    PLAN_CUDA(alloc(&p->d_slot_rec, n_slots));
    PLAN_CUDA(alloc(&p->d_pairs, cnt.n_padded));
    PLAN_CUDA(alloc(&p->d_active, cnt.n_active));
    if (fused) {
      // + 3 zero slots: the grouped reduce (reduce_slots2g) reads up to 3 weight vectors past a
      // tile's last slot (their sums are discarded)
      const int64_t n_w4 = (n_slots + 3) * (TILE_CELLS / 4);
      PLAN_CUDA(alloc(&p->d_slot_w4, n_w4));
      PLAN_CUDA(cudaMemsetAsync(p->d_slot_w4, 0, (size_t)n_w4 * sizeof(float4), st));
      PLAN_CUDA(alloc(&p->d_slot_ident, n_slots));
      PLAN_CUDA(alloc(&p->d_row_slot_ptr, (int64_t)n_bus + 1));
      PLAN_CUDA(alloc(&p->d_row_slots, n_slots));
    }
    k_lower_bounds<<<blocks_for(n_tiles + 1), BUILD_THREADS, 0, st>>>(slot_key, n_slots, (int64_t)n_bus,
                                                                      p->d_tile_slot_ptr, n_tiles + 1);
    ++g_launches;
    if (n_slots > 0) {
      k_slots<<<blocks_for(n_slots), BUILD_THREADS, 0, st>>>(slot_key, slot_pair0, padded, pad_scan, tile_head,
                                                             tile_scan, (int32_t)n_slots, cnt.n_pairs, n_bus,
                                                             p->d_slot_row, p->d_slot_rec, p->d_pairs, p->d_active,
                                                             p->d_slot_ident);
      k_pairs<<<blocks_for(nnz), BUILD_THREADS, 0, st>>>(key, pos, data, pair_id, slot_id, slot_pair0, padded,
                                                         pad_scan, nnz, p->d_pairs,
                                                         fused ? (float*)p->d_slot_w4 : nullptr);
      g_launches += 2;
    }
    if (fused) {
      // deterministic mode: the slots of every bus in ascending slot (= tile) order -- a stable
      // sort of the slot ids by bus -- and where each bus's list starts
      int32_t* bus_sorted = pos_in;  // free again after the entry sort; n_slots <= nnz
      if (n_slots > 0) {
        size_t tb = temp_bytes;
        PLAN_CUDA(cub::DeviceRadixSort::SortPairs(temp, tb, p->d_slot_row, bus_sorted, p->d_slot_ident,
                                                  p->d_row_slots, (int)n_slots, 0,
                                                  bits_for((unsigned long long)std::max(n_bus - 1, 1)), st));
        ++g_launches;
      }
      k_lower_bounds<<<blocks_for((int64_t)n_bus + 1), BUILD_THREADS, 0, st>>>(bus_sorted, n_slots, 1,
                                                                               p->d_row_slot_ptr, (int64_t)n_bus + 1);
      ++g_launches;
    }
  }
  // CSR copy (float weights) for the gather SpMM
  PLAN_CUDA(alloc(&p->d_indptr, (int64_t)n_bus + 1));
  PLAN_CUDA(alloc(&p->d_indices, nnz));
  PLAN_CUDA(alloc(&p->d_vals, nnz));
  PLAN_CUDA(cudaMemcpyAsync(p->d_indptr, indptr, ((size_t)n_bus + 1) * 8, cudaMemcpyDeviceToDevice, st));
  if (nnz > 0) {
    PLAN_CUDA(cudaMemcpyAsync(p->d_indices, indices, (size_t)nnz * 4, cudaMemcpyDeviceToDevice, st));
    k_vals<<<blocks_for(nnz), BUILD_THREADS, 0, st>>>(data, nnz, p->d_vals);
    ++g_launches;
  }
  PLAN_CUDA(cudaGetLastError());
  PLAN_CUDA(cudaStreamSynchronize(st));
#undef PLAN_CUDA
  *plan_out = p;
  return ATL_OK;
}

}  // namespace atl

extern "C" {

int atl_plan_create_device(int device, int32_t ny, int32_t nx, int32_t pitch, int32_t n_bus, int64_t nnz,
                           const int64_t* indptr_dev, const int32_t* indices_dev, const double* data_dev,
                           int entries, void* stream, AtlPlan** plan_out) {
  return atl::plan_build_device(device, ny, nx, pitch, n_bus, nnz, indptr_dev, indices_dev, data_dev, entries != 0,
                                (cudaStream_t)stream, plan_out);
}

int atl_plan_export(const AtlPlan* plan, int32_t array_id, void* dst_host, int64_t capacity_bytes,
                    int64_t* bytes_out) {
  ATL_REQUIRE(plan && bytes_out, "NULL argument");
  const int64_t ns = plan->n_slots;
  const void* src = nullptr;
  int64_t bytes = 0;
  switch (array_id) {
    case ATL_PLAN_TILE_SLOT_PTR: src = plan->d_tile_slot_ptr; bytes = ((int64_t)plan->n_tiles + 1) * 4; break;
    case ATL_PLAN_SLOT_ROW: src = plan->d_slot_row; bytes = ns * 4; break;
    case ATL_PLAN_SLOT_W4: src = plan->d_slot_w4; bytes = (ns + 3) * atl::TILE_CELLS * 4; break;
    case ATL_PLAN_SLOT_REC: src = plan->d_slot_rec; bytes = ns * 8; break;
    case ATL_PLAN_PAIRS: src = plan->d_pairs; bytes = plan->n_pairs_padded * 8; break;
    case ATL_PLAN_ACTIVE: src = plan->d_active; bytes = (int64_t)plan->n_active * 4; break;
    case ATL_PLAN_SLOT_IDENT: src = plan->d_slot_ident; bytes = ns * 4; break;
    case ATL_PLAN_ROW_SLOT_PTR: src = plan->d_row_slot_ptr; bytes = ((int64_t)plan->n_bus + 1) * 4; break;
    case ATL_PLAN_ROW_SLOTS: src = plan->d_row_slots; bytes = ns * 4; break;
    case ATL_PLAN_INDPTR: src = plan->d_indptr; bytes = ((int64_t)plan->n_bus + 1) * 8; break;
    case ATL_PLAN_INDICES: src = plan->d_indices; bytes = plan->nnz * 4; break;
    case ATL_PLAN_VALS: src = plan->d_vals; bytes = plan->nnz * 4; break;
    default: ATL_REQUIRE(false, "unknown plan array");
  }
  if (!src) bytes = 0;  // not part of this plan
  *bytes_out = bytes;
  if (!dst_host || bytes == 0) return ATL_OK;
  ATL_REQUIRE(capacity_bytes >= bytes, "capacity_bytes too small");
  ATL_CUDA(cudaSetDevice(plan->device));
  ATL_CUDA(cudaMemcpy(dst_host, src, (size_t)bytes, cudaMemcpyDeviceToHost));
  return ATL_OK;
}

}  // extern "C"
