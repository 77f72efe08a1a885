// decode.cu -- cutout ingest: decode compressed chunks of a (time, y, x) variable straight
// into a host slab (pinned or pageable), on many host threads.
//
// The reference stores cutouts as NetCDF-4 / HDF5 with zlib level 9 + byte shuffle
// (atlite/data.py:139,245-248) and reads them back through
// xarray -> netCDF4 -> libhdf5, which inflates chunk after chunk on ONE thread while holding a
// global lock.  Here the hot part of that read -- pread of the raw chunk, inflate, un-shuffle,
// scatter into the slab -- runs as a parallel loop over chunks; the (cold) metadata, i.e. where
// each chunk lives in the file, comes from the caller as a chunk index (atlite_b200/ingest.py
// builds it with h5py when that is installed, or reads a kerchunk-style JSON side-car).
//
// atl_decode_chunks runs on host threads (zlib does the inflate) and fills host slabs.
// atl_decode_chunks_device fills device tensors: the chunks cross PCIe compressed through the
// batch pipeline of inflate.cu, k_inflate decodes them on the GPU and k_chunk_scatter un-shuffles,
// converts to float32 and scatters them into the destination.
#include <fcntl.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <cstddef>
#include <mutex>
#include <cstring>
#include <set>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "inflate.cuh"

using namespace atl;

namespace {

// HDF5 shuffle filter (H5Zshuffle.c semantics): byte k of element i is stored at k * n + i.
void unshuffle(const uint8_t* src, uint8_t* dst, size_t n_elem, size_t elem) {
  if (elem == 4) {
    const uint8_t *b0 = src, *b1 = src + n_elem, *b2 = src + 2 * n_elem, *b3 = src + 3 * n_elem;
    for (size_t i = 0; i < n_elem; ++i) {
      dst[4 * i] = b0[i];
      dst[4 * i + 1] = b1[i];
      dst[4 * i + 2] = b2[i];
      dst[4 * i + 3] = b3[i];
    }
    return;
  }
  for (size_t k = 0; k < elem; ++k)
    for (size_t i = 0; i < n_elem; ++i) dst[i * elem + k] = src[k * n_elem + i];
}


// ---------------------------------------------------------------- device path
struct ChunkDev {
  InflSpan span;  // compressed bytes in the transfer buffer, decoded bytes in the decode buffer
  int64_t ot, oy, ox;
};
static_assert(offsetof(ChunkDev, span) == 0, "k_inflate reads the span at the start of the descriptor");

struct ScatterArgs {
  int64_t ct, cy, cx;           // chunk shape
  int64_t t0, nt, y0, wy, x0, wx, pitch;
  int32_t shuffle;
  AtlChunkConvert conv;
};

// IEEE operations without flushing subnormals (the library builds with -ftz=true; the host does not
// flush), and with NaN operands propagated as x86 SSE does: the first NaN operand, quietened.
__device__ __forceinline__ bool f32_isnan(float v) { return (__float_as_uint(v) & 0x7fffffffu) > 0x7f800000u; }
__device__ __forceinline__ float f32_quiet(float v) { return __uint_as_float(__float_as_uint(v) | 0x00400000u); }
__device__ __forceinline__ float mul_sse(float a, float b) {
  if (f32_isnan(a)) return f32_quiet(a);
  if (f32_isnan(b)) return f32_quiet(b);
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float add_sse(float a, float b) {
  if (f32_isnan(a)) return f32_quiet(a);
  if (f32_isnan(b)) return f32_quiet(b);
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ double f32_to_f64(float v) {
  double r;
  asm("cvt.f64.f32 %0, %1;" : "=d"(r) : "f"(v));
  return r;
}
__device__ __forceinline__ float f64_to_f32(double v) {  // cvtsd2ss: a NaN keeps sign and top payload bits
  const uint64_t b = (uint64_t)__double_as_longlong(v);
  if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull)
    return __uint_as_float((uint32_t)(b >> 32 & 0x80000000u) | 0x7fc00000u | (uint32_t)(b >> 29 & 0x003fffffu));
  float r;
  asm("cvt.rn.f32.f64 %0, %1;" : "=f"(r) : "d"(v));
  return r;
}

template <int E>
__device__ __forceinline__ uint64_t bswap_n(uint64_t v) {
  if constexpr (E == 2) {
    return ((v & 0xff) << 8) | ((v >> 8) & 0xff);
  } else if constexpr (E == 4) {
    return __byte_perm((uint32_t)v, 0, 0x0123);
  } else {
    return ((uint64_t)__byte_perm((uint32_t)v, 0, 0x0123) << 32) | __byte_perm((uint32_t)(v >> 32), 0, 0x0123);
  }
}

// One raw element (E bytes as stored, in the low bytes of `bits`) -> float32, as ChunkedVariable.load.
template <int E>
__device__ __forceinline__ float chunk_convert(uint64_t bits, const AtlChunkConvert& c) {
  if (c.big_endian) bits = bswap_n<E>(bits);
  if (!c.convert) return __uint_as_float((uint32_t)bits);
  float v;
  bool fill = false;
  if (c.kind == ATL_RAW_FLOAT) {
    if constexpr (E == 8) {
      const double d = __longlong_as_double((long long)bits);
      v = f64_to_f32(d);
      fill = c.has_fill && d == c.fill;
    } else if constexpr (E == 4) {
      v = __uint_as_float((uint32_t)bits);
      fill = c.has_fill && f32_to_f64(v) == c.fill;
    } else {
      v = 0.f;  // float16 is refused on the host
    }
  } else {
    int64_t i;
    if (c.kind == ATL_RAW_INT) {
      i = E == 2 ? (int64_t)(int16_t)bits : E == 4 ? (int64_t)(int32_t)bits : (int64_t)bits;
      v = E == 8 ? __ll2float_rn(i) : __int2float_rn((int)i);
    } else {
      i = (int64_t)bits;
      v = E == 8 ? __ull2float_rn(bits) : __uint2float_rn((uint32_t)bits);
    }
    if (c.has_fill)
      fill = c.fill_as_int ? i == c.fill_int
                           : (c.kind == ATL_RAW_INT ? (double)i : (double)(uint64_t)bits) == c.fill;
  }
  if (fill) v = __uint_as_float(0x7fc00000u);  // NumPy's NaN
  if (c.has_scale) v = mul_sse(v, c.scale);
  if (c.has_offset) v = add_sse(v, c.offset);
  return v;
}

constexpr int SCATTER_THREADS = 256;

// Block (k, part): rows (t, y) of chunk k's part of the window, one warp per row, lanes along x.
template <int E>
__global__ void __launch_bounds__(SCATTER_THREADS) k_chunk_scatter(const uint8_t* __restrict__ dec,
                                                                   const ChunkDev* __restrict__ chunks, ScatterArgs A,
                                                                   float* __restrict__ dst) {
  const ChunkDev g = chunks[blockIdx.x];
  const int64_t ta = max(g.ot, A.t0), tb = min(g.ot + A.ct, A.t0 + A.nt);
  const int64_t ya = max(g.oy, A.y0), yb = min(g.oy + A.cy, A.y0 + A.wy);
  const int64_t xa = max(g.ox, A.x0), xb = min(g.ox + A.cx, A.x0 + A.wx);
  if (ta >= tb || ya >= yb || xa >= xb) return;
  const int64_t rows = (tb - ta) * (yb - ya), n_elem = A.ct * A.cy * A.cx;
  const uint8_t* base = dec + g.span.out_off;
  const int lane = threadIdx.x & 31, warps = SCATTER_THREADS / 32;
  for (int64_t r = (int64_t)blockIdx.y * warps + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.y * warps) {
    const int64_t t = ta + r / (yb - ya), y = ya + r % (yb - ya);
    const int64_t row = ((t - g.ot) * A.cy + (y - g.oy)) * A.cx - g.ox;  // element index of column 0
    float* o = dst + ((t - A.t0) * A.wy + (y - A.y0)) * A.pitch - A.x0;
    for (int64_t x = xa + lane; x < xb; x += 32) {
      const int64_t i = row + x;
      uint64_t bits = 0;
      if (A.shuffle) {
#pragma unroll
        for (int k = 0; k < E; ++k) bits |= (uint64_t)base[(int64_t)k * n_elem + i] << (8 * k);
      } else if constexpr (E == 2) {
        bits = reinterpret_cast<const uint16_t*>(base)[i];
      } else if constexpr (E == 4) {
        bits = reinterpret_cast<const uint32_t*>(base)[i];
      } else {
        bits = reinterpret_cast<const uint64_t*>(base)[i];
      }
      o[x] = chunk_convert<E>(bits, A.conv);
    }
  }
}

// Every window element as a raw zero converts (chunks missing from the index), padding columns 0.
template <int E>
__global__ void k_chunk_fill(float* dst, int64_t rows, int64_t wx, int64_t pitch, AtlChunkConvert conv) {
  const float v = chunk_convert<E>(0, conv);
  const int64_t n = rows * pitch;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = i % pitch < wx ? v : 0.f;
}

template <int E>
cudaError_t launch_scatter(const uint8_t* dec, const ChunkDev* chunks, int n, int64_t max_rows, const ScatterArgs& A,
                           float* dst, cudaStream_t st) {
  const int parts = (int)std::min<int64_t>(std::max<int64_t>(1, (max_rows + 63) / 64), 256);
  k_chunk_scatter<E><<<dim3(n, parts), SCATTER_THREADS, 0, st>>>(dec, chunks, A, dst);
  ++g_launches;
  return cudaGetLastError();
}

template <int E>
cudaError_t launch_fill(float* dst, int64_t rows, int64_t wx, int64_t pitch, const AtlChunkConvert& c,
                        cudaStream_t st) {
  const int64_t n = rows * pitch;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, 16 * sm_count());
  k_chunk_fill<E><<<grid, 256, 0, st>>>(dst, rows, wx, pitch, c);
  ++g_launches;
  return cudaGetLastError();
}

}  // namespace

extern "C" {

int atl_decode_chunks(const char* path, const AtlChunkSpec* spec, int64_t n_chunks,
                      const int64_t* file_offset, const int64_t* stored_bytes,
                      const int64_t* chunk_origin /* n_chunks x 3: (t, y, x) of the chunk's first element */,
                      int64_t t0, int64_t nt, void* dst_host, int32_t n_threads) {
  using namespace atl;
  ATL_REQUIRE(path && spec && dst_host, "NULL argument");
  ATL_REQUIRE(n_chunks >= 0 && (n_chunks == 0 || (file_offset && stored_bytes && chunk_origin)), "chunk index missing");
  ATL_REQUIRE(spec->elem_bytes == 4 || spec->elem_bytes == 8 || spec->elem_bytes == 2, "element size must be 2, 4 or 8");
  ATL_REQUIRE(spec->chunk[0] > 0 && spec->chunk[1] > 0 && spec->chunk[2] > 0, "bad chunk shape");
  ATL_REQUIRE(spec->ny > 0 && spec->nx > 0 && nt >= 0 && t0 >= 0, "bad variable shape");
  if (nt == 0 || n_chunks == 0) return ATL_OK;
  const int fd = open(path, O_RDONLY);
  if (fd < 0) {
    set_error(std::string("cannot open ") + path);
    return ATL_ERR_INVALID;
  }
  const size_t elem = (size_t)spec->elem_bytes;
  const int64_t ct = spec->chunk[0], cy = spec->chunk[1], cx = spec->chunk[2];
  const size_t n_elem = (size_t)ct * cy * cx, raw_bytes = n_elem * elem;
  unsigned hw = std::thread::hardware_concurrency();
  int nthr = n_threads > 0 ? n_threads : (int)(hw ? hw : 4);
  if (nthr > 64) nthr = 64;
  if ((int64_t)nthr > n_chunks) nthr = (int)n_chunks;
  std::atomic<int64_t> next{0};
  std::atomic<int> failed{0};
  std::string err;
  std::mutex err_mu;
  auto fail = [&](const std::string& m) {
    std::lock_guard<std::mutex> lk(err_mu);
    if (!failed.exchange(1)) err = m;
  };
  auto worker = [&]() {
    std::vector<uint8_t> comp, raw(raw_bytes), plain(spec->shuffle ? raw_bytes : 0);
    for (;;) {
      const int64_t c = next.fetch_add(1);
      if (c >= n_chunks || failed.load()) return;
      const int64_t ot = chunk_origin[3 * c], oy = chunk_origin[3 * c + 1], ox = chunk_origin[3 * c + 2];
      // rows of this chunk that fall into [t0, t0 + nt) x the grid (edge chunks are stored whole)
      const int64_t ta = ot > t0 ? ot : t0, tb = (ot + ct < t0 + nt) ? ot + ct : t0 + nt;
      if (ta >= tb || oy >= spec->ny || ox >= spec->nx) continue;
      const size_t sb = (size_t)stored_bytes[c];
      comp.resize(sb);
      size_t got = 0;
      while (got < sb) {
        const ssize_t r = pread(fd, comp.data() + got, sb - got, (off_t)(file_offset[c] + (int64_t)got));
        if (r <= 0) {
          fail("short read of a chunk");
          return;
        }
        got += (size_t)r;
      }
      const uint8_t* data = comp.data();
      if (spec->deflate) {
        uLongf out_len = (uLongf)raw_bytes;
        const int zr = uncompress(raw.data(), &out_len, comp.data(), (uLong)sb);
        if (zr != Z_OK || out_len != raw_bytes) {
          fail("zlib: corrupt chunk or wrong chunk shape");
          return;
        }
        data = raw.data();
      } else if (sb != raw_bytes) {
        fail("uncompressed chunk has the wrong size");
        return;
      }
      if (spec->shuffle) {
        unshuffle(data, plain.data(), n_elem, elem);
        data = plain.data();
      }
      const int64_t ya = oy, yb = (oy + cy < spec->ny) ? oy + cy : spec->ny;
      const int64_t xb = (ox + cx < spec->nx) ? ox + cx : spec->nx;
      const size_t run = (size_t)(xb - ox) * elem;
      for (int64_t t = ta; t < tb; ++t)
        for (int64_t y = ya; y < yb; ++y) {
          const uint8_t* s = data + (((size_t)(t - ot) * cy + (size_t)(y - oy)) * cx) * elem;
          uint8_t* d = (uint8_t*)dst_host + (((size_t)(t - t0) * spec->ny + (size_t)y) * spec->nx + (size_t)ox) * elem;
          std::memcpy(d, s, run);
        }
    }
  };
  std::vector<std::thread> th;
  for (int k = 1; k < nthr; ++k) th.emplace_back(worker);
  worker();
  for (auto& t : th) t.join();
  close(fd);
  if (failed.load()) {
    set_error(err);
    return ATL_ERR_INVALID;
  }
  return ATL_OK;
}

int atl_decode_chunks_device(int device, const char* path, const AtlChunkSpec* spec, int64_t n_chunks,
                             const int64_t* file_offset, const int64_t* stored_bytes,
                             const int64_t* chunk_origin, int64_t t0, int64_t nt, int64_t y0, int64_t wy,
                             int64_t x0, int64_t wx, const AtlChunkConvert* conv, float* dst_dev,
                             int64_t pitch, int64_t batch_bytes, int32_t n_threads, void* stream) {
  using namespace atl;
  ATL_REQUIRE(path && spec && conv && dst_dev, "NULL argument");
  ATL_REQUIRE(n_chunks >= 0 && (n_chunks == 0 || (file_offset && stored_bytes && chunk_origin)), "chunk index missing");
  const int E = spec->elem_bytes;
  ATL_REQUIRE(E == 4 || E == 8 || E == 2, "element size must be 2, 4 or 8");
  ATL_REQUIRE(spec->chunk[0] > 0 && spec->chunk[1] > 0 && spec->chunk[2] > 0, "bad chunk shape");
  ATL_REQUIRE(spec->ny > 0 && spec->nx > 0 && nt >= 0 && t0 >= 0, "bad variable shape");
  ATL_REQUIRE(y0 >= 0 && wy >= 0 && y0 + wy <= spec->ny && x0 >= 0 && wx >= 0 && x0 + wx <= spec->nx,
              "window outside the grid");
  ATL_REQUIRE(pitch >= wx, "pitch below the window width");
  ATL_REQUIRE(conv->kind == ATL_RAW_FLOAT || conv->kind == ATL_RAW_INT || conv->kind == ATL_RAW_UINT, "bad element kind");
  ATL_REQUIRE(conv->convert || (conv->kind == ATL_RAW_FLOAT && E == 4), "only float32 elements are copied as they are");
  ATL_REQUIRE(conv->kind != ATL_RAW_FLOAT || E != 2, "float16 elements are not supported");
  ATL_REQUIRE(batch_bytes > 0, "batch_bytes must be positive");
  if (nt == 0 || wy == 0 || pitch == 0) return ATL_OK;
  const int64_t ct = spec->chunk[0], cy = spec->chunk[1], cx = spec->chunk[2];
  const int64_t raw_bytes = ct * cy * cx * E;
  const bool deflate = spec->deflate != 0;

  // the chunks that meet the window, and whether the index covers every chunk position it meets
  std::vector<int64_t> sel;
  std::set<std::tuple<int64_t, int64_t, int64_t>> present;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const int64_t ot = chunk_origin[3 * c], oy = chunk_origin[3 * c + 1], ox = chunk_origin[3 * c + 2];
    if (ot + ct <= t0 || ot >= t0 + nt || oy + cy <= y0 || oy >= y0 + wy || ox + cx <= x0 || ox >= x0 + wx) continue;
    sel.push_back(c);
    present.emplace(ot, oy, ox);
  }
  auto span_of = [](int64_t lo, int64_t n, int64_t c) { return (lo + n - 1) / c - lo / c + 1; };
  const bool missing = wx > 0 && (int64_t)present.size() < span_of(t0, nt, ct) * span_of(y0, wy, cy) * span_of(x0, wx, cx);

  // descriptors and batches: consecutive chunks whose compressed and decoded bytes fit batch_bytes
  const int64_t n_sel = (int64_t)sel.size();
  std::vector<ChunkDev> desc(n_sel);
  std::vector<int64_t> offs(n_sel), reads(n_sel), xoff(n_sel);
  SegmentBatches S;
  S.batch_start.push_back(0);
  int64_t bx = 0, bd = 0, max_dec = 0, max_rows = 0;
  for (int64_t k = 0; k < n_sel; ++k) {
    const int64_t c = sel[k];
    if (!deflate && stored_bytes[c] != raw_bytes) {
      set_error("uncompressed chunk has the wrong size");
      return ATL_ERR_INVALID;
    }
    ChunkDev& g = desc[k];
    g.ot = chunk_origin[3 * c];
    g.oy = chunk_origin[3 * c + 1];
    g.ox = chunk_origin[3 * c + 2];
    g.span.in_bytes = stored_bytes[c];
    g.span.out_bytes = raw_bytes;
    const int64_t x = seg_align_up(stored_bytes[c]), d = deflate ? seg_align_up(raw_bytes) : 0;
    if (k > S.batch_start.back() && (bx + x > batch_bytes || bd + d > batch_bytes)) {
      S.batch_start.push_back(k);
      bx = bd = 0;
    }
    g.span.in_off = bx;
    g.span.out_off = deflate ? bd : bx;
    bx += x;
    bd += d;
    S.max_xfer = std::max(S.max_xfer, bx);
    max_dec = std::max(max_dec, bd);
    offs[k] = file_offset[c];
    reads[k] = stored_bytes[c];
    xoff[k] = g.span.in_off;
    const int64_t rt = std::min(g.ot + ct, t0 + nt) - std::max(g.ot, t0);
    const int64_t ry = std::min(g.oy + cy, y0 + wy) - std::max(g.oy, y0);
    max_rows = std::max(max_rows, rt * ry);
  }
  S.batch_start.push_back(n_sel);
  S.file_offset = offs.data();
  S.read_bytes = reads.data();
  S.xfer_off = xoff.data();
  S.desc = desc.data();
  S.desc_bytes = sizeof(ChunkDev);
  S.n_threads = n_threads;

  ATL_CUDA(cudaSetDevice(device));
  const cudaStream_t st = (cudaStream_t)stream;
  const AtlChunkConvert cv = *conv;
  if (missing) {
    switch (E) {
      case 2: ATL_CUDA(launch_fill<2>(dst_dev, nt * wy, wx, pitch, cv, st)); break;
      case 4: ATL_CUDA(launch_fill<4>(dst_dev, nt * wy, wx, pitch, cv, st)); break;
      default: ATL_CUDA(launch_fill<8>(dst_dev, nt * wy, wx, pitch, cv, st)); break;
    }
  } else if (pitch > wx) {
    ATL_CUDA(cudaMemset2DAsync(dst_dev + wx, pitch * sizeof(float), 0, (pitch - wx) * sizeof(float), nt * wy, st));
  }
  if (n_sel == 0) {
    ATL_CUDA(cudaStreamSynchronize(st));
    return ATL_OK;
  }

  struct DecBuffers {
    uint8_t* p[2] = {nullptr, nullptr};
    ~DecBuffers() {
      cudaFree(p[0]);
      cudaFree(p[1]);
    }
  } dec;
  if (deflate) {
    const int n_buf = S.batch_start.size() > 2 ? 2 : 1;
    for (int s = 0; s < n_buf; ++s) ATL_CUDA(cudaMalloc(&dec.p[s], std::max<int64_t>(max_dec, SEG_ALIGN)));
  }
  const ScatterArgs A{ct, cy, cx, t0, nt, y0, wy, x0, wx, pitch, spec->shuffle, cv};
  auto launch = [&](int slot, int64_t, int n, const uint8_t* xfer, const void* d, int32_t* status) -> cudaError_t {
    const ChunkDev* cd = static_cast<const ChunkDev*>(d);
    const uint8_t* src = xfer;
    if (deflate) {
      const cudaError_t e = launch_inflate(xfer, dec.p[slot], cd, sizeof(ChunkDev), n, status, st);
      if (e != cudaSuccess) return e;
      src = dec.p[slot];
    }
    switch (E) {
      case 2: return launch_scatter<2>(src, cd, n, max_rows, A, dst_dev, st);
      case 4: return launch_scatter<4>(src, cd, n, max_rows, A, dst_dev, st);
      default: return launch_scatter<8>(src, cd, n, max_rows, A, dst_dev, st);
    }
  };
  std::vector<int32_t> status;
  int64_t bad = -1;
  const int rc = run_segment_batches(device, path, S, st, launch, status, &bad);
  if (rc != ATL_OK) {
    if (bad >= 0) set_error("short read of a chunk");
    return rc;
  }
  for (int64_t k = 0; k < n_sel; ++k)
    if (status[k] != ATL_INFLATE_OK) {
      const ChunkDev& g = desc[k];
      set_error("zlib: chunk at (t, y, x) = (" + std::to_string(g.ot) + ", " + std::to_string(g.oy) + ", " +
                std::to_string(g.ox) + "): " + inflate_status_text(status[k]));
      return ATL_ERR_INVALID;
    }
  return ATL_OK;
}

}  // extern "C"
