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
// Host code only (compiled by nvcc with the rest of the library; zlib does the inflate).
#include <fcntl.h>
#include <unistd.h>
#include <zlib.h>

#include <atomic>
#include <mutex>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

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

}  // extern "C"
