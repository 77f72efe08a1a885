// geotiff.cu -- decode the segments (tiles or strips) of a single-band GeoTIFF into a device
// raster (atlite_b200/geotiff.py parses the file's IFD and picks the segments a window needs).
//
// What crosses PCIe is as small as the file allows: LZW and Deflate segments go to the device
// compressed and are decoded there (k_tiff_lzw here, k_inflate in inflate.cu), and uncompressed
// ones are copied as they are.  One placement kernel (k_tiff_place) then undoes the
// predictor, swaps big-endian samples and writes each segment's pixels into the window of the
// result, clipping padded edge tiles.
//
// LZW (TIFF 6.0 section 13, libtiff's tif_lzw.c conventions): codes packed MSB-first, Clear 256,
// EOI 257, first free code 258, code width 9 bits growing to 10, 11 and 12 when the next code to
// be assigned reaches 511, 1023 and 2047, reset by Clear.  Every string a code stands for is an
// earlier span of the segment's own output plus the byte that follows that span, so the table is
// (offset, length) pairs into the output and decoding a code is a copy the warp's lanes share.  One
// warp decodes one segment; its table (4096 x 6 bytes) lives in shared memory.  Every code and
// every copy is checked against the segment's output span, and a corrupt segment only sets its
// status.
//
// The I/O (atl_geotiff_read) is the batch pipeline of inflate.cu that the cutout chunks use too:
// the segments of a batch are read with parallel pread into a pinned buffer, and the next batch is
// read and copied on a copy stream while the current one decodes.
#include <algorithm>
#include <cstddef>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "inflate.cuh"

namespace atl {

constexpr int TIFF_LZW_WARPS = 4;        // decoders per CTA
constexpr int TIFF_LZW_TABLE = 4096;     // 12-bit codes
constexpr int TIFF_PLACE_THREADS = 256;  // 8 warps, one segment row each

// Begins with the fields of an InflSpan, so that k_inflate reads the segments' spans in place.
struct TiffSegDev {
  int64_t xfer_off;   // compressed (LZW, Deflate) or decoded bytes in the transfer buffer
  int64_t xfer_bytes;
  int64_t dec_off;    // decoded bytes in the buffer the placement reads
  int64_t dec_bytes;
  int32_t row0, col0, rows, cols;  // image rows / columns of the segment; cols = samples per segment row
};
static_assert(offsetof(TiffSegDev, xfer_off) == offsetof(InflSpan, in_off) &&
                  offsetof(TiffSegDev, xfer_bytes) == offsetof(InflSpan, in_bytes) &&
                  offsetof(TiffSegDev, dec_off) == offsetof(InflSpan, out_off) &&
                  offsetof(TiffSegDev, dec_bytes) == offsetof(InflSpan, out_bytes),
              "TiffSegDev must begin with an InflSpan's layout");

// ---------------------------------------------------------------- LZW
__device__ __forceinline__ int lzw_width(int next) { return next < 511 ? 9 : next < 1023 ? 10 : next < 2047 ? 11 : 12; }

// Decode one segment with the calling warp (every lane keeps the same state).  Returns an
// ATL_TIFF_* status.
__device__ int lzw_decode_warp(const uint8_t* __restrict__ in, int64_t n_in, uint8_t* out, int64_t size,
                               uint32_t* s_off, uint16_t* s_len) {
  const int lane = threadIdx.x & 31;
  if (n_in >= 2 && in[0] == 0 && (in[1] & 1)) return ATL_TIFF_LZW_OLD_STYLE;  // libtiff's test
  uint64_t acc = 0;  // the next unread bits, MSB-aligned
  int nacc = 0;
  int64_t ip = 0, pos = 0, prev_start = -1;
  int prev_len = 0, next = 258, width = 9;
  for (;;) {
    while (nacc <= 56 && ip < n_in) {
      acc |= (uint64_t)__ldg(in + ip++) << (56 - nacc);
      nacc += 8;
    }
    if (nacc < width) return pos == size ? ATL_TIFF_OK : ATL_TIFF_LZW_TRUNCATED;  // no EOI: fine once full
    const int code = (int)(acc >> (64 - width));
    acc <<= width;
    nacc -= width;
    if (code == 257) return pos == size ? ATL_TIFF_OK : ATL_TIFF_LZW_SHORT;
    if (code == 256) {
      next = 258;
      width = 9;
      prev_start = -1;
      continue;
    }
    if (pos == size) return ATL_TIFF_LZW_LONG;  // data beyond the segment's size
    if (code > next || (code == next && prev_start < 0)) return ATL_TIFF_LZW_BAD_CODE;
    int64_t off;
    int len;
    if (code < 256) {
      off = -1;
      len = 1;
    } else if (code < next) {
      off = s_off[code];
      len = s_len[code];
    } else {  // KwKwK: the previous string plus its own first byte
      off = prev_start;
      len = prev_len + 1;
    }
    if (len > size - pos) return ATL_TIFF_LZW_LONG;
    if (code < 256) {
      if (lane == 0) out[pos] = (uint8_t)code;
    } else {
      // the source span ends before pos, except for KwKwK, whose last byte is the string's first
      const int body = code < next ? len : len - 1;
      for (int k = lane; k < body; k += 32) out[pos + k] = out[off + k];
      if (code == next && lane == 0) out[pos + len - 1] = out[off];
    }
    if (prev_start >= 0 && next < TIFF_LZW_TABLE) {  // previous string + this one's first byte
      if (lane == 0) {
        s_off[next] = (uint32_t)prev_start;
        s_len[next] = (uint16_t)(prev_len + 1);
      }
      ++next;
      width = lzw_width(next);
    }
    prev_start = pos;
    prev_len = len;
    pos += len;
    __syncwarp();  // the copy and the table entry are visible to every lane before the next code
  }
}

__global__ void __launch_bounds__(TIFF_LZW_WARPS * 32) k_tiff_lzw(const uint8_t* __restrict__ xfer, uint8_t* dec,
                                                                   const TiffSegDev* __restrict__ segs, int n,
                                                                   int32_t* status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int w = threadIdx.x >> 5;
  uint32_t* s_off = reinterpret_cast<uint32_t*>(smem_raw) + (size_t)w * TIFF_LZW_TABLE;
  uint16_t* s_len =
      reinterpret_cast<uint16_t*>(smem_raw + (size_t)TIFF_LZW_WARPS * TIFF_LZW_TABLE * sizeof(uint32_t)) +
      (size_t)w * TIFF_LZW_TABLE;
  for (int s = blockIdx.x * TIFF_LZW_WARPS + w; s < n; s += gridDim.x * TIFF_LZW_WARPS) {
    const TiffSegDev g = segs[s];
    const int st = lzw_decode_warp(xfer + g.xfer_off, g.xfer_bytes, dec + g.dec_off, g.dec_bytes, s_off, s_len);
    if ((threadIdx.x & 31) == 0) status[s] = st;
    __syncwarp();
  }
}

// ---------------------------------------------------------------- placement
struct TiffPlace {
  int32_t predictor, swap;
  int64_t height, width;           // image
  int64_t win_r0, win_c0, win_ny, win_nx;
};

template <typename U>
__device__ __forceinline__ U bswap(U v) {
  if constexpr (sizeof(U) == 1) {
    return v;
  } else if constexpr (sizeof(U) == 2) {
    return (U)(((uint32_t)v >> 8) | (((uint32_t)v & 0xff) << 8));
  } else if constexpr (sizeof(U) == 4) {
    return __byte_perm(v, 0, 0x0123);
  } else {
    return ((uint64_t)__byte_perm((uint32_t)v, 0, 0x0123) << 32) | __byte_perm((uint32_t)(v >> 32), 0, 0x0123);
  }
}

template <typename S>
__device__ __forceinline__ S warp_inclusive_sum(S v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const S o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += o;
  }
  return v;
}

// U: the unsigned type of the sample width.  One warp per segment row.
template <typename U>
__global__ void __launch_bounds__(TIFF_PLACE_THREADS, 1) k_tiff_place(uint8_t* dec, const TiffSegDev* __restrict__ segs,
                                                                    TiffPlace P, U* __restrict__ out) {
  const TiffSegDev g = segs[blockIdx.x];
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  // the segment columns that land in the window: [c_lo, c_hi)
  const int64_t c_lo = max((int64_t)0, P.win_c0 - g.col0);
  const int64_t c_hi = min((int64_t)g.cols, min(P.width, P.win_c0 + P.win_nx) - g.col0);
  for (int r = threadIdx.x >> 5; r < g.rows; r += warps) {
    const int64_t R = (int64_t)g.row0 + r;
    if (R < P.win_r0 || R >= P.win_r0 + P.win_ny || R >= P.height || c_hi <= c_lo) continue;
    U* o = out + (R - P.win_r0) * P.win_nx + (g.col0 - P.win_c0);
    uint8_t* rowb = dec + g.dec_off + (int64_t)r * g.cols * sizeof(U);
    const U* row = reinterpret_cast<const U*>(rowb);
    if (P.predictor == 1) {
      for (int64_t c = c_lo + lane; c < c_hi; c += 32) o[c] = P.swap ? bswap(row[c]) : row[c];
    } else if (P.predictor == 2) {  // running sum along the row, modulo 2^bits
      using S = typename std::conditional<sizeof(U) == 8, uint64_t, uint32_t>::type;
      S carry = 0;
      for (int64_t c0 = 0; c0 < c_hi; c0 += 32) {
        const int64_t c = c0 + lane;
        S v = c < c_hi ? (S)(P.swap ? bswap(row[c]) : row[c]) : (S)0;
        v = warp_inclusive_sum(v) + carry;
        carry = __shfl_sync(0xffffffffu, v, 31);
        if (c >= c_lo && c < c_hi) o[c] = (U)v;
      }
    } else {  // 3: running byte sum over the row, then byte planes, most significant first
      const int64_t nb = (int64_t)g.cols * sizeof(U);
      uint32_t carry = 0;
      for (int64_t b0 = 0; b0 < nb; b0 += 32) {
        const int64_t b = b0 + lane;
        uint32_t v = b < nb ? rowb[b] : 0u;
        v = warp_inclusive_sum(v) + carry;
        carry = __shfl_sync(0xffffffffu, v, 31);
        __syncwarp();
        if (b < nb) rowb[b] = (uint8_t)v;
      }
      __syncwarp();
      for (int64_t c = c_lo + lane; c < c_hi; c += 32) {
        U v = 0;
#pragma unroll
        for (int p = 0; p < (int)sizeof(U); ++p) v = (U)((v << 8) | (U)rowb[(int64_t)p * g.cols + c]);
        o[c] = v;
      }
    }
  }
}

template <typename U>
cudaError_t launch_place(uint8_t* dec, const TiffSegDev* segs, int n, const TiffPlace& P, void* out,
                         cudaStream_t st) {
  k_tiff_place<U><<<n, TIFF_PLACE_THREADS, 0, st>>>(dec, segs, P, static_cast<U*>(out));
  ++g_launches;
  return cudaGetLastError();
}

const char* tiff_status_text(int s) {
  switch (s) {
    case ATL_TIFF_LZW_TRUNCATED: return "LZW stream ends before the segment is complete (truncated)";
    case ATL_TIFF_LZW_BAD_CODE: return "LZW code past the end of the string table";
    case ATL_TIFF_LZW_LONG: return "LZW data decodes to more bytes than the segment holds";
    case ATL_TIFF_LZW_SHORT: return "LZW end-of-information before the segment is complete";
    case ATL_TIFF_LZW_OLD_STYLE: return "old-style (pre-TIFF 6.0, LSB-first) LZW is not supported";
  }
  return "unknown status";
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_geotiff_read(int device, const char* path, const AtlTiffLayout* L, int64_t n_segs, const int64_t* seg_index,
                     const int64_t* file_offset, const int64_t* stored_bytes, int64_t batch_bytes, int32_t n_threads,
                     void* out_dev, int64_t* bad_segment, AtlTiffStats* stats, void* stream) {
  ATL_REQUIRE(path && L && out_dev && bad_segment && stats, "NULL argument");
  *bad_segment = -1;
  *stats = AtlTiffStats{};
  ATL_REQUIRE(n_segs >= 0 && (n_segs == 0 || (seg_index && file_offset && stored_bytes)), "segment table missing");
  ATL_REQUIRE(L->compression == ATL_TIFF_NONE || L->compression == ATL_TIFF_LZW || L->compression == ATL_TIFF_DEFLATE,
              "compression must be ATL_TIFF_NONE, _LZW or _DEFLATE");
  ATL_REQUIRE(L->predictor >= 1 && L->predictor <= 3, "predictor must be 1, 2 or 3");
  const int bps = L->sample_bytes;
  ATL_REQUIRE(bps == 1 || bps == 2 || bps == 4 || bps == 8, "sample size must be 1, 2, 4 or 8 bytes");
  ATL_REQUIRE(L->width > 0 && L->height > 0 && L->seg_w > 0 && L->seg_h > 0, "bad image or segment size");
  ATL_REQUIRE(L->width < INT32_MAX && L->height < INT32_MAX && L->seg_w < INT32_MAX && L->seg_h < INT32_MAX,
              "image too large");
  ATL_REQUIRE(L->tiled || L->seg_w == L->width, "a strip spans the image width");
  ATL_REQUIRE(L->win_r0 >= 0 && L->win_c0 >= 0 && L->win_ny > 0 && L->win_nx > 0 &&
                  L->win_r0 + L->win_ny <= L->height && L->win_c0 + L->win_nx <= L->width,
              "window outside the image");
  ATL_REQUIRE(batch_bytes > 0, "batch_bytes must be positive");
  const int64_t across = L->tiled ? (L->width + L->seg_w - 1) / L->seg_w : 1;
  const int64_t down = (L->height + L->seg_h - 1) / L->seg_h;
  const int comp = L->compression;

  // segment geometry and the batches: consecutive segments whose transfer and decoded bytes fit
  const bool coded = comp != ATL_TIFF_NONE;  // decoded on the device into a buffer of its own
  std::vector<TiffSegDev> seg(n_segs);
  std::vector<int64_t> reads(n_segs), xoff(n_segs);
  SegmentBatches S;
  S.batch_start.push_back(0);
  int64_t max_dec = 0, bx = 0, bd = 0;
  for (int64_t k = 0; k < n_segs; ++k) {
    const int64_t i = seg_index[k];
    ATL_REQUIRE(i >= 0 && i < across * down, "segment index outside the image's segments");
    ATL_REQUIRE(file_offset[k] >= 0 && stored_bytes[k] >= 0, "bad segment offset or size");
    TiffSegDev& g = seg[k];
    g.row0 = (int32_t)((i / across) * L->seg_h);
    g.col0 = (int32_t)((i % across) * L->seg_w);
    g.cols = (int32_t)L->seg_w;
    g.rows = (int32_t)(L->tiled ? L->seg_h : std::min<int64_t>(L->seg_h, L->height - g.row0));
    g.dec_bytes = (int64_t)g.rows * g.cols * bps;
    ATL_REQUIRE(comp != ATL_TIFF_LZW || g.dec_bytes < ((int64_t)1 << 32), "an LZW segment above 4 GiB");
    g.xfer_bytes = coded ? stored_bytes[k] : g.dec_bytes;
    if (comp == ATL_TIFF_NONE && stored_bytes[k] < g.dec_bytes) {
      *bad_segment = i;
      set_error("segment " + std::to_string(i) + ": uncompressed segment shorter than its pixels");
      return ATL_ERR_INVALID;
    }
    const int64_t x = seg_align_up(g.xfer_bytes), d = coded ? seg_align_up(g.dec_bytes) : 0;
    if (k > S.batch_start.back() && (bx + x > batch_bytes || bd + d > batch_bytes)) {
      S.batch_start.push_back(k);
      bx = bd = 0;
    }
    g.xfer_off = bx;
    g.dec_off = coded ? bd : bx;
    bx += x;
    bd += d;
    S.max_xfer = std::max(S.max_xfer, bx);
    max_dec = std::max(max_dec, bd);
    reads[k] = g.xfer_bytes;
    xoff[k] = g.xfer_off;
  }
  S.batch_start.push_back(n_segs);
  if (n_segs == 0) return ATL_OK;
  S.file_offset = file_offset;
  S.read_bytes = reads.data();
  S.xfer_off = xoff.data();
  S.desc = seg.data();
  S.desc_bytes = sizeof(TiffSegDev);
  S.n_threads = n_threads;
  const int n_batches = (int)S.batch_start.size() - 1;

  ATL_CUDA(cudaSetDevice(device));
  const cudaStream_t st = (cudaStream_t)stream;
  struct DecBuffers {
    uint8_t* p[2] = {nullptr, nullptr};
    ~DecBuffers() {
      cudaFree(p[0]);
      cudaFree(p[1]);
    }
  } dec;
  if (coded)
    for (int s = 0; s < (n_batches > 1 ? 2 : 1); ++s) ATL_CUDA(cudaMalloc(&dec.p[s], std::max(max_dec, SEG_ALIGN)));
  int smem_lzw = TIFF_LZW_WARPS * TIFF_LZW_TABLE * (int)(sizeof(uint32_t) + sizeof(uint16_t));
  if (comp == ATL_TIFF_LZW) ATL_CUDA(cudaFuncSetAttribute(k_tiff_lzw, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_lzw));
  const TiffPlace P{L->predictor, L->big_endian && L->predictor != 3 ? 1 : 0, L->height, L->width,
                    L->win_r0,    L->win_c0,                                   L->win_ny, L->win_nx};

  auto launch = [&](int slot, int64_t, int n, const uint8_t* xfer, const void* d, int32_t* status) -> cudaError_t {
    const TiffSegDev* segs = static_cast<const TiffSegDev*>(d);
    uint8_t* src = const_cast<uint8_t*>(xfer);  // the placement undoes predictor 3 in place
    cudaError_t e = cudaSuccess;
    if (comp == ATL_TIFF_LZW) {
      const int grid = std::max(1, std::min((n + TIFF_LZW_WARPS - 1) / TIFF_LZW_WARPS, 2 * sm_count()));
      k_tiff_lzw<<<grid, TIFF_LZW_WARPS * 32, smem_lzw, st>>>(xfer, dec.p[slot], segs, n, status);
      ++g_launches;
      e = cudaGetLastError();
      src = dec.p[slot];
    } else if (comp == ATL_TIFF_DEFLATE) {
      e = launch_inflate(xfer, dec.p[slot], segs, sizeof(TiffSegDev), n, status, st);
      src = dec.p[slot];
    }
    if (e != cudaSuccess) return e;
    switch (bps) {
      case 1: return launch_place<uint8_t>(src, segs, n, P, out_dev, st);
      case 2: return launch_place<uint16_t>(src, segs, n, P, out_dev, st);
      case 4: return launch_place<uint32_t>(src, segs, n, P, out_dev, st);
      default: return launch_place<uint64_t>(src, segs, n, P, out_dev, st);
    }
  };
  std::vector<int32_t> status;
  int64_t bad = -1;
  const int rc = run_segment_batches(device, path, S, st, launch, status, &bad);
  if (rc != ATL_OK) {
    if (bad >= 0) {
      *bad_segment = seg_index[bad];
      set_error("segment " + std::to_string(seg_index[bad]) + ": the file ends inside the segment");
    }
    return rc;
  }
  for (int64_t k = 0; k < n_segs; ++k) {
    stats->stored_bytes += stored_bytes[k];
    stats->xfer_bytes += seg[k].xfer_bytes;
  }
  stats->batches = n_batches;
  stats->segments = n_segs;
  for (int64_t k = 0; k < n_segs; ++k)
    if (status[k] != ATL_TIFF_OK) {
      *bad_segment = seg_index[k];
      set_error("segment " + std::to_string(seg_index[k]) + ": " +
                (comp == ATL_TIFF_DEFLATE ? std::string("Deflate data is corrupt: ") + inflate_status_text(status[k])
                                          : std::string(tiff_status_text(status[k]))));
      return ATL_ERR_INVALID;
    }
  return ATL_OK;
}

}  // extern "C"
