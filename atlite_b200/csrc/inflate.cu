// inflate.cu -- zlib streams (RFC 1950 framing around RFC 1951 Deflate) decoded on the GPU, one
// warp per stream, many independent streams per launch (k_inflate), and the batch pipeline that
// feeds compressed segments from a file to the device (run_segment_batches).  Users: geotiff.cu
// (Deflate segments) and decode.cu (cutout chunks), through inflate.cuh.
//
// Every lane of the warp keeps the same decoder state (bit buffer, position, tables), so the
// control flow never diverges; the lanes share the work that is wide: building the Huffman tables,
// match copies, stored-block copies and the Adler-32 of the output.  Accepted streams are the
// ones zlib's uncompress() accepts into an output buffer of exactly the span's size:
//   * header CM = 8, CINFO <= 7, FCHECK valid; FDICT = 1 is refused (no preset dictionaries);
//   * stored blocks (LEN = ~NLEN), fixed and dynamic Huffman blocks; code sets as inflate_table
//     accepts them: over-subscribed sets are refused, incomplete ones only when their longest
//     code has one bit (a single code of length 1) or, for distances, when there is no code at all
//     (a literal-only block); literal/length symbols 286/287 and distance codes 30/31 are invalid;
//   * the Adler-32 trailer must match the output; bytes after it are ignored;
//   * the stream must fill the output span exactly.
// A corrupt stream only sets its status (ATL_INFLATE_*); every read is checked against the input
// span and every write against the output span.
//
// Tables (per warp, shared memory): a 2^10-entry root table per code whose entries are
// (symbol | length << 9); codes longer than 10 bits (rare: only long-tailed dynamic codes) are
// marked in the root table and decoded canonically from the per-length counts and the symbols
// sorted by code, as zlib's puff does.
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstring>
#include <mutex>
#include <thread>

#include "common.cuh"
#include "inflate.cuh"

namespace atl {
namespace {

constexpr int INFL_ROOT = 10;  // root table bits
constexpr int INFL_ROOT_SIZE = 1 << INFL_ROOT;
constexpr uint16_t INFL_LONG = 0xffff;  // root entry: the code is longer than INFL_ROOT bits
constexpr int INFL_WARPS = 4;           // decoders per CTA
constexpr uint32_t ADLER_MOD = 65521;

// One warp's tables.  lens holds the code lengths of the current block (litlen then distance).
struct InflTables {
  uint16_t lit_root[INFL_ROOT_SIZE];
  uint16_t dist_root[INFL_ROOT_SIZE];
  uint16_t lit_sym[288];
  uint16_t dist_sym[32];
  uint16_t lit_count[16];
  uint16_t dist_count[16];
  uint16_t first[16];  // scratch of the table builder: first sorted index per length,
  uint16_t next[16];   // and the next free one
  uint8_t lens[320];
  int32_t flag;        // lane 0 -> warp broadcast of the builder's verdict
};

__device__ __forceinline__ uint32_t infl_rev(uint32_t code, int len) { return __brev(code) >> (32 - len); }

// Canonical Huffman tables for lens[0..n): root entries, per-length counts and the symbols sorted by
// (length, symbol).  kind: 0 code-length code (must be complete), 1 literal/length, 2 distance.
// Returns false for a set zlib's inflate_table refuses.
__device__ bool infl_build(InflTables& T, const uint8_t* lens, int n, uint16_t* root, uint16_t* count, uint16_t* sym,
                           int kind) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) count[l] = 0;
    for (int s = 0; s < n; ++s) ++count[lens[s]];
    int left = 1, max = 0;
    bool ok = true;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - count[l];
      if (left < 0) ok = false;  // over-subscribed
      if (count[l]) max = l;
    }
    // incomplete: allowed for a single one-bit code, and (as an empty set) for distances
    if (ok && left > 0 && max != 0 && (kind == 0 || max != 1)) ok = false;
    if (ok && max == 0 && kind == 0) ok = false;
    int idx = 0;
    for (int l = 1; l < 16; ++l) {
      T.first[l] = (uint16_t)idx;
      idx += count[l];
    }
    T.first[0] = (uint16_t)idx;  // number of coded symbols
    for (int l = 1; l < 16; ++l) T.next[l] = T.first[l];
    for (int s = 0; s < n; ++s)
      if (lens[s]) sym[T.next[lens[s]]++] = (uint16_t)s;
    T.flag = ok;
  }
  __syncwarp();
  const bool ok = T.flag != 0;
  for (int i = lane; i < INFL_ROOT_SIZE; i += 32) root[i] = 0;
  __syncwarp();
  if (ok) {
    const int coded = T.first[0];
    for (int k = lane; k < coded; k += 32) {
      const int s = sym[k], len = lens[s];
      // canonical code of sorted position k: first code of its length + rank within the length
      uint32_t code = 0;
      for (int l = 1; l <= len; ++l) code = (code + (l > 1 ? count[l - 1] : 0)) << 1;  // next_code[len]
      code += (uint32_t)(k - T.first[len]);
      if (len <= INFL_ROOT) {
        const uint16_t e = (uint16_t)(s | (len << 9));
        for (uint32_t r = infl_rev(code, len); r < (uint32_t)INFL_ROOT_SIZE; r += 1u << len) root[r] = e;
      } else {
        root[infl_rev(code >> (len - INFL_ROOT), INFL_ROOT)] = INFL_LONG;
      }
    }
  }
  __syncwarp();
  return ok;
}

// The warp's bit reader: bits are consumed LSB first; every lane holds the same state.
struct InflBits {
  const uint8_t* in;
  int64_t n, ip;  // input bytes, next byte to load
  uint64_t bb;
  int nb;

  __device__ __forceinline__ void refill() {
    while (nb <= 32 && ip < n) {
      if ((ip & 3) == 0 && ip + 4 <= n) {
        bb |= (uint64_t)__ldg(reinterpret_cast<const uint32_t*>(in + ip)) << nb;
        ip += 4;
        nb += 32;
      } else {
        bb |= (uint64_t)__ldg(in + ip) << nb;
        ++ip;
        nb += 8;
      }
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) const { return (uint32_t)(bb & ((1ull << k) - 1)); }
  __device__ __forceinline__ void drop(int k) {
    bb >>= k;
    nb -= k;
  }
};

// Decode one symbol; returns the symbol, or -1 for a bit pattern without a code, -2 when the input
// ends inside the code.  The caller has refilled (>= 15 bits unless the input is ending).
__device__ __forceinline__ int infl_decode(InflBits& B, const uint16_t* root, const uint16_t* count,
                                           const uint16_t* sym) {
  const uint16_t e = root[B.peek(INFL_ROOT)];
  if (e != INFL_LONG) {
    const int len = e >> 9;
    // no code: only incomplete sets leave entries empty (a single one-bit code, or no code at all), and
    // one bit decides those, as in zlib's tables
    if (len == 0) return B.nb < 1 ? -2 : -1;
    if (len > B.nb) return -2;
    B.drop(len);
    return e & 511;
  }
  int code = 0, first = 0, index = 0;  // puff's canonical decode, one bit at a time
  for (int len = 1; len < 16; ++len) {
    if (len > B.nb) return -2;
    code |= (int)((B.bb >> (len - 1)) & 1);
    const int c = count[len];
    if (code - c < first) {
      B.drop(len);
      return sym[index + (code - first)];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

__constant__ uint16_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Adler-32 of out[0, n) with the warp: lane sums over 4-byte words, combined as
// A = 1 + S1, B = n + n * S1 - sum(i * x_i)  (mod 65521).
__device__ uint32_t infl_adler_warp(const uint8_t* out, int64_t n) {
  const int lane = threadIdx.x & 31;
  uint64_t s1 = 0, si = 0;
  const int64_t nw = n >> 2;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(out);
  uint32_t im = (uint32_t)(((int64_t)lane * 4) % ADLER_MOD);  // byte index of the lane's word, mod 65521
  const uint32_t step = 128 % ADLER_MOD;
  int64_t cnt = 0;
  for (int64_t j = lane; j < nw; j += 32) {
    const uint32_t v = w[j];
    const uint32_t x0 = v & 255, x1 = (v >> 8) & 255, x2 = (v >> 16) & 255, x3 = v >> 24;
    const uint32_t sum = x0 + x1 + x2 + x3;
    s1 += sum;
    si += (uint64_t)im * sum + x1 + 2 * x2 + 3 * x3;
    im += step;
    if (im >= ADLER_MOD) im -= ADLER_MOD;
    if (++cnt == (1 << 20)) {  // keep the sums far from overflow
      s1 %= ADLER_MOD;
      si %= ADLER_MOD;
      cnt = 0;
    }
  }
  for (int64_t i = nw * 4 + lane; i < n; i += 32) {
    s1 += out[i];
    si += (uint64_t)(i % ADLER_MOD) * out[i];
  }
  s1 %= ADLER_MOD;
  si %= ADLER_MOD;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, d);
    si += __shfl_xor_sync(0xffffffffu, si, d);
  }
  s1 %= ADLER_MOD;
  si %= ADLER_MOD;
  const uint64_t nm = (uint64_t)(n % ADLER_MOD);
  const uint32_t a = (uint32_t)((1 + s1) % ADLER_MOD);
  const uint32_t b = (uint32_t)((nm + nm * s1 + (uint64_t)ADLER_MOD * ADLER_MOD - si) % ADLER_MOD);
  return (b << 16) | a;
}

// Inflate one zlib stream with the calling warp into out[0, size).  Returns an ATL_INFLATE_* status.
__device__ int inflate_warp(const uint8_t* __restrict__ in, int64_t n_in, uint8_t* out, int64_t size, InflTables& T) {
  const int lane = threadIdx.x & 31;
  InflBits B{in, n_in, 0, 0, 0};
  B.refill();
  if (B.nb < 16) return ATL_INFLATE_TRUNCATED;
  {
    const uint32_t cmf = B.peek(8), flg = (B.peek(16) >> 8);
    if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0) return ATL_INFLATE_BAD_HEADER;
    if (flg & 32) return ATL_INFLATE_DICTIONARY;
    B.drop(16);
  }
  int64_t pos = 0;
  int tables = 0;  // 1: the fixed tables are loaded
  for (;;) {
    B.refill();
    if (B.nb < 3) return ATL_INFLATE_TRUNCATED;
    const int final = B.peek(1), type = (B.peek(3) >> 1);
    B.drop(3);
    if (type == 0) {  // stored: LEN, NLEN at the next byte boundary, then LEN bytes
      B.drop(B.nb & 7);
      B.refill();
      if (B.nb < 32) return ATL_INFLATE_TRUNCATED;
      const uint32_t len = B.peek(16), nlen = B.peek(32) >> 16;
      B.drop(32);
      if (len != (~nlen & 0xffff)) return ATL_INFLATE_STORED_LENGTH;
      const int64_t p = B.ip - (B.nb >> 3);  // the bit buffer holds whole bytes only now
      if (p + (int64_t)len > n_in) return ATL_INFLATE_TRUNCATED;
      if ((int64_t)len > size - pos) return ATL_INFLATE_LONG;
      for (int64_t k = lane; k < (int64_t)len; k += 32) out[pos + k] = __ldg(in + p + k);
      pos += len;
      B.ip = p + len;
      B.bb = 0;
      B.nb = 0;
      __syncwarp();
    } else if (type == 3) {
      return ATL_INFLATE_BAD_BLOCK_TYPE;
    } else {
      if (type == 1) {
        if (tables != 1) {
          for (int s = lane; s < 320; s += 32) T.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
          __syncwarp();
          infl_build(T, T.lens, 288, T.lit_root, T.lit_count, T.lit_sym, 1);
          infl_build(T, T.lens + 288, 32, T.dist_root, T.dist_count, T.dist_sym, 2);
          tables = 1;
        }
      } else {
        B.refill();
        if (B.nb < 14) return ATL_INFLATE_TRUNCATED;
        const int nlen = B.peek(5) + 257, ndist = (B.peek(10) >> 5) + 1, ncode = (B.peek(14) >> 10) + 4;
        B.drop(14);
        if (nlen > 286) return ATL_INFLATE_BAD_LITLEN_SET;
        if (ndist > 30) return ATL_INFLATE_BAD_DIST_SET;
        // the code-length code's lengths go to lens[300, 319): past every length but the last 16
        // of the 316 read below, which are only written once this table is built
        uint8_t* cl = T.lens + 300;
        if (lane < 19) cl[lane] = 0;
        __syncwarp();
        for (int i = 0; i < ncode; ++i) {
          B.refill();
          if (B.nb < 3) return ATL_INFLATE_TRUNCATED;
          if (lane == 0) cl[c_clen_order[i]] = (uint8_t)B.peek(3);
          B.drop(3);
        }
        __syncwarp();
        // the code-length code goes into the distance tables, which this block rebuilds anyway
        if (!infl_build(T, cl, 19, T.dist_root, T.dist_count, T.dist_sym, 0)) return ATL_INFLATE_BAD_CODELEN_SET;
        int i = 0, prev = 0, bad = 0;
        while (i < nlen + ndist) {
          B.refill();
          const int s = infl_decode(B, T.dist_root, T.dist_count, T.dist_sym);
          if (s == -2) return ATL_INFLATE_TRUNCATED;
          if (s < 0) {
            bad = 1;
            break;
          }
          if (s < 16) {
            if (lane == 0) T.lens[i] = (uint8_t)s;
            prev = s;
            ++i;
            continue;
          }
          int rep, val = 0;
          if (s == 16) {  // repeat the previous length 3-6 times
            if (i == 0) {
              bad = 1;
              break;
            }
            if (B.nb < 2) return ATL_INFLATE_TRUNCATED;
            rep = 3 + (int)B.peek(2);
            B.drop(2);
            val = prev;
          } else if (s == 17) {  // 3-10 zeros
            if (B.nb < 3) return ATL_INFLATE_TRUNCATED;
            rep = 3 + (int)B.peek(3);
            B.drop(3);
          } else {  // 11-138 zeros
            if (B.nb < 7) return ATL_INFLATE_TRUNCATED;
            rep = 11 + (int)B.peek(7);
            B.drop(7);
          }
          if (i + rep > nlen + ndist) {
            bad = 1;
            break;
          }
          if (lane == 0)
            for (int k = 0; k < rep; ++k) T.lens[i + k] = (uint8_t)val;
          prev = val;
          i += rep;
        }
        if (bad) return ATL_INFLATE_BAD_CODELEN_SET;
        __syncwarp();
        if (T.lens[256] == 0) return ATL_INFLATE_BAD_LITLEN_SET;  // no end-of-block code
        if (!infl_build(T, T.lens, nlen, T.lit_root, T.lit_count, T.lit_sym, 1)) return ATL_INFLATE_BAD_LITLEN_SET;
        if (!infl_build(T, T.lens + nlen, ndist, T.dist_root, T.dist_count, T.dist_sym, 2))
          return ATL_INFLATE_BAD_DIST_SET;
        tables = 2;
      }
      // the block's symbols
      for (;;) {
        B.refill();
        int s = infl_decode(B, T.lit_root, T.lit_count, T.lit_sym);
        if (s == -2) return ATL_INFLATE_TRUNCATED;
        if (s < 0 || s > 285) return ATL_INFLATE_BAD_SYMBOL;
        if (s < 256) {
          if (pos >= size) return ATL_INFLATE_LONG;
          if (lane == 0) out[pos] = (uint8_t)s;
          ++pos;
          continue;  // the write is ordered before any later read by the __syncwarp of a copy
        }
        if (s == 256) break;
        s -= 257;
        const int le = c_len_extra[s];
        if (B.nb < le) return ATL_INFLATE_TRUNCATED;
        const int len = c_len_base[s] + (int)B.peek(le);
        B.drop(le);
        B.refill();
        const int d = infl_decode(B, T.dist_root, T.dist_count, T.dist_sym);
        if (d == -2) return ATL_INFLATE_TRUNCATED;
        if (d < 0 || d > 29) return ATL_INFLATE_BAD_SYMBOL;
        const int de = c_dist_extra[d];
        if (B.nb < de) return ATL_INFLATE_TRUNCATED;
        const int dist = c_dist_base[d] + (int)B.peek(de);
        B.drop(de);
        if (dist > pos) return ATL_INFLATE_TOO_FAR;
        if (len > size - pos) return ATL_INFLATE_LONG;
        __syncwarp();  // literals written by lane 0 are visible to every lane
        // byte i of the copy is out[pos - dist + (i mod dist)]: always bytes written before pos
        const uint8_t* src = out + pos - dist;
        for (int k = lane; k < len; k += 32) out[pos + k] = src[k < dist ? k : k % dist];
        pos += len;
        __syncwarp();
      }
    }
    if (final) break;
  }
  __syncwarp();
  // trailer: the Adler-32 of the output, big-endian, at the next byte boundary
  B.drop(B.nb & 7);
  B.refill();
  if (B.nb < 32) return ATL_INFLATE_TRUNCATED;
  const uint32_t t = B.peek(32);
  const uint32_t want = __byte_perm(t, 0, 0x0123);
  if (infl_adler_warp(out, pos) != want) return ATL_INFLATE_ADLER;
  if (pos != size) return ATL_INFLATE_SHORT;
  return ATL_INFLATE_OK;
}

// Inflate stream k of a batch, described by the InflSpan at spans + k * stride: stream k reads in[in_off, in_off + in_bytes) and fills
// out[out_off, out_off + out_bytes) (16-byte aligned starts).  status[k] gets its ATL_INFLATE_*.
__global__ void __launch_bounds__(INFL_WARPS * 32) k_inflate(const uint8_t* __restrict__ in, uint8_t* out,
                                                             const uint8_t* __restrict__ spans, size_t stride,
                                                             int n, int32_t* status) {
  __shared__ InflTables tables[INFL_WARPS];
  const int w = threadIdx.x >> 5;
  for (int s = blockIdx.x * INFL_WARPS + w; s < n; s += gridDim.x * INFL_WARPS) {
    const InflSpan g = *reinterpret_cast<const InflSpan*>(spans + (size_t)s * stride);
    const int st = inflate_warp(in + g.in_off, g.in_bytes, out + g.out_off, g.out_bytes, tables[w]);
    if ((threadIdx.x & 31) == 0) status[s] = st;
    __syncwarp();
  }
}

}  // namespace

cudaError_t launch_inflate(const uint8_t* in, uint8_t* out, const void* spans, size_t stride, int n,
                           int32_t* status, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const int grid = std::max(1, std::min((n + INFL_WARPS - 1) / INFL_WARPS, 8 * sm_count()));
  k_inflate<<<grid, INFL_WARPS * 32, 0, st>>>(in, out, static_cast<const uint8_t*>(spans), stride, n, status);
  ++g_launches;
  return cudaGetLastError();
}

const char* inflate_status_text(int s) {
  switch (s) {
    case ATL_INFLATE_BAD_HEADER: return "bad zlib header (not CM 8 with CINFO <= 7, or FCHECK wrong)";
    case ATL_INFLATE_DICTIONARY: return "the stream needs a preset dictionary (FDICT), which is not supported";
    case ATL_INFLATE_BAD_BLOCK_TYPE: return "invalid block type";
    case ATL_INFLATE_STORED_LENGTH: return "stored block length does not match its complement";
    case ATL_INFLATE_BAD_CODELEN_SET: return "invalid code-length set";
    case ATL_INFLATE_BAD_LITLEN_SET: return "invalid literal/length code set";
    case ATL_INFLATE_BAD_DIST_SET: return "invalid distance code set";
    case ATL_INFLATE_BAD_SYMBOL: return "invalid literal/length or distance symbol";
    case ATL_INFLATE_TOO_FAR: return "distance too far back";
    case ATL_INFLATE_LONG: return "decodes to more bytes than its span (output longer)";
    case ATL_INFLATE_TRUNCATED: return "the stream ends early (truncated)";
    case ATL_INFLATE_SHORT: return "decodes to fewer bytes than its span (output shorter)";
    case ATL_INFLATE_ADLER: return "Adler-32 mismatch";
  }
  return "unknown status";
}


namespace {

// Per-call device and pinned buffers; freed on every return path.
struct BatchBuffers {
  uint8_t* pinned[2] = {nullptr, nullptr};
  uint8_t* pinned_desc[2] = {nullptr, nullptr};
  uint8_t* xfer[2] = {nullptr, nullptr};
  uint8_t* desc[2] = {nullptr, nullptr};
  int32_t* status = nullptr;
  cudaStream_t copy = nullptr;
  cudaEvent_t copied[2] = {nullptr, nullptr}, used[2] = {nullptr, nullptr};
  int fd = -1;
  ~BatchBuffers() {
    if (copy) cudaStreamSynchronize(copy);
    for (int s = 0; s < 2; ++s) {
      if (used[s]) cudaEventSynchronize(used[s]);
      cudaFreeHost(pinned[s]);
      cudaFreeHost(pinned_desc[s]);
      cudaFree(xfer[s]);
      cudaFree(desc[s]);
      if (copied[s]) cudaEventDestroy(copied[s]);
      if (used[s]) cudaEventDestroy(used[s]);
    }
    cudaFree(status);
    if (copy) cudaStreamDestroy(copy);
    if (fd >= 0) close(fd);
  }
};

}  // namespace

int run_segment_batches(int device, const char* path, const SegmentBatches& S, cudaStream_t st,
                        const SegmentLaunch& launch, std::vector<int32_t>& status, int64_t* bad_k) {
  *bad_k = -1;
  const int n_batches = (int)S.batch_start.size() - 1;
  const int64_t n_segs = n_batches > 0 ? S.batch_start.back() : 0;
  status.assign(n_segs, 0);
  if (n_segs == 0) return ATL_OK;
  int64_t max_n = 0;
  for (int b = 0; b < n_batches; ++b) max_n = std::max(max_n, S.batch_start[b + 1] - S.batch_start[b]);
  const size_t desc_max = std::max<size_t>(1, max_n * S.desc_bytes);
  const int64_t xfer_max = std::max(S.max_xfer, SEG_ALIGN);

  BatchBuffers B;
  B.fd = open(path, O_RDONLY);
  if (B.fd < 0) {
    set_error(std::string("cannot open ") + path);
    return ATL_ERR_INVALID;
  }
  ATL_CUDA(cudaSetDevice(device));
  const int n_buf = n_batches > 1 ? 2 : 1;
  for (int s = 0; s < n_buf; ++s) {
    ATL_CUDA(cudaHostAlloc(&B.pinned[s], xfer_max, cudaHostAllocDefault));
    ATL_CUDA(cudaHostAlloc(&B.pinned_desc[s], desc_max, cudaHostAllocDefault));
    ATL_CUDA(cudaMalloc(&B.xfer[s], xfer_max));
    ATL_CUDA(cudaMalloc(&B.desc[s], desc_max));
    ATL_CUDA(cudaEventCreateWithFlags(&B.copied[s], cudaEventDisableTiming));
    ATL_CUDA(cudaEventCreateWithFlags(&B.used[s], cudaEventDisableTiming));
  }
  ATL_CUDA(cudaMalloc(&B.status, n_segs * sizeof(int32_t)));
  ATL_CUDA(cudaMemsetAsync(B.status, 0, n_segs * sizeof(int32_t), st));
  ATL_CUDA(cudaStreamCreateWithFlags(&B.copy, cudaStreamNonBlocking));
  ATL_CUDA(cudaEventRecord(B.used[0], st));  // the status reset precedes every kernel
  if (n_buf > 1) ATL_CUDA(cudaEventRecord(B.used[1], st));
  unsigned hw = std::thread::hardware_concurrency();
  int nthr_max = S.n_threads > 0 ? S.n_threads : (int)(hw ? hw : 4);
  if (nthr_max > 64) nthr_max = 64;

  for (int b = 0; b < n_batches; ++b) {
    const int s = b % n_buf;
    const int64_t k0 = S.batch_start[b], k1 = S.batch_start[b + 1];
    const int n = (int)(k1 - k0);
    if (b >= n_buf) ATL_CUDA(cudaEventSynchronize(B.copied[s]));  // the pinned buffer's previous copy has left it
    // read the batch's segments on host threads
    std::atomic<int64_t> next{k0};
    std::atomic<int64_t> failed{-1};
    auto worker = [&]() {
      for (;;) {
        const int64_t k = next.fetch_add(1);
        if (k >= k1 || failed.load() >= 0) return;
        const size_t want = (size_t)S.read_bytes[k];
        uint8_t* dst = B.pinned[s] + S.xfer_off[k];
        size_t got = 0;
        while (got < want) {
          const ssize_t r = pread(B.fd, dst + got, want - got, (off_t)(S.file_offset[k] + (int64_t)got));
          if (r <= 0) {
            int64_t none = -1;
            failed.compare_exchange_strong(none, k);
            return;
          }
          got += (size_t)r;
        }
      }
    };
    const int nthr = std::min(nthr_max, n);
    std::vector<std::thread> th;
    for (int t = 1; t < nthr; ++t) th.emplace_back(worker);
    worker();
    for (auto& t : th) t.join();
    if (failed.load() >= 0) {
      *bad_k = failed.load();
      return ATL_ERR_INVALID;
    }
    if (S.desc_bytes) memcpy(B.pinned_desc[s], static_cast<const uint8_t*>(S.desc) + k0 * S.desc_bytes, n * S.desc_bytes);
    int64_t xbytes = 0;
    for (int64_t k = k0; k < k1; ++k) xbytes = std::max(xbytes, S.xfer_off[k] + S.read_bytes[k]);
    // copy on the copy stream once the device buffers' previous kernels are done with them
    ATL_CUDA(cudaStreamWaitEvent(B.copy, B.used[s], 0));
    if (xbytes) ATL_CUDA(cudaMemcpyAsync(B.xfer[s], B.pinned[s], xbytes, cudaMemcpyHostToDevice, B.copy));
    if (S.desc_bytes)
      ATL_CUDA(cudaMemcpyAsync(B.desc[s], B.pinned_desc[s], n * S.desc_bytes, cudaMemcpyHostToDevice, B.copy));
    ATL_CUDA(cudaEventRecord(B.copied[s], B.copy));
    ATL_CUDA(cudaStreamWaitEvent(st, B.copied[s], 0));
    ATL_CUDA(launch(s, k0, n, B.xfer[s], B.desc[s], B.status + k0));
    ATL_CUDA(cudaEventRecord(B.used[s], st));
  }
  ATL_CUDA(cudaMemcpyAsync(status.data(), B.status, n_segs * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  ATL_CUDA(cudaStreamSynchronize(st));
  return ATL_OK;
}

}  // namespace atl
