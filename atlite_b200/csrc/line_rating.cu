// line_rating.cu -- dynamic line rating (convert.py:1152-1367): the IEEE-738 heat balance of
// every (line, cell, step), min-reduced over the cells of each line, NaN cells skipped.
//
// The physics depends on the line (azimuth, resistance, diameter, surface temperature,
// emissivity, absorptivity), so it runs per STORED entry of the (line x cell) intersection
// matrix, not per cell.  The plan (plan.cu) already lists them per (tile, line) slot.  A warp owns
// one active tile and walks a block of time steps in chunks of LR_STAGE steps:
//   1. stage: every lane evaluates the line-independent quantities of its 4 cells for the LR_STAGE
//      steps (temperature, wind speed, cos / sin of the wind azimuth, direct influx, the sun vector
//      X = cos alt cos az, Y = cos alt sin az) and parks them in the warp's shared memory;
//   2. reduce: lane (q, r) takes step r of the chunk and the entries q, q + NQ, ... of each slot,
//      evaluates the line's heat balance on them, min-reduces over the q lanes and issues one
//      atomicMin per (slot, step).
// Algorithmic traffic: 16 B per cell-step (4 float32 fields; height is static), + 8 / 16 B with a
// stored float32 / float64 solar position.  Nothing per cell or per entry goes to HBM.
//
// No inverse trigonometry is needed: with d = wind azimuth - radians(psi),
//   Phi = |mod(d + pi/2, pi) - pi/2|  gives  cos Phi = |cos d|, cos 2 Phi = cos 2d, sin 2 Phi = |sin 2d|
// (Phi is d reduced modulo pi into [0, pi/2]), and
//   cos(Phi_s) = cos alt cos(az - radians(psi)) = X cos psi' + Y sin psi',  sin(Phi_s) = sqrt(1 - (.)^2).
#include <cmath>
#include <vector>

#include "era5_derive.cuh"
#include "kernels.cuh"
#include "solar_host.cuh"

namespace atl {

// Per-line constants, hoisted out of the per-entry physics (convert.py:1196-1251)
struct __align__(16) LineConst {
  float cpsi, spsi;  // cos / sin of radians(psi)
  float inv_R;       // 1 / R
  float D, Ts;
  float D075;        // D ** 0.75
  float qr_c;        // 17.8 * D * epsilon
  float Ts4;         // (Ts / 100) ** 4
  float qs_c;        // alpha * D  (projected area A = D * 1)
  float pad[3];
};

__host__ __device__ inline LineConst make_line_const(double psi, double R, double D, double Ts, double eps,
                                                     double alpha) {
  const double p = psi * (3.14159265358979323846 / 180.0);  // radians(psi)  :1215
  LineConst c;
  c.cpsi = (float)cos(p);
  c.spsi = (float)sin(p);
  c.inv_R = (float)(1.0 / R);
  c.D = (float)D;
  c.Ts = (float)Ts;
  c.D075 = (float)pow(D, 0.75);
  c.qr_c = (float)(17.8 * D * eps);
  const double t = Ts / 100.0;
  c.Ts4 = (float)(t * t * t * t);
  c.qs_c = (float)(alpha * D);
  c.pad[0] = c.pad[1] = c.pad[2] = 0.f;
  return c;
}

// The line-independent quantities of one (cell, step)
struct LrCell {
  float Ta, V, cw, sw, Q, X, Y, hn;  // hn = rho's numerator in the height (14a)
};

__device__ __forceinline__ float rho_numerator(float H) {
  return fmaf(fmaf(6.379e-9f, H, -1.525e-4f), H, 1.293f);  // 1.293 - 1.525e-4 H + 6.379e-9 H^2  :1206
}

// Maximal current of one (line, cell, step): convert.py:1196-1251, float32.  NaN wherever the
// reference's float64 arithmetic gives NaN (negative radicand, Ta > Ts, NaN inputs).
__device__ __forceinline__ float line_imax(const LineConst& L, const LrCell& c) {
  const float T0 = 273.15f;
  const float Tfilm = 0.5f * (c.Ta + L.Ts);  // :1197
  const float dT = Tfilm - T0;
  // mu = 1.458e-6 Tfilm^1.5 / (Tfilm + 383.4 - T0)  (13a); rho = hn / (1 + 0.00367 (Tfilm - T0))  (14a)
  // reynold = D V rho / mu as ONE quotient
  const float tf15 = Tfilm * sqrtf(Tfilm);
  const float rho_den = fmaf(0.00367f, dT, 1.f);
  const float num = L.D * c.V * c.hn * (Tfilm + (383.4f - 273.15f));
  const float reynold = __fdividef(num, 1.458e-6f * tf15 * rho_den);
  const float k = fmaf(fmaf(-4.407e-9f, dT, 7.477e-5f), dT, 2.424e-2f);  // :1212-1214
  // wind direction factor K (:1215-1220) through cos / sin of d = wnd_azimuth - radians(psi)
  const float cd = fmaf(c.cw, L.cpsi, c.sw * L.spsi);
  const float sd = fmaf(c.sw, L.cpsi, -c.cw * L.spsi);
  const float K = 1.194f - fabsf(cd) + 0.194f * fmaf(2.f * cd, cd, -1.f) + 0.368f * fabsf(2.f * sd * cd);
  const float Tdiff = L.Ts - c.Ta;  // :1221
  const float kT = K * k * Tdiff;
  const float qcf1 = kT * fmaf(1.347f, __powf(reynold, 0.52f), 1.01f);  // (3a)  :1222
  const float qcf2 = kT * 0.754f * __powf(reynold, 0.6f);               // (3b)  :1223
  const float qcf = fmax_nan(qcf1, qcf2);                               // np.maximum keeps NaN  :1225
  const float rho = __fdividef(c.hn, rho_den);
  const float qcn = 3.645f * sqrtf(rho) * L.D075 * __powf(Tdiff, 1.25f);  // :1228 (Tdiff < 0 -> NaN)
  const float qc = fmax_nan(qcf, qcn);                                      // :1231
  const float ta = c.Ta * 0.01f;
  const float qr = L.qr_c * (L.Ts4 - (ta * ta) * (ta * ta));  // :1234
  const float u = fmaf(c.X, L.cpsi, c.Y * L.spsi);            // cos(Phi_s)  :1245-1247
  const float sin_s = sqrtf(fmax_nan(fmaf(-u, u, 1.f), 0.f));
  const float qs = L.qs_c * c.Q * sin_s;                      // :1249
  return sqrtf((qc + qr - qs) * L.inv_R);                     // :1251
}

// Imax >= 0 or NaN: as uint32 bit patterns the order of non-negative floats is the order of
// their bits, and 0xFFFFFFFF (the output's initial value, a NaN) lies above +inf.  -0 is made +0.
__device__ __forceinline__ uint32_t min_key(float v) {
  return v == v ? __float_as_uint(v == 0.f ? 0.f : v) : 0xFFFFFFFFu;
}

constexpr int LR_STAGE = 4;                // steps a warp parks in shared memory per chunk
constexpr int LR_ROW = TILE_CELLS + 1;     // floats per staged (quantity, step) row: +1 spreads
                                           // the LR_STAGE lanes reading one cell over 4 banks
constexpr int LR_NQ = 32 / LR_STAGE;       // lanes sharing a step split a slot's entries
static_assert(LR_NQ == PAIR_PAD, "one padded entry group per lane group");
constexpr int LR_FIELDS = 7;               // Ta, V, cw, sw, Q, X, Y (+ the static hn row)
constexpr int LR_WARP_FLOATS = LR_FIELDS * LR_STAGE * LR_ROW + LR_ROW;
constexpr int LR_WARPS = WARPS_PER_CTA;
constexpr size_t LR_SMEM = (size_t)LR_WARPS * LR_WARP_FLOATS * sizeof(float);

struct LrParams {
  // RAW: temp, wnd, waz, dir point to the raw ERA5 t2m, u100, v100, fdir
  const float *temp, *wnd, *waz, *dir, *height;
  const void *salt, *saz;
  const float4* tt;  // computed solar position: per step {sin dec, cos dec, cos H0, sin H0}
  const float2* xt;  // per column {cos lon, sin lon}
  const float2* yt;  // per row {sin lat, cos lat}
  const LineConst* lines;
  int t_off;         // index of the slab's first step in the operator's time axis
};

// SOLAR: ATL_SOLAR_COMPUTED / _STORED_F32 / _STORED_F64.  RAW: the four loaded fields are t2m, u100,
// v100, fdir; the wind speed, wind azimuth and direct influx are derived in registers with
// era5.prepare's arithmetic (era5_derive.cuh), sanitized, so the staged rows are bit for bit those
// of the prepared fields.  Same 16 B per cell-step.
template <bool VEC, int SOLAR, bool RAW>
__global__ void __launch_bounds__(CTA_THREADS, 3)
    k_line_rating(const LrParams p, const GridDev gd, const PlanDev plan, uint32_t* __restrict__ out, int nt,
                  int tb) {
  extern __shared__ __align__(16) float lr_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ai = blockIdx.x * LR_WARPS + warp;
  if (ai >= plan.n_active) return;
  const int tile = __ldg(plan.active_tiles + ai);
  const int s_beg = __ldg(plan.tile_slot_ptr + tile), s_end = __ldg(plan.tile_slot_ptr + tile + 1);
  const TileGeomT<VEC> g = make_geom<VEC>(tile, lane, gd);
  float* const st = lr_smem + warp * LR_WARP_FLOATS;
  float* const st_hn = st + LR_FIELDS * LR_STAGE * LR_ROW;
  {  // static: rho's numerator of the lane's 4 cells; value i of lane l at position 32 i + l
    float h[4];
    load4(p.height, 0, g, h);
#pragma unroll
    for (int i = 0; i < 4; ++i) st_hn[32 * i + lane] = rho_numerator(h[i]);
  }
  // computed solar position: the lane's column(s) and row(s)
  float clon[4], slon[4], sl[4], cl[4];
  if (SOLAR == ATL_SOLAR_COMPUTED) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 xc = __ldg(p.xt + min(g.cell_x(i), gd.nx - 1));
      const float2 yc = __ldg(p.yt + min(g.cell_y(i), gd.ny - 1));
      clon[i] = xc.x; slon[i] = xc.y; sl[i] = yc.x; cl[i] = yc.y;
    }
  }
  const int t0 = blockIdx.y * tb, t1 = min(nt, t0 + tb);
  const int64_t S4 = gd.S * 4;
  const int r = lane & (LR_STAGE - 1), q = lane / LR_STAGE;
  const int nl = plan.n_bus;
#pragma unroll 1
  for (int tc = t0; tc < t1; tc += LR_STAGE) {
    const int n = min(LR_STAGE, t1 - tc);
    // ---- stage
#pragma unroll 1
    for (int k = 0; k < n; ++k) {
      const int t = tc + k;
      const int64_t tbyte = (int64_t)t * S4;
      float Ta[4], V[4], wa[4], Q[4], X[4], Y[4];
      load4(p.temp, tbyte, g, Ta);
      load4(p.wnd, tbyte, g, V);
      load4(p.waz, tbyte, g, wa);
      load4(p.dir, tbyte, g, Q);
      if (RAW) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float u = V[i], v = wa[i];  // u100, v100
          V[i] = era5_wind_speed(u, v);     // era5.py:121
          wa[i] = era5_wind_azimuth(u, v);  // :129-130
          Q[i] = era5_direct(Q[i], 1);      // :168, 175, 199-200
        }
      }
      if (SOLAR == ATL_SOLAR_COMPUTED) {
        const float4 tq = __ldg(p.tt + p.t_off + t);  // pv/solar_position.py:103-114, as PvPhys
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float ch = fmaf(clon[i], tq.z, -slon[i] * tq.w);
          const float sh = fmaf(tq.w, clon[i], tq.z * slon[i]);
          X[i] = fmaf(-(tq.y * sl[i]), ch, tq.x * cl[i]);
          Y[i] = -tq.y * sh;
        }
      } else {
        float alt[4], az[4];
        if (SOLAR == ATL_SOLAR_STORED_F64) {
          load4(static_cast<const double*>(p.salt), tbyte, g, alt);
          load4(static_cast<const double*>(p.saz), tbyte, g, az);
        } else {
          load4(static_cast<const float*>(p.salt), tbyte, g, alt);
          load4(static_cast<const float*>(p.saz), tbyte, g, az);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float sa, ca, sz, cz;
          sincosf(alt[i], &sa, &ca);
          sincosf(az[i], &sz, &cz);
          X[i] = ca * cz;
          Y[i] = ca * sz;
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float sw, cw;
        sincosf(wa[i], &sw, &cw);
        float* const o = st + k * LR_ROW + 32 * i + lane;
        o[0 * LR_STAGE * LR_ROW] = Ta[i];
        o[1 * LR_STAGE * LR_ROW] = V[i];
        o[2 * LR_STAGE * LR_ROW] = cw;
        o[3 * LR_STAGE * LR_ROW] = sw;
        o[4 * LR_STAGE * LR_ROW] = Q[i];
        o[5 * LR_STAGE * LR_ROW] = X[i];
        o[6 * LR_STAGE * LR_ROW] = Y[i];
      }
    }
    __syncwarp();
    // ---- reduce: lane (q, r) = entry group q of step r; lanes past the chunk's last step compute
    // on stale rows and write nothing (every lane takes part in the shuffles)
    const bool live = r < n;
    const float* const rd = st + r * LR_ROW;
    uint32_t* const o_row = out + (size_t)(tc + r) * nl;
#pragma unroll 1
    for (int s = s_beg; s < s_end; ++s) {
      const int2 rec = __ldg(plan.slot_rec + s);
      const int line = __ldg(plan.slot_row + s);
      const LineConst L = p.lines[line];
      const PairEnt* e = plan.pairs + rec.x + q;
      uint32_t m = 0xFFFFFFFFu;
#pragma unroll 1
      for (int it = 0; it < rec.y; ++it, e += PAIR_PAD) {
        const PairEnt pe = *e;
        if (pe.w != 0.f) {  // weight 0: the plan's padding (the intersection matrix stores only 1.0)
          const int c = pe.off >> 3;
          LrCell v;
          v.Ta = rd[c];
          v.V = rd[c + 1 * LR_STAGE * LR_ROW];
          v.cw = rd[c + 2 * LR_STAGE * LR_ROW];
          v.sw = rd[c + 3 * LR_STAGE * LR_ROW];
          v.Q = rd[c + 4 * LR_STAGE * LR_ROW];
          v.X = rd[c + 5 * LR_STAGE * LR_ROW];
          v.Y = rd[c + 6 * LR_STAGE * LR_ROW];
          v.hn = st_hn[c];
          m = min(m, min_key(line_imax(L, v)));
        }
      }
#pragma unroll
      for (int o = LR_STAGE; o < 32; o <<= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (live && q == 0 && m != 0xFFFFFFFFu) atomicMin(o_row + line, m);
    }
    __syncwarp();
  }
}

__global__ void k_line_rating_flat(AtlLineRatingFlat f, int64_t n, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const LineConst L = make_line_const(f.psi[i], f.R[i], f.D[i], f.Ts[i], f.epsilon[i], f.alpha[i]);
    LrCell c;
    c.Ta = f.temperature[i];
    c.V = f.wnd100m[i];
    sincosf(f.wnd_azimuth[i], &c.sw, &c.cw);
    c.Q = f.influx_direct[i];
    float sa, ca, sz, cz;
    sincosf(f.solar_altitude[i], &sa, &ca);
    sincosf(f.solar_azimuth[i], &sz, &cz);
    c.X = ca * cz;
    c.Y = ca * sz;
    c.hn = rho_numerator(f.height[i]);
    out[i] = line_imax(L, c);
  }
}

}  // namespace atl

using namespace atl;

struct AtlLineRatingOp {
  int device;
  GridDev grid;
  int64_t nt;
  int solar_src;
  int32_t n_lines;
  float4* d_tt = nullptr;
  float2* d_xt = nullptr;
  float2* d_yt = nullptr;
  LineConst* d_lines = nullptr;
};

extern "C" {

int atl_line_rating_create(int device, const AtlLineRatingConfig* cfg, AtlLineRatingOp** op_out) {
  ATL_REQUIRE(cfg && op_out, "NULL argument");
  *op_out = nullptr;
  ATL_REQUIRE(cfg->ny > 0 && cfg->nx > 0 && cfg->nt >= 0 && cfg->n_lines >= 0, "bad shape");
  ATL_REQUIRE(cfg->pitch == 0 || cfg->pitch >= cfg->nx, "pitch must be >= nx");
  ATL_REQUIRE(cfg->solar_src >= 0 && cfg->solar_src <= 2, "bad solar source");
  ATL_REQUIRE(cfg->solar_src != ATL_SOLAR_COMPUTED || ((cfg->time_ns || cfg->nt == 0) && cfg->lon_deg && cfg->lat_deg),
              "time axis / coordinates missing");
  ATL_REQUIRE(cfg->n_lines == 0 || (cfg->psi && cfg->R && cfg->D && cfg->Ts && cfg->epsilon && cfg->alpha),
              "line parameters missing");
  std::vector<LineConst> lines((size_t)std::max(cfg->n_lines, 1));
  for (int32_t i = 0; i < cfg->n_lines; ++i)
    lines[(size_t)i] = make_line_const(cfg->psi[i], cfg->R[i], cfg->D[i], cfg->Ts[i], cfg->epsilon[i], cfg->alpha[i]);
  std::vector<float4> tt;
  std::vector<float2> xt((size_t)cfg->nx, make_float2(1.f, 0.f)), yt((size_t)cfg->ny, make_float2(0.f, 1.f));
  if (cfg->solar_src == ATL_SOLAR_COMPUTED) {
    solar_almanac(cfg->time_ns, cfg->nt, cfg->time_shift_ns, tt);
    const double D2R = 3.14159265358979323846 / 180.0;
    for (int i = 0; i < cfg->nx; ++i)
      xt[(size_t)i] = make_float2((float)std::cos(cfg->lon_deg[i] * D2R), (float)std::sin(cfg->lon_deg[i] * D2R));
    for (int j = 0; j < cfg->ny; ++j)
      yt[(size_t)j] = make_float2((float)std::sin(cfg->lat_deg[j] * D2R), (float)std::cos(cfg->lat_deg[j] * D2R));
  } else {
    tt.assign(1, make_float4(0.f, 1.f, 1.f, 0.f));
  }
  AtlLineRatingOp* op = new AtlLineRatingOp();
  op->device = device;
  op->grid = make_grid(cfg->ny, cfg->nx, cfg->pitch);
  op->nt = cfg->nt;
  op->solar_src = cfg->solar_src;
  op->n_lines = cfg->n_lines;
  cudaError_t e = cudaSetDevice(device);
  auto up = [&](auto** dst, const auto& v) {
    if (e == cudaSuccess) e = cudaMalloc((void**)dst, v.size() * sizeof(v[0]));
    if (e == cudaSuccess) e = cudaMemcpy(*dst, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
  };
  up(&op->d_tt, tt);
  up(&op->d_xt, xt);
  up(&op->d_yt, yt);
  up(&op->d_lines, lines);
  if (e != cudaSuccess) {
    atl_line_rating_destroy(op);
    return cuda_fail(e, "atl_line_rating_create");
  }
  *op_out = op;
  return ATL_OK;
}

void atl_line_rating_destroy(AtlLineRatingOp* op) {
  if (!op) return;
  cudaSetDevice(op->device);
  cudaFree(op->d_tt);
  cudaFree(op->d_xt);
  cudaFree(op->d_yt);
  cudaFree(op->d_lines);
  delete op;
}

}  // extern "C"

// One slab of either field set: the pointers go to the kernel's four field slots in this order
// (temperature / t2m, wnd100m / u100, wnd_azimuth / v100, influx_direct / fdir).
static int line_rating_launch(const AtlLineRatingOp* op, const AtlPlan* plan, const void* const fld[4],
                              const float* height, const void* salt, const void* saz, bool raw, int64_t t0,
                              int64_t nt, float* out_dev, void* stream) {
  ATL_REQUIRE(op->solar_src == ATL_SOLAR_COMPUTED || (salt && saz), "stored solar position fields missing");
  ATL_REQUIRE(t0 >= 0 && nt >= 0 && (op->solar_src != ATL_SOLAR_COMPUTED || t0 + nt <= op->nt),
              "slab outside the operator's time axis");
  ATL_REQUIRE(nt < (1LL << 31), "slab too long");
  ATL_REQUIRE(plan->grid.nx == op->grid.nx && plan->grid.ny == op->grid.ny && plan->grid.pitch == op->grid.pitch,
              "plan / operator grid (or pitch) mismatch");
  ATL_REQUIRE(plan->n_bus == op->n_lines, "plan rows / line count mismatch");
  ATL_REQUIRE(plan->n_active == 0 || (plan->d_pairs && plan->d_slot_rec),
              "the plan has no entry lists (create it with atl_plan_create_entries)");
  ATL_CUDA(cudaSetDevice(op->device));
  cudaStream_t st = (cudaStream_t)stream;
  ATL_CUDA(cudaMemsetAsync(out_dev, 0xFF, (size_t)nt * plan->n_bus * sizeof(float), st));  // NaN: no valid cell
  if (nt == 0 || plan->n_active == 0) return ATL_OK;
  const void* ps[] = {fld[0], fld[1], fld[2], fld[3], height, salt, saz};
  bool al = true;
  for (const void* q : ps) al = al && aligned16(q);
  ATL_REQUIRE(!plan->vec || al, "field pointers must be 16-byte aligned (pitch % 4 == 0 uses 128-bit loads)");
  LrParams p;
  p.temp = static_cast<const float*>(fld[0]);
  p.wnd = static_cast<const float*>(fld[1]);
  p.waz = static_cast<const float*>(fld[2]);
  p.dir = static_cast<const float*>(fld[3]);
  p.height = height;
  p.salt = salt;
  p.saz = saz;
  p.tt = op->d_tt;
  p.xt = op->d_xt;
  p.yt = op->d_yt;
  p.lines = op->d_lines;
  p.t_off = (int)t0;
  const int gx = (plan->n_active + LR_WARPS - 1) / LR_WARPS;
  int tb = pick_tb(gx, nt);
  tb = (tb + LR_STAGE - 1) / LR_STAGE * LR_STAGE;
  const dim3 grid(gx, (unsigned)((nt + tb - 1) / tb));
  const PlanDev pd = plan->dev();
  uint32_t* out = reinterpret_cast<uint32_t*>(out_dev);
#define LR_LAUNCH(V, S, R)                                                                    \
  do {                                                                                        \
    ATL_CUDA(cudaFuncSetAttribute(k_line_rating<V, S, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LR_SMEM)); \
    k_line_rating<V, S, R><<<grid, CTA_THREADS, LR_SMEM, st>>>(p, plan->grid, pd, out, (int)nt, tb);  \
  } while (0)
#define LR_LAUNCH_SOLAR(V, R)                                                     \
  do {                                                                            \
    if (op->solar_src == ATL_SOLAR_COMPUTED) LR_LAUNCH(V, ATL_SOLAR_COMPUTED, R);     \
    else if (op->solar_src == ATL_SOLAR_STORED_F32) LR_LAUNCH(V, ATL_SOLAR_STORED_F32, R); \
    else LR_LAUNCH(V, ATL_SOLAR_STORED_F64, R);                                   \
  } while (0)
  if (plan->vec) {
    if (raw) LR_LAUNCH_SOLAR(true, true);
    else LR_LAUNCH_SOLAR(true, false);
  } else {
    if (raw) LR_LAUNCH_SOLAR(false, true);
    else LR_LAUNCH_SOLAR(false, false);
  }
#undef LR_LAUNCH_SOLAR
#undef LR_LAUNCH
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

extern "C" {

int atl_line_rating_reduce(const AtlLineRatingOp* op, const AtlPlan* plan, const AtlLineRatingFields* f,
                           int64_t t0, int64_t nt, float* out_dev, void* stream) {
  ATL_REQUIRE(op && plan && f && out_dev, "NULL argument");
  ATL_REQUIRE(f->temperature && f->wnd100m && f->wnd_azimuth && f->influx_direct && f->height,
              "line rating fields missing: temperature, wnd100m, wnd_azimuth, influx_direct, height");
  const void* fld[4] = {f->temperature, f->wnd100m, f->wnd_azimuth, f->influx_direct};
  return line_rating_launch(op, plan, fld, f->height, f->solar_altitude, f->solar_azimuth, false, t0, nt, out_dev,
                            stream);
}

int atl_line_rating_raw_reduce(const AtlLineRatingOp* op, const AtlPlan* plan, const AtlLineRatingRawFields* f,
                               int64_t t0, int64_t nt, float* out_dev, void* stream) {
  ATL_REQUIRE(op && plan && f && out_dev, "NULL argument");
  ATL_REQUIRE(f->t2m && f->u100 && f->v100 && f->fdir && f->height,
              "raw line rating fields missing: t2m, u100, v100, fdir, height");
  const void* fld[4] = {f->t2m, f->u100, f->v100, f->fdir};
  return line_rating_launch(op, plan, fld, f->height, f->solar_altitude, f->solar_azimuth, true, t0, nt, out_dev,
                            stream);
}

int atl_line_rating_eval(int device, int64_t n, const AtlLineRatingFlat* f, float* out_dev, void* stream) {
  ATL_REQUIRE(f && n >= 0, "bad arguments");
  if (n == 0) return ATL_OK;
  ATL_REQUIRE(out_dev && f->temperature && f->wnd100m && f->wnd_azimuth && f->influx_direct && f->height &&
                  f->solar_altitude && f->solar_azimuth && f->psi && f->R && f->D && f->Ts && f->epsilon &&
                  f->alpha,
              "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  const int threads = 256;
  const int64_t blocks = std::min<int64_t>((n + threads - 1) / threads, (int64_t)sm_count() * 16);
  k_line_rating_flat<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(*f, n, out_dev);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // extern "C"
