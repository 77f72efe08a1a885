// host_stream.cu -- host-buffer entry points: the cutout lives in host memory
// (NumPy arrays / NetCDF-backed), time slabs are streamed through a
// double-buffered device ring so H2D copies overlap the fused kernels, and the
// (time, bus) result is returned in host memory.  This is the call behind the
// reference-facing `Cutout.pv/wind/heat_demand(...)` when no device-resident
// copy of the cutout exists (bench.py "e2e").
//
// Pinned (cudaHostAlloc / cudaHostRegister'ed) inputs are DMA'd directly;
// pageable inputs go through a pinned staging ring (memcpy -> async H2D).
#include <sched.h>

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <type_traits>
#include <vector>

#include "kernels.cuh"

namespace atl {

constexpr int NBUF = 2;

struct SlabField {
  const char* host;  // nullptr = unused
  size_t elem;       // bytes per element
};

static bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

// Pinned staging buffers for pageable inputs are kept across calls (cudaHostAlloc
// of a few hundred MiB costs more than the transfer it serves); a call takes
// buffers out of the pool and puts them back when it returns.
struct StagePool {
  std::mutex mu;
  std::vector<std::pair<char*, size_t>> free_list;
  char* take(size_t bytes) {
    {
      std::lock_guard<std::mutex> lk(mu);
      int best = -1;
      for (int i = 0; i < (int)free_list.size(); ++i)
        if (free_list[i].second >= bytes && (best < 0 || free_list[i].second < free_list[best].second))
          best = i;
      if (best >= 0) {
        char* p = free_list[best].first;
        sizes.push_back({p, free_list[best].second});
        free_list.erase(free_list.begin() + best);
        return p;
      }
    }
    char* p = nullptr;
    if (cudaHostAlloc((void**)&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
      cudaGetLastError();
      release();  // drop cached buffers and retry once
      if (cudaHostAlloc((void**)&p, bytes, cudaHostAllocPortable) != cudaSuccess) return nullptr;
    }
    std::lock_guard<std::mutex> lk(mu);
    sizes.push_back({p, bytes});
    return p;
  }
  void give(char* p) {
    std::lock_guard<std::mutex> lk(mu);
    for (size_t i = 0; i < sizes.size(); ++i)
      if (sizes[i].first == p) {
        free_list.push_back(sizes[i]);
        sizes.erase(sizes.begin() + i);
        return;
      }
  }
  void release() {
    std::lock_guard<std::mutex> lk(mu);
    for (auto& b : free_list) cudaFreeHost(b.first);
    free_list.clear();
  }
  std::vector<std::pair<char*, size_t>> sizes;  // buffers currently lent out
};
// One pool per device: its buffers are allocated (and first touched) by a thread bound to
// the CPUs next to that GPU, so they live on the GPU's NUMA node.
static StagePool g_stage_pool[64];
static StagePool& stage_pool(int device) { return g_stage_pool[(device >= 0 && device < 64) ? device : 0]; }

// ---- NUMA placement.  On a two-socket box half of the GPUs hang off each socket; a host
// thread that stages data for (or allocates pinned memory for) a GPU of the other socket
// pays the inter-socket link for every byte.  While a call streams slabs to device d, the
// calling thread -- and the staging-copy threads it spawns, which inherit the mask -- run on
// the CPUs the kernel lists as local to that PCI device
// (/sys/bus/pci/devices/<bus id>/local_cpulist).  ATL_NUMA_BIND=0 turns this off.
static bool device_local_cpus(int device, cpu_set_t* out) {
  static std::mutex mu;
  static bool known[64] = {false}, ok[64] = {false};
  static cpu_set_t sets[64];
  if (device < 0 || device >= 64) return false;
  std::lock_guard<std::mutex> lk(mu);
  if (!known[device]) {
    known[device] = true;
    const char* env = getenv("ATL_NUMA_BIND");
    char bus[64] = {0};
    if (!(env && atoi(env) == 0) && cudaDeviceGetPCIBusId(bus, sizeof bus, device) == cudaSuccess) {
      for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
      char path[160];
      snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/local_cpulist", bus);
      if (FILE* fh = fopen(path, "r")) {
        char line[4096] = {0};
        if (fgets(line, sizeof line, fh)) {
          CPU_ZERO(&sets[device]);
          int n = 0;
          for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int a = -1, b = -1;
            if (sscanf(tok, "%d-%d", &a, &b) == 2) {
            } else if (sscanf(tok, "%d", &a) == 1) {
              b = a;
            }
            for (int c = a; c >= 0 && c <= b && c < CPU_SETSIZE; ++c, ++n) CPU_SET(c, &sets[device]);
          }
          ok[device] = n > 0;
        }
        fclose(fh);
      }
    } else {
      cudaGetLastError();
    }
  }
  if (ok[device]) *out = sets[device];
  return ok[device];
}

// RAII: bind the calling thread to the device's local CPUs (intersected with the mask it
// already has), restore on scope exit.
struct NumaBind {
  cpu_set_t saved;
  bool active = false;
  explicit NumaBind(int device) {
    cpu_set_t local;
    if (!device_local_cpus(device, &local)) return;
    if (sched_getaffinity(0, sizeof saved, &saved) != 0) return;
    cpu_set_t both;
    CPU_AND(&both, &saved, &local);
    if (CPU_COUNT(&both) == 0) return;
    active = sched_setaffinity(0, sizeof both, &both) == 0;
  }
  ~NumaBind() {
    if (active) sched_setaffinity(0, sizeof saved, &saved);
  }
};

// Pageable -> pinned copy on several host threads (one thread moves ~10 GB/s, the
// PCIe link wants 50+).
static void par_memcpy(char* dst, const char* src, size_t bytes) {
  static const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
  const size_t kMin = 1u << 20;  // measured: 4 threads move ~13 GB/s on the bench box
  unsigned nthr = (unsigned)std::min<size_t>(std::min(16u, hw), bytes / kMin);
  if (nthr <= 1) {
    std::memcpy(dst, src, bytes);
    return;
  }
  const size_t part = ((bytes / nthr) + 4095) & ~(size_t)4095;
  std::vector<std::thread> th;
  for (unsigned k = 1; k < nthr; ++k) {
    const size_t off = (size_t)k * part;
    if (off >= bytes) break;
    th.emplace_back([=] { std::memcpy(dst + off, src + off, std::min(part, bytes - off)); });
  }
  std::memcpy(dst, src, std::min(part, bytes));
  for (auto& t : th) t.join();
}

static void pool_keep_memory(int device) {
  static bool done[64] = {false};
  if (device < 0 || device >= 64 || done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done[device] = true;
}

// A job's own slab schedule: slab k covers units [unit[k], unit[k + 1]) = steps [step[k], step[k + 1]).
// It is the schedule the job's single-operator call streams, so that every launch -- and with it
// every result bit -- is the same whether the job runs alone or shares a pass: the kernels pair up
// consecutive steps from the start of each launch, and a NaN in one step of a pair sends both down
// the exact path, which may round the other step differently.
struct Schedule {
  std::vector<int64_t> unit, step;
  int64_t max_steps() const {
    int64_t m = 0;
    for (size_t k = 0; k + 1 < step.size(); ++k) m = std::max(m, step[k + 1] - step[k]);
    return m;
  }
};

// `n_units` units, unit u starting at step unit_start(u) (identity + `first` without a table), in
// slabs of `chunk` units; chunk <= 0: ~192 MiB of `bytes_per_step` input per slab.
static Schedule make_schedule(int64_t n_units, const int64_t* unit_start, int64_t first, int64_t chunk,
                              size_t bytes_per_step) {
  auto ustart = [&](int64_t u) { return unit_start ? unit_start[u] : first + u; };
  Schedule s;
  if (n_units <= 0) return s;
  if (chunk <= 0) {
    // ~192 MiB of input per slab: long enough to amortise launch + copy setup,
    // short enough that the first kernel starts early
    const double steps_per_unit = (double)(ustart(n_units) - ustart(0)) / (double)n_units;
    chunk = (int64_t)((192.0 * (1 << 20)) / ((double)bytes_per_step * steps_per_unit));
    if (chunk < 2) chunk = 2;
  }
  for (int64_t u = 0; u < n_units; u += chunk) {
    s.unit.push_back(u);
    s.step.push_back(ustart(u));
  }
  s.unit.push_back(n_units);
  s.step.push_back(ustart(n_units));
  return s;
}

// One reduce the ring feeds: the ring field behind each member of its field struct, its own slab
// schedule, where its output rows go, and its device reduce of one slab.
struct SlabJob {
  std::vector<int> slot;  // ring field of each member of the job's field struct, -1 = absent
  Schedule own;
  bool per_unit;          // one output row per unit (heat days); else one per step
  int32_t n_bus;
  int64_t rows;
  float* out_host;
  // launch(members, u, e, step0, n, out_dev, stream): the reduce of units [u, e) = steps
  // [step0, step0 + n) of the host arrays, whose device copies `members` point at, into out_dev
  std::function<int(const std::vector<void*>& members, int64_t u, int64_t e, int64_t step0, int64_t n,
                    float* out_dev, cudaStream_t st)>
      launch;
};

// Stream the union `fields` of the jobs' host fields through the device ring once, in the slabs of
// `ring`: every field is copied host -> device once per slab however many jobs read it.  A job whose
// own schedule is the ring's reduces each ring slot in place; any other job gets its own two-slot
// window, which its slabs are assembled in from the ring slots (device -> device), and reduces each
// of its slabs there as soon as the slab is complete.
static int stream_slabs(int device, const std::vector<SlabField>& fields, int64_t S, const Schedule& ring,
                        const std::vector<SlabJob>& jobs, AtlStreamStats* stats) {
  for (const auto& j : jobs) ATL_REQUIRE(j.out_host, "NULL output");
  const int64_t n_ring = (int64_t)ring.step.size() - 1;
  if (n_ring <= 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  NumaBind numa(device);
  StagePool& g_stage = stage_pool(device);
  pool_keep_memory(device);
  size_t bytes_per_step = 0;
  for (const auto& f : fields)
    if (f.host) bytes_per_step += (size_t)S * f.elem;
  ATL_REQUIRE(bytes_per_step > 0, "no input fields");
  const int64_t max_steps = ring.max_steps();
  const size_t nj = jobs.size();

  cudaStream_t s_copy = nullptr, s_comp = nullptr;
  cudaEvent_t ev_copied[NBUF] = {nullptr}, ev_done[NBUF] = {nullptr}, ev_staged[NBUF] = {nullptr};
  std::vector<std::vector<void*>> dev(NBUF, std::vector<void*>(fields.size(), nullptr));
  std::vector<std::vector<char*>> stage(NBUF, std::vector<char*>(fields.size(), nullptr));
  std::vector<float*> out_dev(nj, nullptr);
  // windowed jobs: window slot w of job j, member m; its events; the next slab it reduces
  std::vector<bool> direct(nj, false);
  std::vector<std::vector<std::vector<void*>>> win(nj);
  std::vector<std::vector<cudaEvent_t>> wev_copied(nj, std::vector<cudaEvent_t>(NBUF, nullptr)),
      wev_done(nj, std::vector<cudaEvent_t>(NBUF, nullptr));
  std::vector<size_t> next(nj, 0);
  std::vector<void*> members;
  int rc = ATL_OK;
  std::vector<bool> pinned(fields.size(), false);
  AtlStreamStats count{0, 0};

#define SS_CUDA(call)                      \
  do {                                     \
    cudaError_t _e = (call);               \
    if (_e != cudaSuccess) {               \
      rc = cuda_fail(_e, #call);           \
      goto cleanup;                        \
    }                                      \
  } while (0)

  SS_CUDA(cudaStreamCreateWithFlags(&s_copy, cudaStreamNonBlocking));
  SS_CUDA(cudaStreamCreateWithFlags(&s_comp, cudaStreamNonBlocking));
  for (int b = 0; b < NBUF; ++b) {
    SS_CUDA(cudaEventCreateWithFlags(&ev_copied[b], cudaEventDisableTiming));
    SS_CUDA(cudaEventCreateWithFlags(&ev_done[b], cudaEventDisableTiming));
    SS_CUDA(cudaEventCreateWithFlags(&ev_staged[b], cudaEventDisableTiming));
  }
  for (size_t i = 0; i < fields.size(); ++i) {
    if (!fields[i].host) continue;
    pinned[i] = is_pinned(fields[i].host);
    const size_t bytes = (size_t)max_steps * S * fields[i].elem;
    for (int b = 0; b < NBUF; ++b) {
      SS_CUDA(cudaMallocAsync(&dev[b][i], bytes, s_copy));
      if (!pinned[i]) {
        stage[b][i] = g_stage.take(bytes);
        if (!stage[b][i]) {
          set_error("out of pinned host memory for the staging ring");
          rc = ATL_ERR_CUDA;
          goto cleanup;
        }
      }
    }
  }
  for (size_t j = 0; j < nj; ++j) {
    SS_CUDA(cudaMallocAsync((void**)&out_dev[j], (size_t)jobs[j].rows * jobs[j].n_bus * sizeof(float) + 16, s_copy));
    direct[j] = jobs[j].own.step == ring.step;
    if (direct[j]) continue;
    const int64_t w_steps = jobs[j].own.max_steps();
    win[j].assign(NBUF, std::vector<void*>(jobs[j].slot.size(), nullptr));
    for (int w = 0; w < NBUF; ++w) {
      SS_CUDA(cudaEventCreateWithFlags(&wev_copied[j][w], cudaEventDisableTiming));
      SS_CUDA(cudaEventCreateWithFlags(&wev_done[j][w], cudaEventDisableTiming));
      for (size_t m = 0; m < jobs[j].slot.size(); ++m)
        if (jobs[j].slot[m] >= 0)
          SS_CUDA(cudaMallocAsync(&win[j][w][m], (size_t)w_steps * S * fields[jobs[j].slot[m]].elem, s_copy));
    }
  }
  SS_CUDA(cudaStreamSynchronize(s_copy));

  for (int64_t it = 0; it < n_ring; ++it) {
    const int b = (int)(it % NBUF);
    const int64_t r0 = ring.step[it], r1 = ring.step[it + 1];
    // the ring slot is free once the kernels that read it in place have finished
    if (it >= NBUF) SS_CUDA(cudaStreamWaitEvent(s_copy, ev_done[b], 0));
    for (size_t i = 0; i < fields.size(); ++i) {
      if (!fields[i].host) continue;
      const size_t off = (size_t)r0 * S * fields[i].elem;
      const size_t bytes = (size_t)(r1 - r0) * S * fields[i].elem;
      const char* src = fields[i].host + off;
      if (!pinned[i]) {
        if (it >= NBUF) SS_CUDA(cudaEventSynchronize(ev_staged[b]));  // staging slot drained
        par_memcpy(stage[b][i], src, bytes);
        src = stage[b][i];
      }
      SS_CUDA(cudaMemcpyAsync(dev[b][i], src, bytes, cudaMemcpyHostToDevice, s_copy));
      count.h2d_bytes += (int64_t)bytes;
    }
    ++count.n_slabs;
    SS_CUDA(cudaEventRecord(ev_staged[b], s_copy));
    SS_CUDA(cudaEventRecord(ev_copied[b], s_copy));
    SS_CUDA(cudaStreamWaitEvent(s_comp, ev_copied[b], 0));
    for (size_t j = 0; j < nj; ++j) {
      const SlabJob& job = jobs[j];
      const auto& own = job.own;
      auto launch = [&](size_t k, const std::vector<void*>& mem) {
        const int64_t row0 = job.per_unit ? own.unit[k] : own.step[k];
        return job.launch(mem, own.unit[k], own.unit[k + 1], own.step[k], own.step[k + 1] - own.step[k],
                          out_dev[j] + (size_t)row0 * job.n_bus, s_comp);
      };
      if (direct[j]) {
        members.assign(job.slot.size(), nullptr);
        for (size_t m = 0; m < job.slot.size(); ++m)
          if (job.slot[m] >= 0) members[m] = dev[b][job.slot[m]];
        rc = launch((size_t)it, members);
        if (rc != ATL_OK) goto cleanup;
        continue;
      }
      // the job's slabs that overlap this ring slab: copy the overlap into the slab's window slot,
      // and reduce every slab this ring slab completes
      for (size_t k = next[j]; k + 1 < own.step.size(); ++k) {
        const int64_t a = own.step[k], e = own.step[k + 1];
        if (e > r1 && a >= r1) break;  // starts with a later ring slab
        const int64_t lo = std::max(a, r0), hi = std::min(e, r1);
        const int w = (int)(k % NBUF);
        if (hi > lo) {
          if (lo == a && k >= (size_t)NBUF) SS_CUDA(cudaStreamWaitEvent(s_copy, wev_done[j][w], 0));
          for (size_t m = 0; m < job.slot.size(); ++m) {
            if (job.slot[m] < 0) continue;
            const size_t el = fields[job.slot[m]].elem;
            SS_CUDA(cudaMemcpyAsync((char*)win[j][w][m] + (size_t)(lo - a) * S * el,
                                    (const char*)dev[b][job.slot[m]] + (size_t)(lo - r0) * S * el,
                                    (size_t)(hi - lo) * S * el, cudaMemcpyDeviceToDevice, s_copy));
          }
        }
        if (e > r1) break;  // the rest of this slab comes with the next ring slab
        SS_CUDA(cudaEventRecord(wev_copied[j][w], s_copy));
        SS_CUDA(cudaStreamWaitEvent(s_comp, wev_copied[j][w], 0));
        rc = launch(k, win[j][w]);
        if (rc != ATL_OK) goto cleanup;
        SS_CUDA(cudaEventRecord(wev_done[j][w], s_comp));
        next[j] = k + 1;
      }
    }
    SS_CUDA(cudaEventRecord(ev_done[b], s_comp));
  }
  for (size_t j = 0; j < nj; ++j)
    SS_CUDA(cudaMemcpyAsync(jobs[j].out_host, out_dev[j], (size_t)jobs[j].rows * jobs[j].n_bus * sizeof(float),
                            cudaMemcpyDeviceToHost, s_comp));
  SS_CUDA(cudaStreamSynchronize(s_comp));
  SS_CUDA(cudaStreamSynchronize(s_copy));
  if (stats) *stats = count;

cleanup:
  if (s_comp) cudaStreamSynchronize(s_comp);
  if (s_copy) cudaStreamSynchronize(s_copy);
  for (int b = 0; b < NBUF; ++b) {
    for (size_t i = 0; i < fields.size(); ++i) {
      if (dev[b][i]) cudaFreeAsync(dev[b][i], s_copy ? s_copy : 0);
      if (stage[b][i]) g_stage.give(stage[b][i]);
    }
    if (ev_copied[b]) cudaEventDestroy(ev_copied[b]);
    if (ev_done[b]) cudaEventDestroy(ev_done[b]);
    if (ev_staged[b]) cudaEventDestroy(ev_staged[b]);
  }
  for (size_t j = 0; j < nj; ++j) {
    if (out_dev[j]) cudaFreeAsync(out_dev[j], s_copy ? s_copy : 0);
    for (auto& w : win[j])
      for (void* p : w)
        if (p) cudaFreeAsync(p, s_copy ? s_copy : 0);
    for (int w = 0; w < NBUF; ++w) {
      if (wev_copied[j][w]) cudaEventDestroy(wev_copied[j][w]);
      if (wev_done[j][w]) cudaEventDestroy(wev_done[j][w]);
    }
  }
  if (s_copy) {
    cudaStreamSynchronize(s_copy);
    cudaStreamDestroy(s_copy);
  }
  if (s_comp) cudaStreamDestroy(s_comp);
#undef SS_CUDA
  return rc;
}

int heat_launch_core(int mode, const AtlHeatOp* op, const AtlPlan* plan, const float* temp,
                     const int32_t* d_days, int32_t base, const int64_t* day_start_host,
                     int64_t n_days, float* out, cudaStream_t st, float* cnt_out);
int heat_upload_days(const int64_t* day_start, int64_t n_days, int32_t** d_out, cudaStream_t st);

// A field struct from the device copies `d` of its members (all of them pointers, in member order).
template <class F>
static F unpack(const std::vector<void*>& d) {
  static_assert(std::is_trivially_copyable<F>::value && sizeof(F) % sizeof(void*) == 0, "a struct of pointers");
  F f;
  std::memcpy(&f, d.data(), sizeof(F));
  return f;
}

// The host pointer of each member of job `j`'s field struct with its bytes per element (8 B for a
// stored float64 solar position, 4 B otherwise), and the operator's device and grid.
static int job_fields(const AtlStreamJob& j, std::vector<SlabField>& m, int32_t* device, int32_t* ny,
                      int32_t* nx) {
  int32_t solar_src = ATL_SOLAR_COMPUTED;
  auto members = [&](std::initializer_list<size_t> elem) {
    const char* host[16];
    std::memcpy(host, j.fields, elem.size() * sizeof(void*));
    m.clear();
    for (size_t e : elem) m.push_back({host[m.size()], e});
  };
  switch (j.kind) {
    case ATL_JOB_PV: {
      static_assert(sizeof(AtlPvFields) == 10 * sizeof(void*), "ten PV fields");
      atl_pv_op_info((const AtlPvOp*)j.op, device, ny, nx, &solar_src);
      const size_t sol = solar_src == ATL_SOLAR_STORED_F64 ? 8 : 4;
      members({4, 4, 4, 4, 4, 4, 4, 4, sol, sol});
      return ATL_OK;
    }
    case ATL_JOB_WIND:
      static_assert(sizeof(AtlWindFields) == 2 * sizeof(void*), "two wind fields");
      atl_wind_op_info((const AtlWindOp*)j.op, device, ny, nx);
      members({4, 4});
      return ATL_OK;
    case ATL_JOB_WIND_RAW:
      static_assert(sizeof(AtlWindRawFields) == 5 * sizeof(void*), "five raw wind fields");
      atl_wind_op_info((const AtlWindOp*)j.op, device, ny, nx);
      members({4, 4, 4, 4, 4});
      return ATL_OK;
    case ATL_JOB_CSP: {
      static_assert(sizeof(AtlCspFields) == 3 * sizeof(void*), "three CSP fields");
      atl_csp_op_info((const AtlCspOp*)j.op, device, ny, nx, &solar_src);
      const size_t sol = solar_src == ATL_SOLAR_STORED_F64 ? 8 : 4;
      members({4, sol, sol});
      return ATL_OK;
    }
    case ATL_JOB_POINTWISE:
      atl_pointwise_op_info((const AtlPointwiseOp*)j.op, device, ny, nx);
      m.assign(1, {(const char*)j.fields, 4});
      return ATL_OK;
    case ATL_JOB_HEAT:
      atl_heat_op_info((const AtlHeatOp*)j.op, device, ny, nx);
      m.assign(1, {(const char*)j.fields, 4});
      return ATL_OK;
  }
  set_error("unknown stream job kind");
  return ATL_ERR_INVALID;
}

using SlabLaunch = decltype(SlabJob::launch);

// Job `j`'s device reduce of one of its slabs: a step job at its operator's step t0 + the slab's
// first step, a heat job over the slab's days (`d_days`: the job's whole day table on the device).
static SlabLaunch job_launch(const AtlStreamJob& j, const int32_t* d_days) {
  const AtlPlan* plan = j.plan;
  const void* op = j.op;
  const int64_t t0 = j.t0;
  const int64_t* day_start = j.day_start;
  switch (j.kind) {
    case ATL_JOB_PV:
      return [=](const std::vector<void*>& d, int64_t, int64_t, int64_t s0, int64_t n, float* out, cudaStream_t st) {
        const AtlPvFields f = unpack<AtlPvFields>(d);
        return atl_pv_reduce((const AtlPvOp*)op, plan, &f, t0 + s0, n, out, (void*)st);
      };
    case ATL_JOB_WIND:
      return [=](const std::vector<void*>& d, int64_t, int64_t, int64_t, int64_t n, float* out, cudaStream_t st) {
        const AtlWindFields f = unpack<AtlWindFields>(d);
        return atl_wind_reduce((const AtlWindOp*)op, plan, &f, n, out, (void*)st);
      };
    case ATL_JOB_WIND_RAW:
      return [=](const std::vector<void*>& d, int64_t, int64_t, int64_t, int64_t n, float* out, cudaStream_t st) {
        const AtlWindRawFields f = unpack<AtlWindRawFields>(d);
        return atl_wind_raw_reduce((const AtlWindOp*)op, plan, &f, n, out, (void*)st);
      };
    case ATL_JOB_CSP:
      return [=](const std::vector<void*>& d, int64_t, int64_t, int64_t s0, int64_t n, float* out, cudaStream_t st) {
        const AtlCspFields f = unpack<AtlCspFields>(d);
        return atl_csp_reduce((const AtlCspOp*)op, plan, &f, t0 + s0, n, out, (void*)st);
      };
    case ATL_JOB_POINTWISE:
      return [=](const std::vector<void*>& d, int64_t, int64_t, int64_t, int64_t n, float* out, cudaStream_t st) {
        return atl_pointwise_reduce((const AtlPointwiseOp*)op, plan, (const float*)d[0], n, out, (void*)st);
      };
    default:  // ATL_JOB_HEAT (job_fields has rejected every other kind)
      return [=](const std::vector<void*>& d, int64_t u, int64_t e, int64_t, int64_t, float* out, cudaStream_t st) {
        return heat_launch_core(0, (const AtlHeatOp*)op, plan, (const float*)d[0], d_days + u,
                                (int32_t)day_start[u], day_start + u, e - u, out, st, nullptr);
      };
  }
}

// Every job is checked against the call's device and grid, and its day table against the steps,
// before anything is allocated or launched; then the union of the jobs' fields streams once, in the
// slabs of `ring` (NULL: chunk_steps, or ~192 MiB of the union's input, per slab).
static int reduce_host_many(int32_t device, int32_t ny, int32_t nx, int64_t nt, const AtlStreamJob* jobs,
                            int32_t n_jobs, int64_t chunk_steps, const Schedule* ring, AtlStreamStats* stats) {
  if (stats) *stats = AtlStreamStats{0, 0};
  ATL_REQUIRE(n_jobs >= 0 && (jobs || n_jobs == 0), "NULL jobs");
  ATL_REQUIRE(ny > 0 && nx > 0 && nt >= 0, "bad grid or step count");
  const int64_t S = (int64_t)ny * nx;
  std::vector<SlabField> fields, m;
  std::vector<SlabJob> slab_jobs(n_jobs);
  int64_t lo = nt, hi = 0;  // the steps some job reads
  for (int32_t k = 0; k < n_jobs; ++k) {
    const AtlStreamJob& j = jobs[k];
    ATL_REQUIRE(j.op && j.plan && j.fields, "NULL argument");
    ATL_REQUIRE(j.out_host, "NULL output");
    int32_t d = -1, gy = 0, gx = 0;
    int rc = job_fields(j, m, &d, &gy, &gx);
    if (rc != ATL_OK) return rc;
    AtlPlanInfo pi;
    atl_plan_info(j.plan, &pi);
    if (d != device || gy != ny || gx != nx || pi.ny != ny || pi.nx != nx) {
      char msg[200];
      snprintf(msg, sizeof msg, "job %d: operator on device %d with grid %dx%d, plan grid %dx%d; the call is on "
               "device %d with grid %dx%d", k, d, gy, gx, pi.ny, pi.nx, device, ny, nx);
      set_error(msg);
      return ATL_ERR_INVALID;
    }
    SlabJob& s = slab_jobs[k];
    s.per_unit = j.kind == ATL_JOB_HEAT;
    if (s.per_unit) {
      ATL_REQUIRE(j.day_start && j.n_days >= 0 && j.n_days < (1LL << 31), "a heat job needs its day table");
      for (int64_t u = 0; u < j.n_days; ++u) ATL_REQUIRE(j.day_start[u] <= j.day_start[u + 1], "day table not ascending");
      ATL_REQUIRE(j.day_start[0] >= 0 && j.day_start[j.n_days] <= nt, "the day table reaches past the fields' steps");
    }
    s.n_bus = pi.n_bus;
    s.out_host = j.out_host;
    size_t own_bytes = 0;  // its single call's input per step (a field it reads twice counts twice)
    for (const SlabField& f : m) {
      int slot = -1;
      if (f.host) {  // one ring field per host array, however many jobs read it
        own_bytes += (size_t)S * f.elem;
        for (size_t i = 0; i < fields.size() && slot < 0; ++i)
          if (fields[i].host == f.host && fields[i].elem == f.elem) slot = (int)i;
        if (slot < 0) {
          slot = (int)fields.size();
          fields.push_back(f);
        }
      }
      s.slot.push_back(slot);
    }
    ATL_REQUIRE(own_bytes > 0, "no input fields");
    s.rows = s.per_unit ? j.n_days : nt;
    s.own = s.per_unit ? make_schedule(j.n_days, j.day_start, 0, j.chunk, own_bytes)
                       : make_schedule(nt, nullptr, 0, j.chunk, own_bytes);
    if (s.own.step.size() > 1) {
      lo = std::min(lo, s.own.step.front());
      hi = std::max(hi, s.own.step.back());
    }
  }
  if (n_jobs == 0 || hi <= lo) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  std::vector<int32_t*> d_days(n_jobs, nullptr);
  int rc = ATL_OK;
  for (int32_t k = 0; k < n_jobs && rc == ATL_OK; ++k) {
    if (jobs[k].kind == ATL_JOB_HEAT && jobs[k].n_days > 0)  // one upload of its day table; slabs index into it
      rc = heat_upload_days(jobs[k].day_start, jobs[k].n_days, &d_days[k], 0);
    slab_jobs[k].launch = job_launch(jobs[k], d_days[k]);
  }
  if (rc == ATL_OK) {
    size_t union_bytes = 0;
    for (const auto& f : fields) union_bytes += (size_t)S * f.elem;
    const Schedule own_ring = ring ? *ring : make_schedule(hi - lo, nullptr, lo, chunk_steps, union_bytes);
    rc = stream_slabs(device, fields, S, own_ring, slab_jobs, stats);
  }
  for (int32_t* p : d_days)
    if (p) cudaFree(p);
  return rc;
}

// A single-operator host entry point: one job whose slabs are the ring's, on its operator's device
// and grid.  `nt` steps, or the `n_days` days of `day_start` for heat demand, in slabs of `chunk`.
static int reduce_host_one(int kind, const void* op, const AtlPlan* plan, const void* f, int64_t t0, int64_t nt,
                           const int64_t* day_start, int64_t n_days, float* out_host, int64_t chunk) {
  ATL_REQUIRE(op && plan && f, "NULL argument");
  ATL_REQUIRE(out_host, "NULL output");
  if (day_start ? n_days <= 0 : nt <= 0) return ATL_OK;
  const AtlStreamJob job{kind, op, plan, f, t0, day_start, day_start ? n_days : 0, chunk, out_host};
  std::vector<SlabField> m;
  int32_t device = 0, ny = 0, nx = 0;
  int rc = job_fields(job, m, &device, &ny, &nx);
  if (rc != ATL_OK) return rc;
  size_t bytes = 0;
  for (const SlabField& x : m)
    if (x.host) bytes += (size_t)ny * nx * x.elem;
  ATL_REQUIRE(bytes > 0, "no input fields");
  const Schedule ring = day_start ? make_schedule(n_days, day_start, 0, chunk, bytes)
                                  : make_schedule(nt, nullptr, 0, chunk, bytes);
  return reduce_host_many(device, ny, nx, day_start ? day_start[n_days] : nt, &job, 1, 0, &ring, nullptr);
}

}  // namespace atl

using namespace atl;

extern "C" {

void atl_release_host_staging(void) {
  for (auto& p : g_stage_pool) p.release();
}

int atl_device_local_cpus(int device, int32_t* cpus_out, int32_t capacity, int32_t* n_out) {
  ATL_REQUIRE(n_out, "n_out is NULL");
  *n_out = 0;
  cpu_set_t set;
  if (!device_local_cpus(device, &set)) return ATL_OK;  // unknown topology: empty list
  int32_t n = 0;
  for (int c = 0; c < CPU_SETSIZE; ++c)
    if (CPU_ISSET(c, &set)) {
      if (cpus_out && n < capacity) cpus_out[n] = c;
      ++n;
    }
  *n_out = n;
  return ATL_OK;
}

int atl_pv_reduce_host(const AtlPvOp* op, const AtlPlan* plan, const AtlPvFields* f,
                       int64_t t0, int64_t nt, float* out_host, int64_t chunk_steps) {
  return reduce_host_one(ATL_JOB_PV, op, plan, f, t0, nt, nullptr, 0, out_host, chunk_steps);
}

int atl_wind_reduce_host(const AtlWindOp* op, const AtlPlan* plan, const AtlWindFields* f,
                         int64_t nt, float* out_host, int64_t chunk_steps) {
  return reduce_host_one(ATL_JOB_WIND, op, plan, f, 0, nt, nullptr, 0, out_host, chunk_steps);
}

int atl_wind_raw_reduce_host(const AtlWindOp* op, const AtlPlan* plan, const AtlWindRawFields* f,
                             int64_t nt, float* out_host, int64_t chunk_steps) {
  return reduce_host_one(ATL_JOB_WIND_RAW, op, plan, f, 0, nt, nullptr, 0, out_host, chunk_steps);
}

int atl_csp_reduce_host(const AtlCspOp* op, const AtlPlan* plan, const AtlCspFields* f,
                        int64_t t0, int64_t nt, float* out_host, int64_t chunk_steps) {
  return reduce_host_one(ATL_JOB_CSP, op, plan, f, t0, nt, nullptr, 0, out_host, chunk_steps);
}

int atl_pointwise_reduce_host(const AtlPointwiseOp* op, const AtlPlan* plan,
                              const float* field_host, int64_t nt, float* out_host,
                              int64_t chunk_steps) {
  return reduce_host_one(ATL_JOB_POINTWISE, op, plan, field_host, 0, nt, nullptr, 0, out_host, chunk_steps);
}

int atl_heat_reduce_host(const AtlHeatOp* op, const AtlPlan* plan, const float* temperature,
                         const int64_t* day_start, int64_t n_days, float* out_host,
                         int64_t chunk_days) {
  ATL_REQUIRE(day_start, "NULL argument");
  return reduce_host_one(ATL_JOB_HEAT, op, plan, temperature, 0, 0, day_start, n_days, out_host, chunk_days);
}

int atl_reduce_host_many(int32_t device, int32_t ny, int32_t nx, int64_t nt, const AtlStreamJob* jobs,
                         int32_t n_jobs, int64_t chunk_steps, AtlStreamStats* stats) {
  return reduce_host_many(device, ny, nx, nt, jobs, n_jobs, chunk_steps, nullptr, stats);
}

}  // extern "C"
