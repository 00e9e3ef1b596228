// C-ABI bookkeeping: thread-local error string, ABI version, launch counter.
#include <atomic>
#include <cstring>

#include "common.h"
#include "defaults.h"

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void arb_set_error(const char* msg) {
  std::strncpy(g_err, msg ? msg : "", sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}
void arb_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" const char* arb_last_error(void) { return g_err; }
extern "C" int32_t arb_abi_version(void) { return 4; }
extern "C" int64_t arb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

// programmatic dependent launch: on by default; arb_set_pdl(0) / ARB_PDL=0 launches every kernel fully serialised
static std::atomic<int> g_pdl{ARB_DEFAULT_PDL};
bool arb_pdl_enabled() { return g_pdl.load(std::memory_order_relaxed) != 0; }
extern "C" void arb_set_pdl(int32_t on) { g_pdl.store(on ? 1 : 0, std::memory_order_relaxed); }

// ---------------------------------------------------------------- per-launch timing
#include <mutex>
#include <vector>
namespace {
struct ProfRec { int cls; double work; double bytes; cudaEvent_t e0, e1; char name[56]; };
std::vector<ProfRec> g_recs;
std::mutex g_prof_mu;
bool g_prof_on = false;
constexpr size_t kMaxRecs = 1 << 16;
double g_row_frac = 1.0;
double g_attn_frac = 1.0;
}  // namespace

double arb_row_frac() { return g_row_frac; }
void arb_set_row_frac(double f) { g_row_frac = f; }
double arb_attn_frac() { return g_attn_frac; }
void arb_set_attn_frac(double f) { g_attn_frac = f; }
bool arb_prof_enabled() { return g_prof_on; }

ProfScope::ProfScope(int cls, double work, cudaStream_t s, double bytes, const char* name) : idx(-1), st(s) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_recs.size() >= kMaxRecs) return;
  ProfRec r{cls, work, bytes, nullptr, nullptr, {0}};
  std::strncpy(r.name, name ? name : "?", sizeof(r.name) - 1);
  if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
  cudaEventRecord(r.e0, st);
  g_recs.push_back(r);
  idx = int(g_recs.size()) - 1;
}
ProfScope::~ProfScope() {
  if (idx < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_recs[idx].e1, st);
}

extern "C" void arb_prof_enable(int32_t on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto& r : g_recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  g_recs.clear();
  g_prof_on = on != 0;
}
// Sums device time (ms), work units and launch count of one kernel class since arb_prof_enable(1).
static double g_last_bytes[ARB_PROF_CLASSES] = {0};
extern "C" double arb_prof_last_bytes(int32_t cls) { return (cls >= 0 && cls < ARB_PROF_CLASSES) ? g_last_bytes[cls] : 0.0; }

extern "C" int32_t arb_prof_collect(int32_t cls, double* total_ms, double* total_work, int64_t* launches) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double ms = 0, work = 0, bytes = 0;
  long long n = 0;
  for (auto& r : g_recs) {
    if (r.cls != cls) continue;
    if (cudaEventSynchronize(r.e1) != cudaSuccess) { arb_set_error("arb_prof_collect: event sync failed"); return ARB_E_CUDA; }
    float t = 0;
    cudaEventElapsedTime(&t, r.e0, r.e1);
    ms += t; work += r.work; bytes += r.bytes; ++n;
  }
  if (cls >= 0 && cls < ARB_PROF_CLASSES) g_last_bytes[cls] = bytes;
  if (total_ms) *total_ms = ms;
  if (total_work) *total_work = work;
  if (launches) *launches = n;
  return ARB_OK;
}

// Per-kernel table since arb_prof_enable(1): one line per distinct launch name,
//   name<TAB>class<TAB>launches<TAB>total_ms<TAB>total_work<TAB>total_bytes
// (work = flops for class 0, algorithmic bytes otherwise; bytes = algorithmic HBM bytes where the launcher states
// them).  Returns the number of bytes written (truncated to cap - 1), or ARB_E_CUDA.
#include <cstdio>
#include <map>
#include <string>
extern "C" int64_t arb_prof_report(char* buf, int64_t cap) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  struct Agg { int cls; long long n; double ms, work, bytes; };
  std::map<std::string, Agg> table;
  std::vector<std::string> order;
  for (auto& r : g_recs) {
    if (cudaEventSynchronize(r.e1) != cudaSuccess) { arb_set_error("arb_prof_report: event sync failed"); return ARB_E_CUDA; }
    float t = 0;
    cudaEventElapsedTime(&t, r.e0, r.e1);
    auto it = table.find(r.name);
    if (it == table.end()) { it = table.emplace(r.name, Agg{r.cls, 0, 0, 0, 0}).first; order.push_back(r.name); }
    it->second.n += 1; it->second.ms += t; it->second.work += r.work; it->second.bytes += r.bytes;
  }
  std::string out;
  char line[256];
  for (auto& k : order) {
    const Agg& a = table[k];
    std::snprintf(line, sizeof line, "%s\t%d\t%lld\t%.6f\t%.6e\t%.6e\n", k.c_str(), a.cls, a.n, a.ms, a.work, a.bytes);
    out += line;
  }
  if (!buf || cap <= 0) return int64_t(out.size());
  const int64_t n = std::min<int64_t>(cap - 1, int64_t(out.size()));
  std::memcpy(buf, out.data(), size_t(n));
  buf[n] = 0;
  return n;
}

// ------------------------------------------------------------------------------------------------ deterministic reductions
// Two-level ordered sum over the slots: slot group g = slots 64 g .. 64 g + 63; warp w of a block sums slots
// 64 g + w, + 8, ... in ascending order, the 8 warp sums are combined in warp order.  One block per (32 elements, group):
//   n_groups > 1: out[g * elems + e] = group sum   (the next level sums the groups the same way)
//   n_groups = 1: dst[r * ld + c] += group sum
// The grouping is fixed by the slot count, so the result does not depend on the grid or on the order blocks run in.
constexpr long long DET_GROUP = 64;
__global__ void __launch_bounds__(256) det_reduce_kernel(const float* __restrict__ part, long long n, long long rows,
                                                         long long cols, long long ld, float* __restrict__ out) {
  arb_pdl_wait();
  __shared__ float sh[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long e = (long long)blockIdx.x * 32 + lane, elems = rows * cols;
  const long long s0 = (long long)blockIdx.y * DET_GROUP, s1 = min(n, s0 + DET_GROUP);
  float t = 0.f;
  if (e < elems)
    for (long long s = s0 + w; s < s1; s += 8) t += part[s * elems + e];
  sh[w][lane] = t;
  __syncthreads();
  if (w == 0 && e < elems) {
    float v = sh[0][lane];
#pragma unroll
    for (int g = 1; g < 8; ++g) v += sh[g][lane];
    if (gridDim.y > 1) {
      out[(long long)blockIdx.y * elems + e] = v;
    } else {
      const long long r = e / cols, c = e - r * cols;
      out[r * ld + c] += v;
    }
  }
}

static long long det_groups(long long n) { return (n + DET_GROUP - 1) / DET_GROUP; }

int DetParts::begin(cudaStream_t st) {
  if (k == 0) return ARB_OK;
  stream = st;
  // slots of every registered array, then two buffers for the intermediate levels of the largest one
  size_t slots = 0, lvl1 = 0, lvl2 = 0;
  for (int i = 0; i < k; ++i) {
    const long long elems = reg[i].rows * reg[i].cols;
    slots += size_t(reg[i].n * elems);
    lvl1 = std::max(lvl1, size_t(det_groups(reg[i].n) * elems));
    lvl2 = std::max(lvl2, size_t(det_groups(det_groups(reg[i].n)) * elems));
  }
  static bool pool_set[ARB_MAX_DEVICES] = {};
  const int dev = arb_device_slot();
  if (!pool_set[dev]) {
    // the slots come from the device's stream-ordered pool: keep what it has reserved across synchronisations instead
    // of returning it to the driver after every step (bounded; nothing stays allocated between calls)
    int id = 0;
    cudaGetDevice(&id);
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, id) == cudaSuccess) {
      uint64_t keep = uint64_t(512) << 20;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool_set[dev] = true;
  }
  const size_t total = slots + lvl1 + lvl2;
  void* p = nullptr;
  if (cudaMallocAsync(&p, total * sizeof(float), st) != cudaSuccess) {
    cudaGetLastError();
    arb_set_error("reduction slots: cudaMallocAsync failed");
    return ARB_E_CUDA;
  }
  base = static_cast<float*>(p);
  if (cudaMemsetAsync(base, 0, slots * sizeof(float), st) != cudaSuccess) {
    arb_set_error("reduction slots: memset failed");
    return ARB_E_CUDA;
  }
  float* q = base;
  for (int i = 0; i < k; ++i) {
    *reg[i].var = q;
    q += reg[i].n * reg[i].rows * reg[i].cols;
  }
  tmp[0] = q;
  tmp[1] = q + lvl1;
  return ARB_OK;
}

int DetParts::finish(cudaStream_t st) {
  for (int i = 0; i < k; ++i) {
    const long long elems = reg[i].rows * reg[i].cols;
    const float* src = *reg[i].var;
    long long n = reg[i].n;
    for (int level = 0;; ++level) {
      const long long groups = det_groups(n);
      float* out = groups > 1 ? tmp[level & 1] : reg[i].dst;
      ProfScope ps(ARB_PROF_SCORER_SIMT, 4.0 * double(n) * double(elems), st, 0.0, "det_reduce_kernel");
      arb_launch(det_reduce_kernel, dim3(unsigned((elems + 31) / 32), unsigned(groups)), dim3(256), 0, st, src, n,
                 reg[i].rows, reg[i].cols, reg[i].ld, out);
      arb_count_launch();
      if (groups == 1) break;
      src = out;
      n = groups;
    }
    *reg[i].var = reg[i].dst;
  }
  release();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { arb_set_error(cudaGetErrorString(e)); return ARB_E_CUDA; }
  return ARB_OK;
}

void DetParts::release() {
  if (base) cudaFreeAsync(base, stream);     // stream-ordered: after every launch above has read the slots
  base = nullptr;
}
