// Shared host-side helpers of the C-ABI library (error string, launch counter).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/allrank_b200.h"

void arb_set_error(const char* msg);
// cudaFuncSetAttribute is per DEVICE: "already configured" flags are kept per device ordinal, not per process
constexpr int ARB_MAX_DEVICES = 64;
inline int arb_device_slot() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < ARB_MAX_DEVICES) ? dev : 0;
}
void arb_count_launch(int n = 1);
// Accounting only: the fraction of the nominal B * S rows that launches over packed rows actually process (set by the
// scorer when per-launch profiling is on; 1.0 otherwise).  Never steers a kernel.
double arb_row_frac();
void arb_set_row_frac(double f);
// Likewise for the fused attention kernels when they stop at the slate extents: sum_b round_up(extent_b, 16)^2 over
// B * S^2 -- the fraction of the dense S x S score work that belongs to real items (what their flops are counted as).
double arb_attn_frac();
void arb_set_attn_frac(double f);
bool arb_prof_enabled();

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------------
// The step is a chain of ~50 dependent kernels; at allRank's own batch size (64 slates) every one of them is
// latency-bound, so the gap between a kernel's last wave and its successor's first instruction matters.  Kernels
// launched through arb_launch carry cudaLaunchAttributeProgrammaticStreamSerialization (when enabled): the successor
// may start its prologue (barrier init, tensor-map prefetch, smem carve-up) while the predecessor
// drains, and blocks in arb_pdl_wait() -- griddepcontrol.wait -- until the predecessor has completed and flushed its
// memory.  Every kernel launched this way executes arb_pdl_wait() on every thread before its first access to global
// memory; without the launch attribute the instruction is a no-op.
bool arb_pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void arb_pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
template <typename... KArgs, typename... Args>
inline cudaError_t arb_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = arb_pdl_enabled() ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#endif

// ---- deterministic reductions -------------------------------------------------------------------------------------
// Gradient reductions across blocks do not use floating-point atomics (their order, and so their rounding, changes from
// run to run; Adam turns the rounding noise of a mathematically zero gradient into full-size steps).  Instead every
// block stores its partial result in a slot of its own and dst += sum of the slots in a fixed order afterwards:
//   DetParts dp;  dp.add(grad, n_slots, rows, cols, ld);  ...;  dp.begin(st);   // grad now points at the zeroed slots
//   <launch: slot s writes grad[s * rows * cols + r * cols + c]>;  dp.finish(st);
// The slots are a stream-ordered allocation of this call (cudaMallocAsync / cudaFreeAsync on `st`): calls on different
// streams or host threads never share them, nothing is synchronised, and under stream capture they become memory
// nodes owned by the graph.
struct DetParts {
  struct Reg { float** var; float* dst; long long n, rows, cols, ld; };
  Reg reg[6];
  int k = 0;
  float* base = nullptr;         // the allocation: slots, then two buffers for the intermediate levels of the sum
  float* tmp[2] = {nullptr, nullptr};
  cudaStream_t stream = nullptr;
  // registers the pointer variable `p` (ignored when null) for n slots of a rows x cols block (dst row pitch ld)
  void add(float*& p, long long n, long long rows, long long cols, long long ld) {
    if (p) reg[k++] = Reg{&p, p, n, rows, cols, ld};
  }
  int begin(cudaStream_t st);    // 0 or ARB_E_*: slots allocated and zeroed, registered pointers redirected to them
  int finish(cudaStream_t st);   // 0 or ARB_E_*: dst += slot sums, slots released
  void release();
  ~DetParts() { release(); }
};

// loss = sum(val)/sum(cnt), grad *= 1/sum(cnt); an all-zero count gives loss 0 and zero grad (slate_kernels.cu)
int arb_finalize_mean_over_count(const float* val, const float* cnt, int B, float* loss, float* grad, size_t n_grad,
                                 cudaStream_t st);

// Optional per-launch device timing (bench.py roofline): when enabled, every launch made inside a ProfScope is
// bracketed by CUDA events on its own stream; arb_prof_collect sums durations and work units per kernel class.
enum { ARB_PROF_GEMM = 0, ARB_PROF_SCORER_SIMT = 1, ARB_PROF_LOSS = 2, ARB_PROF_METRICS = 3, ARB_PROF_OPTIM = 4,
       ARB_PROF_SLATES = 5, ARB_PROF_CLASSES = 6 };
struct ProfScope {
  // `name` defaults to the launching host function; GEMM launches pass a shape-derived name so that the per-kernel
  // table of bench.py tells the QKV projection from the first FFN linear (arb_prof_report)
  ProfScope(int cls, double work, cudaStream_t st, double bytes = 0.0, const char* name = __builtin_FUNCTION());
  ~ProfScope();
  int idx;
  cudaStream_t st;
};
