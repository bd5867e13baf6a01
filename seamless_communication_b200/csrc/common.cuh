// Shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <utility>

#include "../../include/seamless_b200.h"

namespace sb {

typedef __half elem_t;  // storage / tensor-core input type of the whole path (the reference runs fp16 on CUDA,
                        // cli/m4t/predict/predict.py:207-212)

void set_error(const char* fmt, ...);
extern long long g_launch_count;
inline void count_launch(int n = 1) { __atomic_fetch_add(&g_launch_count, (long long)n, __ATOMIC_RELAXED); }  // several host threads launch

#define SB_REQUIRE(cond, code, ...)      \
  do {                                   \
    if (!(cond)) {                       \
      sb::set_error(__VA_ARGS__);        \
      return (code);                     \
    }                                    \
  } while (0)

#define SB_CUDA_OK(expr)                                                                 \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      sb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SB_ECUDA;                                                                   \
    }                                                                                    \
  } while (0)

#define SB_LAUNCH_OK()                                                                   \
  do {                                                                                   \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      sb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SB_ECUDA;                                                                   \
    }                                                                                    \
    sb::count_launch();                                                                  \
  } while (0)

// Programmatic dependent launch (PDL, on by default; SB_PDL=0 turns it off): every kernel waits for its prerequisites
// right before it first touches data produced upstream and only THEN lets its own dependents launch, so launch latency,
// prologues (barrier init, descriptor fetch) and - in the GEMMs - the weight loads of kernel N+1 overlap with
// kernel N, while at most one generation of dependents is resident.  (Triggering at kernel entry instead would let the
// whole chain launch ahead, with every waiting kernel pinning shared memory.)
// The rule every kernel launched through launch_k keeps: each CTA runs pdl_wait (griddepcontrol.wait) before
//   (a) it reads anything an earlier kernel wrote,
//   (b) it writes global memory that an earlier kernel reads or writes, and
//   (c) it exits.
// Before the wait a CTA may only touch what no kernel of the stream writes (weights, biases, tensor maps) and its own
// shared memory.  (c) keeps the chain transitive: the wait covers only the immediate predecessor, so a CTA that exited
// early would let its grid complete - and its dependent pass the wait - while the kernel before it still runs.  Threads of
// a CTA that exit without waiting (a producer lane, an idle warp) are fine as long as another thread of the CTA waits.
// Both instructions are no-ops when the kernel was launched without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_wait(); pdl_trigger(); }

bool pdl_enabled();
int sm_count();  // SMs of the current device (cached per device)
// 2D fp16 (esize 2) / fp32 (esize 4) tensor map: inner = channels, box 128 B x box_rows, 128B swizzle, OOB -> 0 (gemm_tcgen05.cu);
// esize 1 (e4m3 bytes): box 64 B x box_rows, no swizzle
int make_tmap(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint64_t ld_elems, uint32_t box_rows,
              int esize = 2);
// sb_gemm with tile_stats at <= 256 rows on the weight-stationary projection kernel (decode_gemm.cu).  Returns false,
// launching nothing, when the shape does not qualify; else true with the launch's status in *rc.
bool vocab_proj(const sb_gemm_t* g, cudaStream_t st, int* rc);

// The beam-search step's small kernels (embedding, LayerNorms, attention, top-K, bookkeeping) ask for the largest shared
// memory carveout of the SM's unified L1 / shared memory.  Under PDL the weight product that follows one of them
// launches while it runs, and its CTAs (110-221 KB of shared memory) can only start on an SM whose carveout already
// holds them; at the small default carveout such kernels leave, they wait for the SM to drain.  Measured on an H100 SXM
// at 700 W: one search step 2.19 ms against 2.25 ms with PDL alone.  Without PDL nothing overlaps and the hint is not set.
template <typename... KArgs>
inline cudaError_t prefer_shared(void (*kernel)(KArgs...)) {
  if (!pdl_enabled()) return cudaSuccess;
  return cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// exact GELU (torch.nn.functional.gelu, approximate='none')
__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  switch (act) {
    case SB_ACT_RELU: return fmaxf(v, 0.f);
    case SB_ACT_SILU: return v / (1.f + __expf(-v));
    case SB_ACT_LRELU: return v > 0.f ? v : v * slope;
    case SB_ACT_TANH: return tanhf(v);
    case SB_ACT_GELU: return gelu_erf(v);
    default: return v;
  }
}

// sequence layout helper: is padded-row q a valid data row?  (q = b*Tp + PH + t, 0 <= t < len[b])
__device__ __forceinline__ bool seq_row_valid(long long q, int Tp, int PH, int T, const int* lens) {
  if (Tp <= 0) return true;
  int b = (int)(q / Tp);
  int pos = (int)(q - (long long)b * Tp) - PH;
  int len = lens ? lens[b] : T;
  return pos >= 0 && pos < len;
}

}  // namespace sb
