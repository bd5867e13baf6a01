// sb_gemm_decode: the decoder-step products at <= 256 rows (one beam-search step: 160 rows) in "transposed" form.
//
// At 160 rows the general kernel (gemm_tcgen05.cu: rows = MMA M, 64 output features per CTA) is bound by L2 -> SM traffic, not
// by HBM: every CTA re-reads its 128-row activation tile for each of its few weight rows.  Here a 128-FEATURE weight tile is
// the wgmma A operand (two consumer warpgroups, 64 features each) and ALL rows are the B operand (N = rows padded to a
// power of two >= 32, or to 160 for a beam-search step of 32 x 5 rows; fp32 accumulators in registers): a CTA reads its
// weight tile once and the activations once per k-block.  One (tile, K-slice) unit per CTA, a TMA ring, one producer warp.
//   split-K mode : slice z writes raw fp32 partial products to partials[(z * slice_rows + row) * n + feature]
//                  (same contract as sb_gemm_splitk / sb_gemm_skinny; reduced by sb_splitk_reduce_ln or the attention kernels)
//   direct mode  : out[row * out_ld + feature] = act(acc + bias) in fp16, act in {none, relu}
// Replaces Linear_forward (fairseq2.cpp:251) at all six decoder-step products of StandardTransformerDecoderLayer_forward
// (fairseq2.cpp:979-1094): self-attention q|k|v and output, cross-attention q and output, FFN inner and output.
//
// Bytes per call at a beam-search step of 160 rows (seamlessM4T_large; the engine passes the row-major chain's splits):
//   product              n x k        tiles x splits   weights (HBM)  activations (L2 -> SM)  fp32 partials written
//   self-attn q|k|v   3072 x 1024        24 x 2   =  48     6.3 MB          7.9 MB                3.9 MB
//   attn out / cross q 1024 x 1024        8 x 8   =  64     2.1 MB          2.6 MB                5.2 MB
//     / cross out
//   FFN inner         8192 x 1024        64 x 1   =  64    16.8 MB         21.0 MB                -  (fp16 out 2.6 MB)
//   FFN out           1024 x 8192         8 x 8   =  64    16.8 MB         21.0 MB                5.2 MB
// A slice sums its k-blocks in order with the same m64 x k16 tensor-core steps as the row-major kernel and the mma.sync
// skinny kernel, so at the same contiguous K slices the partials are bit-identical to theirs (tests/test_decode_gemm.py):
// the search does not depend on which path runs.  More slices would fill more SMs but change the fp32 sums, and measured
// no faster at 160 rows on an H100: q|k|v 8.5 us at 4 slices against 8.8 at 2; FFN out 12.3 us at 16 against 11.9 at 8.
// Activations: tiles x rows x k x 2 B (each (tile, slice) unit reads its K slice of all rows once), so L2 -> SM traffic is
// weights + activations = 2.25x the weight bytes for every product.  FFN inner keeps its fused bias + ReLU at 64 CTAs:
// 64-feature tiles would give 128 CTAs but read the activations twice (42 MB, 3.5x the weights), and splitting K over
// a 2-CTA cluster that adds the halves through distributed shared memory kept the bytes but measured slower on an H100
// (13.5 us per call against 11.8 us for the same kernel at one slice per tile).
// Residency: one CTA per SM.  At N = 160 the 80 fp32 accumulators per consumer thread take the kernel to 106 registers
// (no spills); two CTAs of 9 warps per SM would have to fit in 96 per thread, which ptxas refuses for the N = 160 MMA.
// So the ring takes the SM's shared memory, up to the K slice: a CTA streams at ~77 GB/s with 3 stages (108 KB) in
// flight and ~92 GB/s with 6 (measured on an H100 SXM, 700 W), and the next kernel's weights are pulled into L2
// instead of being loaded by a co-resident CTA (DgArgs::prefetch).
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace sb {
namespace {

constexpr int DG_BK = 64;
constexpr int DG_TM = 128;
constexpr int DG_W_BYTES = DG_TM * DG_BK * 2;
constexpr int DG_THREADS = 288;  // warps 0-7 two consumer warpgroups (MMA + epilogue), warp 8 TMA producer
constexpr int DG_MAX_STAGES = 8;
constexpr int DG_SMEM_MISC = 1024 + 512;  // alignment slack + barriers
constexpr int DG_SP = DG_TM + 4;          // row pitch (floats) of the epilogue's staging tile

struct DgArgs {
  int rows, npad, n_out, kb_total, splits, stages;
  int relu;
  const float* bias;
  float* partials;
  long long slice_rows;
  elem_t* out;
  long long out_ld;
  const char* prefetch;  // the next kernel's weights: pulled into L2 by the producer warp once its loads are issued
  long long prefetch_bytes;
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // warps 0-7
// NT: wgmma N (>= npad).  The activation slot of a stage holds NT rows; TMA fills the first npad (zero past `rows`), the
// MMA columns beyond them are never stored.
template <int NT>
__global__ void __launch_bounds__(DG_THREADS, 1)
decode_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const DgArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int stage_bytes = DG_W_BYTES + NT * DG_BK * 2;
  uint8_t* misc = smem + (size_t)g.stages * stage_bytes;
  uint64_t* full = (uint64_t*)misc;
  uint64_t* empty = full + DG_MAX_STAGES;

  const int u = blockIdx.x;
  const int tile = u / g.splits, split = u - tile * g.splits;
  const int kb0 = (g.kb_total * split) / g.splits, kb1 = (g.kb_total * (split + 1)) / g.splits;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmX)) : "memory");
    for (int s = 0; s < g.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int wg = warp >> 2;
  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  if (warp == 8) {
    // ---- TMA producer: weights first (they do not depend on the upstream kernel: under PDL they stream while it still runs)
    int s = 0;
    uint32_t ph = 0;
    bool waited = false;
    const uint32_t tx = (uint32_t)(DG_W_BYTES + g.npad * DG_BK * 2);
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&empty[s], ph ^ 1);
      uint8_t* st = smem + (size_t)s * stage_bytes;
      if (elect_one()) {
        mbar_expect_tx(&full[s], tx);
        tma_load_2d(st, &tmW, &full[s], kb * DG_BK, tile * DG_TM);
        if (!waited) pdl_wait();
        tma_load_2d(st + DG_W_BYTES, &tmX, &full[s], kb * DG_BK, 0);
      }
      waited = true;
      __syncwarp();
      if (++s == g.stages) { s = 0; ph ^= 1; }
    }
    if (g.prefetch_bytes > 0) {
      constexpr long long CH = 16384;
      const long long share = ((g.prefetch_bytes + gridDim.x - 1) / gridDim.x + 4095) / 4096 * 4096;
      const long long lo = (long long)blockIdx.x * share, hi = min(lo + share, g.prefetch_bytes);
      if (elect_one())
        for (long long o = lo; o < hi; o += CH)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(g.prefetch + o), "r"((uint32_t)min(CH, hi - o)) : "memory");
      __syncwarp();
    }
  } else {
    // ---- consumers: D[feature][row] += W[64 features of warpgroup wg][64] . X[NT rows][64]^T
    int s = 0, prev = 0;
    uint32_t ph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
      const uint64_t da = make_smem_desc(sa + wg * 64 * 128), db = make_smem_desc(sa + DG_W_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < DG_BK / 16; ++k) Wgmma<NT>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
      wg_commit();
      wg_wait<1>();
      wg_fence_regs(acc);
      if (kb > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == g.stages) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
  }
  if (warp == 8) return;
  // both warpgroups are past their last MMA (the other one may still read the last stage): from here the ring is scratch
  consumer_bar();
  // ---- epilogue: register j*4 + 2h + e of the accumulator fragment = (feature fl + 8h, row j*8 + 2*(lane%4) + e).  It
  // goes through shared memory as [row][128 features] (pitch DG_SP floats: the fragment writes hit 32 distinct banks)
  // and leaves as whole rows in 16-byte stores, instead of 4-row x 32-byte scatters
  float* stage = reinterpret_cast<float*>(smem);
  const int fl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < NT / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) stage[(j * 8 + (lane & 3) * 2 + e) * DG_SP + fl + 8 * h] = acc[j * 4 + 2 * h + e];
  consumer_bar();
  pdl_sync();
  const int f_tile = tile * DG_TM;
  const int tid = threadIdx.x;
  if (g.partials != nullptr) {
    // 32 chunks of 4 features per row: one warp writes one 512-byte row segment
    const bool vec = (g.n_out & 3) == 0;
    for (int i = tid; i < g.rows * 32; i += 256) {
      const int r = i >> 5, c = (i & 31) * 4, f = f_tile + c;
      if (f >= g.n_out) continue;
      const float4 v = *reinterpret_cast<const float4*>(stage + r * DG_SP + c);
      float* dst = g.partials + ((long long)split * g.slice_rows + r) * g.n_out + f;
      if (vec && f + 4 <= g.n_out) {
        *reinterpret_cast<float4*>(dst) = v;
      } else {
        const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (f + q < g.n_out) dst[q] = x[q];
      }
    }
  } else {
    // 16 chunks of 8 features per row, bias + activation, fp16
    const bool vec = (g.out_ld & 7) == 0 && ((uintptr_t)g.out & 15) == 0;
    for (int i = tid; i < g.rows * 16; i += 256) {
      const int r = i >> 4, c = (i & 15) * 8, f = f_tile + c;
      if (f >= g.n_out) continue;
      const float4 lo = *reinterpret_cast<const float4*>(stage + r * DG_SP + c);
      const float4 hi = *reinterpret_cast<const float4*>(stage + r * DG_SP + c + 4);
      float x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      const int nq = min(8, g.n_out - f);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        x[q] += (g.bias != nullptr && q < nq) ? g.bias[f + q] : 0.f;
        if (g.relu) x[q] = fmaxf(x[q], 0.f);
      }
      elem_t* dst = g.out + (long long)r * g.out_ld + f;
      if (vec && nq == 8) {
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) hv[q] = __floats2half2_rn(x[2 * q], x[2 * q + 1]);
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hv);
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (q < nq) dst[q] = __float2half_rn(x[q]);
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int dg_map(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint64_t ld_elems, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  SB_REQUIRE(fn != nullptr, SB_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {(cuuint32_t)DG_BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_REQUIRE(r == CUDA_SUCCESS, SB_ECUDA, "sb_gemm_decode: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return SB_OK;
}

bool dg_supported(const sb_gemm_t* g, int splits) {
  return g != nullptr && g->taps == 1 && g->m >= 1 && g->m <= 256 && g->c_in % DG_BK == 0 && g->a_row0 == 0 && !g->glu && splits >= 1 &&
         splits <= g->c_in / DG_BK && (g->a_ld % 8) == 0 && ((uintptr_t)g->a % 16) == 0 && ((uintptr_t)g->w % 16) == 0 &&
         g->res1 == nullptr && g->res2 == nullptr && g->out2 == nullptr && g->seq_rows == 0;
}

template <int NT>
int dg_launch(const CUtensorMap& tmW, const CUtensorMap& tmX, const DgArgs& a, int grid, size_t smem, cudaStream_t st) {
  static size_t configured = 0;
  if (smem > configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(decode_gemm_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  SB_CUDA_OK(launch_k(decode_gemm_kernel<NT>, dim3(grid), dim3(DG_THREADS), smem, st, tmW, tmX, a));
  count_launch();
  return SB_OK;
}

}  // namespace
}  // namespace sb

extern "C" int sb_gemm_decode_supported(const sb_gemm_t* g, int32_t splits) { return sb::dg_supported(g, splits) ? 1 : 0; }

extern "C" int sb_gemm_decode(const sb_gemm_t* g, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(dg_supported(g, splits), SB_ENOSUP, "sb_gemm_decode: shape not supported (rows <= 256, taps 1, c_in %% 64 == 0, no GLU / residual)");
  SB_REQUIRE(partials != nullptr || (splits == 1 && g->out != nullptr && !g->out_f32 && (g->act == SB_ACT_NONE || g->act == SB_ACT_RELU)),
             SB_EINVAL, "sb_gemm_decode: direct mode needs splits == 1, an fp16 output and act in {none, relu}");
  SB_REQUIRE(partials == nullptr || slice_rows >= g->m, SB_EINVAL, "sb_gemm_decode: slice_rows (%lld) < m (%d)", (long long)slice_rows, g->m);
  DgArgs a;
  a.rows = g->m;
  a.npad = (g->m + 15) / 16 * 16;
  a.n_out = g->n;
  a.kb_total = g->c_in / DG_BK;
  const int tiles = (g->n + DG_TM - 1) / DG_TM;
  a.splits = splits;
  a.relu = g->act == SB_ACT_RELU;
  a.bias = g->bias;
  a.partials = partials;
  a.slice_rows = slice_rows;
  a.out = (elem_t*)g->out;
  a.out_ld = g->out_ld;
  a.prefetch = (const char*)g->prefetch;
  a.prefetch_bytes = g->prefetch ? g->prefetch_bytes / 4096 * 4096 : 0;
  const int nt = a.npad <= 32 ? 32 : a.npad <= 64 ? 64 : a.npad <= 128 ? 128 : a.npad <= 160 ? 160 : 256;
  const int stage_bytes = DG_W_BYTES + nt * DG_BK * 2;
  // ring: as deep as shared memory allows, up to the K slice, and large enough for the epilogue's staging tile
  int dev = 0, smem_optin = 0;
  SB_CUDA_OK(cudaGetDevice(&dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int kb_max = (a.kb_total + a.splits - 1) / a.splits;
  int stages = (smem_optin - DG_SMEM_MISC) / stage_bytes;
  if (stages > DG_MAX_STAGES) stages = DG_MAX_STAGES;
  if (stages > kb_max) stages = kb_max;
  const int epi_bytes = nt * DG_SP * 4;
  if (stages * stage_bytes < epi_bytes) stages = (epi_bytes + stage_bytes - 1) / stage_bytes;
  if (stages < 2) stages = 2;
  a.stages = stages;
  const size_t smem = (size_t)stages * stage_bytes + DG_SMEM_MISC;
  CUtensorMap tmW, tmX;
  int rc = dg_map(&tmW, g->w, (uint64_t)g->c_in, (uint64_t)g->n, (uint64_t)g->c_in, DG_TM);
  if (rc) return rc;
  rc = dg_map(&tmX, g->a, (uint64_t)g->c_in, (uint64_t)g->m, (uint64_t)g->a_ld, (uint32_t)a.npad);
  if (rc) return rc;
  const int grid = tiles * a.splits;
  cudaStream_t st = (cudaStream_t)stream;
  if (nt == 32) return dg_launch<32>(tmW, tmX, a, grid, smem, st);
  if (nt == 64) return dg_launch<64>(tmW, tmX, a, grid, smem, st);
  if (nt == 128) return dg_launch<128>(tmW, tmX, a, grid, smem, st);
  if (nt == 160) return dg_launch<160>(tmW, tmX, a, grid, smem, st);
  return dg_launch<256>(tmW, tmX, a, grid, smem, st);
}
