// sb_dwconv_ln_silu: Conformer convolution module core for w2v-BERT 2.0 (conformer_shaw/builder.py:148-156):
//   causal depthwise Conv1d(kernel k, left pad k-1, no bias) -> LayerNorm(C) -> SiLU,   x,y: (B,T,C) fp16.
// sb_dwconv_bias_silu: the same core for w2v-BERT v1 (ConvModule_forward, ggml/examples/unity/fairseq2.cpp:698-731):
//   depthwise Conv1d(k = 31, pad 15 on both sides) -> BatchNorm (eval statistics) -> SiLU, with the BatchNorm scale folded
//   into the depthwise weights by the host, so that only a per-channel bias remains.
// (the pointwise convs and the GLU live in the sb_gemm epilogues around it.)
// One CTA = TT output frames x all C channels.  The (TT+k-1) x C input window is staged once in shared memory
// (each input element is reused k times from smem instead of HBM/L2), conv results stay in smem as fp32 for the
// LayerNorm, so HBM traffic is the algorithmic minimum: read x once (+ halo), write y once.
#include "common.cuh"

namespace sb {

constexpr int DW_TT = 8;
constexpr int DW_THREADS = 256;

__global__ void __launch_bounds__(DW_THREADS) dwconv_ln_silu_kernel(const elem_t* __restrict__ x, elem_t* __restrict__ y,
                                                                    const elem_t* __restrict__ w, const float* __restrict__ ln_w,
                                                                    const float* __restrict__ ln_b, int T, int C, int k) {
  extern __shared__ __align__(16) uint8_t smem_dw[];
  const int rows_in = DW_TT + k - 1;
  elem_t* sx = reinterpret_cast<elem_t*>(smem_dw);                 // [rows_in][C]
  elem_t* sw = sx + (size_t)rows_in * C;                           // [k][C]  (transposed weights)
  float* so = reinterpret_cast<float*>(sw + (size_t)k * C);        // [DW_TT][C]
  const int b = blockIdx.y, t0 = blockIdx.x * DW_TT;
  const elem_t* xb = x + (long long)b * T * C;
  // stage input rows t0-(k-1) .. t0+TT-1 (zeros before the sequence start / after its end)
  const int vec_per_row = C / 8;
  for (int i = threadIdx.x; i < rows_in * vec_per_row; i += DW_THREADS) {
    int r = i / vec_per_row, c = (i - r * vec_per_row) * 8;
    int t = t0 - (k - 1) + r;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (t >= 0 && t < T) u = *reinterpret_cast<const uint4*>(xb + (long long)t * C + c);
    *reinterpret_cast<uint4*>(sx + (size_t)r * C + c) = u;
  }
  for (int i = threadIdx.x; i < C * k; i += DW_THREADS) {  // w is [C][k] (Conv1d weight (C,1,k))
    int c = i / k, j = i - c * k;
    sw[(size_t)j * C + c] = w[i];
  }
  __syncthreads();
  // depthwise conv: each thread owns channel pairs
  for (int c = threadIdx.x * 2; c < C; c += DW_THREADS * 2) {
    float acc[DW_TT][2];
#pragma unroll
    for (int t = 0; t < DW_TT; ++t) acc[t][0] = acc[t][1] = 0.f;
    for (int j = 0; j < k; ++j) {
      float2 wv = __half22float2(*reinterpret_cast<const __half2*>(sw + (size_t)j * C + c));
#pragma unroll
      for (int t = 0; t < DW_TT; ++t) {
        float2 xv = __half22float2(*reinterpret_cast<const __half2*>(sx + (size_t)(t + j) * C + c));
        acc[t][0] += wv.x * xv.x;
        acc[t][1] += wv.y * xv.y;
      }
    }
#pragma unroll
    for (int t = 0; t < DW_TT; ++t) *reinterpret_cast<float2*>(so + (size_t)t * C + c) = make_float2(acc[t][0], acc[t][1]);
  }
  __syncthreads();
  // LayerNorm + SiLU: one warp per output frame
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = warp; t < DW_TT; t += DW_THREADS / 32) {
    if (t0 + t >= T) continue;
    const float* row = so + (size_t)t * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += row[c];
    const float mean = warp_sum(s) / C;
    float sq = 0.f;
    for (int c = lane; c < C; c += 32) {
      float d = row[c] - mean;
      sq += d * d;
    }
    const float rstd = rsqrtf(warp_sum(sq) / C + 1e-5f);
    elem_t* yp = y + ((long long)b * T + t0 + t) * C;
    for (int c = lane * 2; c < C; c += 64) {
      float a0 = (row[c] - mean) * rstd * ln_w[c] + ln_b[c];
      float a1 = (row[c + 1] - mean) * rstd * ln_w[c + 1] + ln_b[c + 1];
      a0 = a0 / (1.f + __expf(-a0));
      a1 = a1 / (1.f + __expf(-a1));
      *reinterpret_cast<__half2*>(yp + c) = __floats2half2_rn(a0, a1);
    }
  }
}

// Fast path for a compile-time kernel size (w2v-BERT 2.0: k = 31).  Same tiling, but the per-channel taps live in
// registers (read straight from the (C, k) weight, no transposed smem copy whose column stores were 31-way bank
// conflicted) and the TT + K - 1 inputs of a channel pair are loaded from smem once and reused from registers by all
// TT outputs: 2 shared loads per 16 FMAs instead of 9.
template <int K>
__global__ void __launch_bounds__(DW_THREADS) dwconv_ln_silu_fixed_kernel(const elem_t* __restrict__ x, elem_t* __restrict__ y,
                                                                          const elem_t* __restrict__ w,
                                                                          const float* __restrict__ ln_w,
                                                                          const float* __restrict__ ln_b, int T, int C) {
  extern __shared__ __align__(16) uint8_t smem_dw[];
  constexpr int ROWS_IN = DW_TT + K - 1;
  elem_t* sx = reinterpret_cast<elem_t*>(smem_dw);                  // [ROWS_IN][C]
  float* so = reinterpret_cast<float*>(sx + (size_t)ROWS_IN * C);   // [DW_TT][C]
  const int b = blockIdx.y, t0 = blockIdx.x * DW_TT;
  const elem_t* xb = x + (long long)b * T * C;
  const int vec_per_row = C / 8;
  for (int i = threadIdx.x; i < ROWS_IN * vec_per_row; i += DW_THREADS) {
    int r = i / vec_per_row, c = (i - r * vec_per_row) * 8;
    int t = t0 - (K - 1) + r;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (t >= 0 && t < T) u = *reinterpret_cast<const uint4*>(xb + (long long)t * C + c);
    *reinterpret_cast<uint4*>(sx + (size_t)r * C + c) = u;
  }
  __syncthreads();
  for (int c = threadIdx.x * 2; c < C; c += DW_THREADS * 2) {
    float2 xr[ROWS_IN];
#pragma unroll
    for (int r = 0; r < ROWS_IN; ++r) xr[r] = __half22float2(*reinterpret_cast<const __half2*>(sx + (size_t)r * C + c));
    float2 acc[DW_TT];
#pragma unroll
    for (int t = 0; t < DW_TT; ++t) acc[t] = make_float2(0.f, 0.f);
    const elem_t* w0 = w + (size_t)c * K;
#pragma unroll
    for (int j = 0; j < K; ++j) {
      const float wa = __half2float(__ldg(w0 + j)), wb = __half2float(__ldg(w0 + K + j));
#pragma unroll
      for (int t = 0; t < DW_TT; ++t) {
        acc[t].x += wa * xr[t + j].x;
        acc[t].y += wb * xr[t + j].y;
      }
    }
#pragma unroll
    for (int t = 0; t < DW_TT; ++t) *reinterpret_cast<float2*>(so + (size_t)t * C + c) = acc[t];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = warp; t < DW_TT; t += DW_THREADS / 32) {
    if (t0 + t >= T) continue;
    const float* row = so + (size_t)t * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += row[c];
    const float mean = warp_sum(s) / C;
    float sq = 0.f;
    for (int c = lane; c < C; c += 32) {
      float d = row[c] - mean;
      sq += d * d;
    }
    const float rstd = rsqrtf(warp_sum(sq) / C + 1e-5f);
    elem_t* yp = y + ((long long)b * T + t0 + t) * C;
    for (int c = lane * 2; c < C; c += 64) {
      float a0 = (row[c] - mean) * rstd * ln_w[c] + ln_b[c];
      float a1 = (row[c + 1] - mean) * rstd * ln_w[c + 1] + ln_b[c + 1];
      a0 = a0 / (1.f + __expf(-a0));
      a1 = a1 / (1.f + __expf(-a1));
      *reinterpret_cast<__half2*>(yp + c) = __floats2half2_rn(a0, a1);
    }
  }
}

// Round-2 kernel for k = 31: 32 output frames per CTA (two passes of 16), one THREAD per channel pair.
//   * the 62-row input window and the whole (C, 31) weight matrix are staged once with cp.async (16 B per request, no
//     registers held); input re-read 62/32 = 1.9x instead of 38/8 = 4.75x, weights once per 32 frames instead of per 8 from
//     global memory with 2-byte uncoalesced loads (the round-1 fixed kernel: 124 such loads per thread);
//   * the 31 taps of a channel pair sit at an ODD word stride (31 words) in shared memory: conflict-free without a transpose;
//   * a pass keeps its 16 outputs per channel in registers; LayerNorm statistics: warp shuffles -> [warps][16] partials ->
//     one warp per frame; nothing but the staged input ever round-trips shared memory.
// fp32 FMA bound: 0.5 GFMA per layer = 16 us at 132 SMs x 128 lanes (H100 SXM, data-sheet clock).
constexpr int DW2_TT = 32, DW2_PASS = 16, DW2_K = 31, DW2_ROWS = DW2_TT + DW2_K - 1;
constexpr int DW2_RED = 3;  // per (warp, frame) partial statistics: sum, sum of squares, sum of squares about the warp's mean

__device__ __forceinline__ void dw_cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}

// V1 = true (sb_dwconv_bias_silu): window t0-15 .. t0+46 (symmetric padding), no LayerNorm; ln_w then holds the per-channel
// bias that follows the folded BatchNorm and ln_b is unused.
template <bool V1>
__global__ void __launch_bounds__(512) dwconv31_tile_kernel(const elem_t* __restrict__ x, elem_t* __restrict__ y,
                                                             const elem_t* __restrict__ w, const float* __restrict__ ln_w,
                                                             const float* __restrict__ ln_b, int T, int C) {
  extern __shared__ __align__(16) uint8_t smem_dw[];
  elem_t* sx = reinterpret_cast<elem_t*>(smem_dw);                                   // [62][C]
  elem_t* sw = sx + (size_t)DW2_ROWS * C;                                            // [C][31] as in global memory
  float* red = reinterpret_cast<float*>(sw + (((size_t)C * DW2_K + 7) & ~(size_t)7)); // [warps][16][DW2_RED]
  const int nwarp = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* stat = red + (size_t)nwarp * DW2_PASS * DW2_RED;                            // [16][2] mean, rstd
  const int b = blockIdx.y, t0 = blockIdx.x * DW2_TT;
  const elem_t* xb = x + (long long)b * T * C;
  const int vec_per_row = C / 8;
  for (int i = threadIdx.x; i < DW2_ROWS * vec_per_row; i += blockDim.x) {
    const int r = i / vec_per_row, c = (i - r * vec_per_row) * 8;
    const int t = t0 - (V1 ? DW2_K / 2 : DW2_K - 1) + r;
    elem_t* dst = sx + (size_t)r * C + c;
    if (t >= 0 && t < T) dw_cp_async16(dst, xb + (long long)t * C + c);
    else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
  const int wvec = (C * DW2_K) / 8;  // C % 8 == 0: the weight matrix is a whole number of 16-byte chunks
  for (int i = threadIdx.x; i < wvec; i += blockDim.x) dw_cp_async16(sw + (size_t)i * 8, w + (size_t)i * 8);
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const int c = threadIdx.x * 2;  // this thread's channel pair (blockDim.x == C / 2)
  // taps: channel c = halves [31c, 31c+31), channel c+1 the next 31: 31 consecutive 32-bit words starting at word 31*(c/2)
  float wa[DW2_K], wb[DW2_K];
  {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(sw) + (size_t)threadIdx.x * DW2_K;
    float h[2 * DW2_K];
#pragma unroll
    for (int n = 0; n < DW2_K; ++n) {
      const uint32_t u = wp[n];
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
      h[2 * n] = f.x; h[2 * n + 1] = f.y;
    }
#pragma unroll
    for (int j = 0; j < DW2_K; ++j) { wa[j] = h[j]; wb[j] = h[DW2_K + j]; }
  }
  const float2 g = *reinterpret_cast<const float2*>(ln_w + c);
  const float2 be = V1 ? make_float2(0.f, 0.f) : *reinterpret_cast<const float2*>(ln_b + c);
#pragma unroll 1
  for (int pass = 0; pass < DW2_TT / DW2_PASS; ++pass) {
    const int f0 = pass * DW2_PASS;  // first output frame of the pass inside the tile; it reads rows f0 .. f0 + 45
    float2 acc[DW2_PASS];
#pragma unroll
    for (int t = 0; t < DW2_PASS; ++t) acc[t] = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < DW2_PASS + DW2_K - 1; ++r) {
      const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(sx + (size_t)(f0 + r) * C + c));
#pragma unroll
      for (int t = 0; t < DW2_PASS; ++t) {
        if (r - t >= 0 && r - t < DW2_K) {  // compile-time after unrolling
          acc[t].x += wa[r - t] * xv.x;
          acc[t].y += wb[r - t] * xv.y;
        }
      }
    }
    if constexpr (V1) {
#pragma unroll
      for (int t = 0; t < DW2_PASS; ++t) {
        const int tt = t0 + f0 + t;
        if (tt < T) {
          float a0 = acc[t].x + g.x, a1 = acc[t].y + g.y;
          a0 = a0 / (1.f + __expf(-a0));
          a1 = a1 / (1.f + __expf(-a1));
          *reinterpret_cast<__half2*>(y + ((long long)b * T + tt) * C + c) = __floats2half2_rn(a0, a1);
        }
      }
      continue;
    }
    // LayerNorm statistics of the 16 frames over all channels.  var = E[a^2] - mean^2 in fp32 is accurate while |mean| is a
    // few sd and loses the variance from |mean| ~ 100 sd on; there the per-warp sums of squares about each warp's own mean
    // (64 channels) are combined instead, with the parallel-variance formula M2 = sum_w M2_w + 64 sum_w (mean_w - mean)^2.
    // Frames with |mean| <= 8 sd keep E[a^2] - mean^2 bit for bit (its error there is ~1e-5 of the variance).
#pragma unroll
    for (int t = 0; t < DW2_PASS; ++t) {
      const float s = warp_sum(acc[t].x + acc[t].y);
      const float q = warp_sum(acc[t].x * acc[t].x + acc[t].y * acc[t].y);
      const float mw = s * (1.f / 64.f);
      const float dx = acc[t].x - mw, dy = acc[t].y - mw;
      const float m2 = warp_sum(dx * dx + dy * dy);
      if (lane == 0) {
        float* r = red + ((size_t)warp * DW2_PASS + t) * DW2_RED;
        r[0] = s; r[1] = q; r[2] = m2;
      }
    }
    __syncthreads();
    for (int f = warp; f < DW2_PASS; f += nwarp) {  // one warp per frame (fewer warps than frames when C < 1024)
      float s = 0.f, q = 0.f;
      for (int i = lane; i < nwarp; i += 32) { s += red[((size_t)i * DW2_PASS + f) * DW2_RED]; q += red[((size_t)i * DW2_PASS + f) * DW2_RED + 1]; }
      s = warp_sum(s); q = warp_sum(q);
      const float mean = s / C;
      float m2 = 0.f;  // every lane takes part in the shuffles; lane 0 decides which variance to keep
      for (int i = lane; i < nwarp; i += 32) {
        const float* r = red + ((size_t)i * DW2_PASS + f) * DW2_RED;
        const float d = r[0] * (1.f / 64.f) - mean;
        m2 += r[2] + 64.f * d * d;
      }
      m2 = warp_sum(m2);
      if (lane == 0) {
        const float e2 = q / C;
        const float var1 = __fsub_rn(e2, __fmul_rn(mean, mean));  // rounded twice, not fused: the established statistics
        stat[f * 2] = mean;
        stat[f * 2 + 1] = e2 > 65.f * var1 ? rsqrtf(m2 / C + 1e-5f) : rsqrtf(fmaxf(var1, 0.f) + 1e-5f);
      }
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < DW2_PASS; ++t) {
      const int tt = t0 + f0 + t;
      if (tt < T) {
        const float mean = stat[t * 2], rstd = stat[t * 2 + 1];
        float a0 = (acc[t].x - mean) * rstd * g.x + be.x;
        float a1 = (acc[t].y - mean) * rstd * g.y + be.y;
        a0 = a0 / (1.f + __expf(-a0));
        a1 = a1 / (1.f + __expf(-a1));
        *reinterpret_cast<__half2*>(y + ((long long)b * T + tt) * C + c) = __floats2half2_rn(a0, a1);
      }
    }
    __syncthreads();  // red / stat are reused by the next pass
  }
}

}  // namespace sb

extern "C" int sb_dwconv_ln_silu(const void* x, void* y, const void* w, const float* ln_w, const float* ln_b,
                                 int32_t batch, int32_t T, int32_t C, int32_t k, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && y && w && ln_w && ln_b && batch > 0 && T > 0 && k > 0, SB_EINVAL, "sb_dwconv_ln_silu: bad args");
  SB_REQUIRE(C % 8 == 0, SB_ENOSUP, "sb_dwconv_ln_silu: C must be a multiple of 8");
  if (k == 31 && C % 64 == 0 && C <= 1024) {
    static int tile_ok = -1;
    if (tile_ok < 0) { const char* e = getenv("SB_DWCONV_TILE"); tile_ok = (e == nullptr || atoi(e) != 0) ? 1 : 0; }
    const int threads = C / 2, nwarp = threads / 32;
    const size_t smem2 = (size_t)DW2_ROWS * C * 2 + (((size_t)C * DW2_K + 7) & ~(size_t)7) * 2 + (size_t)nwarp * DW2_PASS * DW2_RED * 4 + DW2_PASS * 2 * 4;
    if (tile_ok && smem2 <= 220 * 1024) {
      static size_t configured2 = 0;
      if (smem2 > configured2) {
        SB_CUDA_OK(cudaFuncSetAttribute(dwconv31_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        configured2 = smem2;
      }
      dwconv31_tile_kernel<false><<<dim3((T + DW2_TT - 1) / DW2_TT, batch), threads, smem2, (cudaStream_t)stream>>>(
          (const elem_t*)x, (elem_t*)y, (const elem_t*)w, ln_w, ln_b, T, C);
      SB_LAUNCH_OK();
      return SB_OK;
    }
  }
  dim3 grid((T + DW_TT - 1) / DW_TT, batch);
  if (k == 31) {
    const size_t smem31 = (size_t)(DW_TT + 30) * C * 2 + (size_t)DW_TT * C * 4;
    if (smem31 <= 200 * 1024) {
      static size_t configured31 = 0;
      if (smem31 > configured31) {
        SB_CUDA_OK(cudaFuncSetAttribute(dwconv_ln_silu_fixed_kernel<31>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem31));
        configured31 = smem31;
      }
      dwconv_ln_silu_fixed_kernel<31><<<grid, DW_THREADS, smem31, (cudaStream_t)stream>>>(
          (const elem_t*)x, (elem_t*)y, (const elem_t*)w, ln_w, ln_b, T, C);
      SB_LAUNCH_OK();
      return SB_OK;
    }
  }
  size_t smem = (size_t)(DW_TT + k - 1) * C * 2 + (size_t)k * C * 2 + (size_t)DW_TT * C * 4;
  SB_REQUIRE(smem <= 200 * 1024, SB_ENOSUP, "sb_dwconv_ln_silu: C*k too large for shared memory (%zu B)", smem);
  static size_t configured = 0;
  if (smem > configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(dwconv_ln_silu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  dwconv_ln_silu_kernel<<<grid, DW_THREADS, smem, (cudaStream_t)stream>>>((const elem_t*)x, (elem_t*)y, (const elem_t*)w, ln_w,
                                                                         ln_b, T, C, k);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_dwconv_bias_silu(const void* x, void* y, const void* w, const float* bias, int32_t batch, int32_t T, int32_t C,
                                   int32_t k, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && y && w && bias && batch > 0 && T > 0, SB_EINVAL, "sb_dwconv_bias_silu: bad args");
  SB_REQUIRE(k == DW2_K && C % 64 == 0 && C <= 1024, SB_ENOSUP, "sb_dwconv_bias_silu: needs k = 31 and C a multiple of 64 up to 1024");
  const int threads = C / 2;
  const size_t smem = (size_t)DW2_ROWS * C * 2 + (((size_t)C * DW2_K + 7) & ~(size_t)7) * 2 + (size_t)(threads / 32) * DW2_PASS * DW2_RED * 4 +
                      DW2_PASS * 2 * 4;
  static size_t configured = 0;
  if (smem > configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(dwconv31_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  dwconv31_tile_kernel<true><<<dim3((T + DW2_TT - 1) / DW2_TT, batch), threads, smem, (cudaStream_t)stream>>>(
      (const elem_t*)x, (elem_t*)y, (const elem_t*)w, bias, nullptr, T, C);
  SB_LAUNCH_OK();
  return SB_OK;
}
