// sb_layernorm: row LayerNorm (eps 1e-5) with optional residual add, sequence-layout remap and padding mask.
// One warp per row, 16-byte loads, fp32 statistics (two-pass over registers).  HBM-bound: 2*dim*2 B per row.
#include "common.cuh"

namespace sb {

constexpr int LN_MAX_CHUNKS = 8;  // dim <= 8 * 256 = 2048

// ACT: SB_ACT_NONE (sb_layernorm) or SB_ACT_GELU (sb_layernorm_gelu, applied before the fp16 rounding)
template <int ACT>
__global__ void __launch_bounds__(256) layernorm_kernel(const elem_t* __restrict__ x, const elem_t* __restrict__ res,
                                                        elem_t* __restrict__ y, elem_t* __restrict__ sum_out,
                                                        const float* __restrict__ w, const float* __restrict__ bvec, int dim,
                                                        long long total_rows, int T, int in_rows, int in_halo, int out_rows,
                                                        int out_halo, const int* __restrict__ lens, int mask_out) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= total_rows) return;
  const int b = (int)(row / T), t = (int)(row - (long long)b * T);
  const long long rin = (long long)b * in_rows + in_halo + t, rout = (long long)b * out_rows + out_halo + t;
  const elem_t* xp = x + rin * dim;
  elem_t* yp = y + rout * dim;
  const bool masked = mask_out && lens != nullptr && t >= lens[b];
  const int nchunk = (dim + 255) / 256;
  float v[LN_MAX_CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < LN_MAX_CHUNKS; ++c) {
    if (c >= nchunk) break;
    const int off = c * 256 + lane * 8;
    if (off < dim) {
      uint4 u = *reinterpret_cast<const uint4*>(xp + off);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h[e]);
        v[c][2 * e] = f.x;
        v[c][2 * e + 1] = f.y;
      }
      if (res != nullptr) {
        uint4 u2 = *reinterpret_cast<const uint4*>(res + rin * dim + off);
        const __half2* h2 = reinterpret_cast<const __half2*>(&u2);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __half22float2(h2[e]);
          v[c][2 * e] += f.x;
          v[c][2 * e + 1] += f.y;
        }
        if (sum_out != nullptr) {
          uint4 o;
          __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
          for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(v[c][2 * e], v[c][2 * e + 1]);
          *reinterpret_cast<uint4*>(sum_out + rout * dim + off) = o;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[c][e];
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[c][e] = 0.f;
    }
  }
  const float mean = warp_sum(s) / dim;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < LN_MAX_CHUNKS; ++c) {
    if (c >= nchunk) break;
    const int off = c * 256 + lane * 8;
    if (off < dim) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float d = v[c][e] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / dim + 1e-5f);
#pragma unroll
  for (int c = 0; c < LN_MAX_CHUNKS; ++c) {
    if (c >= nchunk) break;
    const int off = c * 256 + lane * 8;
    if (off < dim) {
      float4 w0 = *reinterpret_cast<const float4*>(w + off), w1 = *reinterpret_cast<const float4*>(w + off + 4);
      float4 b0 = *reinterpret_cast<const float4*>(bvec + off), b1 = *reinterpret_cast<const float4*>(bvec + off + 4);
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint4 o;
      __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float a0 = masked ? 0.f : (v[c][2 * e] - mean) * rstd * ww[2 * e] + bb[2 * e];
        float a1 = masked ? 0.f : (v[c][2 * e + 1] - mean) * rstd * ww[2 * e + 1] + bb[2 * e + 1];
        if constexpr (ACT == SB_ACT_GELU) {
          a0 = gelu_erf(a0);
          a1 = gelu_erf(a1);
        }
        ho[e] = __floats2half2_rn(a0, a1);
      }
      *reinterpret_cast<uint4*>(yp + off) = o;
    }
  }
}

// x_new = x + bias + sum_z partial[z]  (fp32 sum in fixed z order, rounded to fp16 like the unfused residual stream),
// h = LN(x_new).  One CTA per row, one warp per 256-column chunk (all slice loads of a chunk are in flight together),
// statistics through shared memory.  Consumer of sb_gemm_splitk for the decoder's residual GEMMs.
__global__ void __launch_bounds__(32 * LN_MAX_CHUNKS) splitk_reduce_ln_kernel(const float* __restrict__ partials, int splits,
                                                                              long long rows, long long slice_rows, int dim,
                                                                              const float* __restrict__ bias, elem_t* __restrict__ x,
                                                                              const float* __restrict__ w,
                                                                              const float* __restrict__ bvec, elem_t* __restrict__ h) {
  __shared__ float s_part[2][LN_MAX_CHUNKS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const long long row = blockIdx.x;
  const int off = warp * 256 + lane * 8;
  const bool act = off < dim;
  pdl_sync();
  float v[8];
  float s = 0.f;
  if (act) {
    float acc[8];
    {
      const uint4 u = *reinterpret_cast<const uint4*>(x + row * dim + off);
      const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); acc[2 * e] = f.x; acc[2 * e + 1] = f.y; }
    }
    if (bias != nullptr) {
      const float4 b0 = *reinterpret_cast<const float4*>(bias + off), b1 = *reinterpret_cast<const float4*>(bias + off + 4);
      acc[0] += b0.x; acc[1] += b0.y; acc[2] += b0.z; acc[3] += b0.w; acc[4] += b1.x; acc[5] += b1.y; acc[6] += b1.z; acc[7] += b1.w;
    }
    int z = 0;
    for (; z + 8 <= splits; z += 8) {  // 16 loads in flight per lane: one round trip for up to 8 slices
      float4 p0[8], p1[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float* pp = partials + ((long long)(z + u) * slice_rows + row) * dim + off;
        p0[u] = *reinterpret_cast<const float4*>(pp);
        p1[u] = *reinterpret_cast<const float4*>(pp + 4);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        acc[0] += p0[u].x; acc[1] += p0[u].y; acc[2] += p0[u].z; acc[3] += p0[u].w;
        acc[4] += p1[u].x; acc[5] += p1[u].y; acc[6] += p1[u].z; acc[7] += p1[u].w;
      }
    }
    for (; z + 4 <= splits; z += 4) {
      float4 p0[4], p1[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float* pp = partials + ((long long)(z + u) * slice_rows + row) * dim + off;
        p0[u] = *reinterpret_cast<const float4*>(pp);
        p1[u] = *reinterpret_cast<const float4*>(pp + 4);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        acc[0] += p0[u].x; acc[1] += p0[u].y; acc[2] += p0[u].z; acc[3] += p0[u].w;
        acc[4] += p1[u].x; acc[5] += p1[u].y; acc[6] += p1[u].z; acc[7] += p1[u].w;
      }
    }
    for (; z < splits; ++z) {
      const float* pp = partials + ((long long)z * slice_rows + row) * dim + off;
      const float4 p0 = *reinterpret_cast<const float4*>(pp), p1 = *reinterpret_cast<const float4*>(pp + 4);
      acc[0] += p0.x; acc[1] += p0.y; acc[2] += p0.z; acc[3] += p0.w; acc[4] += p1.x; acc[5] += p1.y; acc[6] += p1.z; acc[7] += p1.w;
    }
    uint4 o;
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      ho[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
      const float2 f = __half22float2(ho[e]);  // LN sees the fp16-rounded residual stream
      v[2 * e] = f.x; v[2 * e + 1] = f.y;
      s += f.x + f.y;
    }
    *reinterpret_cast<uint4*>(x + row * dim + off) = o;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  }
  s = warp_sum(s);
  if (lane == 0) s_part[0][warp] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < nwarp; ++i) tot += s_part[0][i];
  const float mean = tot / dim;
  float sq = 0.f;
  if (act) {
#pragma unroll
    for (int e = 0; e < 8; ++e) { const float d = v[e] - mean; sq += d * d; }
  }
  sq = warp_sum(sq);
  if (lane == 0) s_part[1][warp] = sq;
  __syncthreads();
  float tsq = 0.f;
  for (int i = 0; i < nwarp; ++i) tsq += s_part[1][i];
  const float rstd = rsqrtf(tsq / dim + 1e-5f);
  if (act) {
    const float4 w0 = *reinterpret_cast<const float4*>(w + off), w1 = *reinterpret_cast<const float4*>(w + off + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(bvec + off), b1 = *reinterpret_cast<const float4*>(bvec + off + 4);
    const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    uint4 o;
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e)
      ho[e] = __floats2half2_rn((v[2 * e] - mean) * rstd * ww[2 * e] + bb[2 * e], (v[2 * e + 1] - mean) * rstd * ww[2 * e + 1] + bb[2 * e + 1]);
    *reinterpret_cast<uint4*>(h + row * dim + off) = o;
  }
}

}  // namespace sb

extern "C" int sb_splitk_reduce_ln(const float* partials, int32_t splits, int32_t rows, int64_t slice_rows, int32_t dim,
                                   const float* bias, void* x,
                                   const float* ln_w, const float* ln_b, void* h, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(partials && x && ln_w && ln_b && h && splits >= 1 && rows > 0, SB_EINVAL, "sb_splitk_reduce_ln: bad args");
  SB_REQUIRE(dim % 8 == 0 && dim <= 256 * LN_MAX_CHUNKS, SB_ENOSUP, "sb_splitk_reduce_ln: dim %d unsupported", dim);
  const int nwarp = (dim + 255) / 256;
  SB_CUDA_OK(prefer_shared(splitk_reduce_ln_kernel));
  SB_CUDA_OK(launch_k(splitk_reduce_ln_kernel, dim3(rows), dim3(nwarp * 32), 0, (cudaStream_t)stream, partials,
                       (int)splits, (long long)rows, (long long)slice_rows, (int)dim, bias, (elem_t*)x, ln_w, ln_b, (elem_t*)h));
  count_launch();
  return SB_OK;
}

extern "C" int sb_layernorm(const void* x, const void* res, void* y, void* sum_out, const float* w, const float* b,
                            int32_t dim, int32_t batch, int32_t T, int32_t in_rows, int32_t in_halo, int32_t out_rows,
                            int32_t out_halo, const int32_t* lens, int32_t mask_out, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && y && w && b && batch > 0 && T > 0, SB_EINVAL, "sb_layernorm: bad args");
  SB_REQUIRE(dim % 8 == 0 && dim <= 256 * LN_MAX_CHUNKS, SB_ENOSUP, "sb_layernorm: dim %d unsupported (multiple of 8, <= 2048)", dim);
  const long long rows = (long long)batch * T;
  const int wpb = rows >= 4096 ? 8 : 2;  // small problems: more CTAs, shorter critical path
  SB_CUDA_OK(prefer_shared((layernorm_kernel<SB_ACT_NONE>)));
  SB_CUDA_OK(launch_k(layernorm_kernel<SB_ACT_NONE>, dim3((unsigned)((rows + wpb - 1) / wpb)), dim3(wpb * 32), 0, (cudaStream_t)stream,
                       (const elem_t*)x, (const elem_t*)res, (elem_t*)y, (elem_t*)sum_out, w, b, (int)dim, rows, (int)T,
                       (int)in_rows, (int)in_halo, (int)out_rows, (int)out_halo, lens, (int)mask_out));
  count_launch();
  return SB_OK;
}

extern "C" int sb_layernorm_gelu(const void* x, void* y, const float* w, const float* b, int32_t dim, int32_t batch, int32_t T,
                                 int32_t in_rows, int32_t in_halo, int32_t out_rows, int32_t out_halo, const int32_t* lens,
                                 int32_t mask_out, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && y && w && b && batch > 0 && T > 0, SB_EINVAL, "sb_layernorm_gelu: bad args");
  SB_REQUIRE(dim % 8 == 0 && dim <= 256 * LN_MAX_CHUNKS, SB_ENOSUP, "sb_layernorm_gelu: dim %d unsupported (multiple of 8, <= 2048)", dim);
  const long long rows = (long long)batch * T;
  const int wpb = rows >= 4096 ? 8 : 2;
  SB_CUDA_OK(launch_k(layernorm_kernel<SB_ACT_GELU>, dim3((unsigned)((rows + wpb - 1) / wpb)), dim3(wpb * 32), 0,
                       (cudaStream_t)stream, (const elem_t*)x, (const elem_t*)nullptr, (elem_t*)y, (elem_t*)nullptr, w, b,
                       (int)dim, rows, (int)T, (int)in_rows, (int)in_halo, (int)out_rows, (int)out_halo, lens, (int)mask_out));
  count_launch();
  return SB_OK;
}
