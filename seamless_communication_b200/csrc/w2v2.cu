// sb_w2v2_front: the waveform end of the XLS-R feature extractor (unit_extractor.py:88-93 + fairseq2's wav2vec2 feature
// extractor layer 0): per-row normalisation statistics, then Conv1d(1 -> 512, k10, s5) -> LayerNorm(512) -> GELU.
// Layer 0 has 10 MACs per output value, so it is bound by writing its fp16 output (B * T0 * 1 KB), not by arithmetic: one
// warp per frame, 16 channels per lane (32-byte stores, a whole 1 KB row per warp), fp32 CUDA-core math.
#include "common.cuh"

namespace sb {

constexpr int W2_C = 512, W2_K = 10, W2_S = 5;

// mean and 1/sqrt(var + 1e-5) of row b over its Lp samples (biased variance, fp64 sums); sample L of an odd row is 1.0
__global__ void __launch_bounds__(1024) w2v2_stats_kernel(const float* __restrict__ wave, long long ld,
                                                          const int* __restrict__ num_samples, float* __restrict__ stats) {
  __shared__ double red[2][32];
  const int b = blockIdx.x, L = num_samples[b], Lp = L + (L & 1);
  const float* x = wave + (long long)b * ld;
  double s = 0.0, s2 = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const double v = x[i];
    s += v;
    s2 += v * v;
  }
  if ((L & 1) && threadIdx.x == 0) { s += 1.0; s2 += 1.0; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[0][warp] = s; red[1][warp] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0, ts2 = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { ts += red[0][w]; ts2 += red[1][w]; }
    const double n = Lp > 0 ? (double)Lp : 1.0;
    const double mean = ts / n, var = fmax(ts2 / n - mean * mean, 0.0);
    stats[2 * b] = (float)mean;
    stats[2 * b + 1] = (float)(1.0 / sqrt(var + 1e-5));
  }
}

__global__ void __launch_bounds__(256) w2v2_conv0_kernel(const float* __restrict__ wave, long long ld,
                                                         const int* __restrict__ num_samples, const float* __restrict__ stats,
                                                         const float* __restrict__ w0, const float* __restrict__ b0,
                                                         const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                                                         elem_t* __restrict__ out, int out_rows) {
  // channel c = 16 * lane + i lives at [i][lane] (and the weights at [k][i][lane]): conflict-free per-lane reads
  __shared__ float ws[W2_K * 16 * 32];
  __shared__ float bs[W2_C], gs[W2_C], hs[W2_C];
  for (int idx = threadIdx.x; idx < W2_C * W2_K; idx += blockDim.x) {
    const int c = idx / W2_K, k = idx - c * W2_K;
    ws[(k * 16 + (c & 15)) * 32 + (c >> 4)] = w0[idx];
  }
  for (int c = threadIdx.x; c < W2_C; c += blockDim.x) {
    const int j = (c & 15) * 32 + (c >> 4);
    bs[j] = b0[c]; gs[j] = ln_w[c]; hs[j] = ln_b[c];
  }
  __syncthreads();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int L = num_samples[b], Lp = L + (L & 1);
  const int T0 = Lp >= W2_K ? (Lp - W2_K) / W2_S + 1 : 0;
  const float mean = stats[2 * b], rstd = stats[2 * b + 1];
  const float* x = wave + (long long)b * ld;
  const int wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < out_rows; t += gridDim.x * wpb) {
    uint4* op = reinterpret_cast<uint4*>(out + ((long long)b * out_rows + t) * W2_C + lane * 16);
    if (t >= T0) {
      op[0] = make_uint4(0, 0, 0, 0);
      op[1] = make_uint4(0, 0, 0, 0);
      continue;
    }
    float xn[W2_K];
#pragma unroll
    for (int k = 0; k < W2_K; ++k) {
      const int i = t * W2_S + k;  // < Lp; i == L only for the appended sample of an odd row
      xn[k] = ((i < L ? x[i] : 1.f) - mean) * rstd;
    }
    float a[16];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      float acc = bs[i * 32 + lane];
#pragma unroll
      for (int k = 0; k < W2_K; ++k) acc = fmaf(ws[(k * 16 + i) * 32 + lane], xn[k], acc);
      a[i] = acc;
      s += acc;
    }
    const float m = warp_sum(s) * (1.f / W2_C);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) { const float d = a[i] - m; sq += d * d; }
    const float r = rsqrtf(warp_sum(sq) * (1.f / W2_C) + 1e-5f);
    uint4 u[2];
    __half2* h = reinterpret_cast<__half2*>(u);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y0 = gelu_erf((a[2 * i] - m) * r * gs[2 * i * 32 + lane] + hs[2 * i * 32 + lane]);
      const float y1 = gelu_erf((a[2 * i + 1] - m) * r * gs[(2 * i + 1) * 32 + lane] + hs[(2 * i + 1) * 32 + lane]);
      h[i] = __floats2half2_rn(y0, y1);
    }
    op[0] = u[0];
    op[1] = u[1];
  }
}

}  // namespace sb

extern "C" int sb_w2v2_front(const float* wave, int64_t wave_ld, const int32_t* num_samples, int32_t batch, const float* w0,
                             const float* b0, const float* ln_w, const float* ln_b, void* out, int32_t out_rows, float* stats,
                             sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(wave && num_samples && w0 && b0 && ln_w && ln_b && out && stats && batch > 0 && out_rows > 0, SB_EINVAL,
             "sb_w2v2_front: bad args");
  SB_REQUIRE(batch <= 65535, SB_EINVAL, "sb_w2v2_front: batch %d exceeds 65535", batch);
  cudaStream_t st = (cudaStream_t)stream;
  w2v2_stats_kernel<<<batch, 1024, 0, st>>>(wave, (long long)wave_ld, num_samples, stats);
  SB_LAUNCH_OK();
  // enough CTAs to fill the GPU several times over, few enough that staging the 26 KB of weights stays negligible
  const int per_row = (2048 + batch - 1) / batch;
  const int bx = min((out_rows + 7) / 8, max(per_row, 1));
  w2v2_conv0_kernel<<<dim3(bx, batch), 256, 0, st>>>(wave, (long long)wave_ld, num_samples, stats, w0, b0, ln_w, ln_b,
                                                    (elem_t*)out, out_rows);
  SB_LAUNCH_OK();
  return SB_OK;
}
