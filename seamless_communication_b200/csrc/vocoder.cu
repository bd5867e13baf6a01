// Code-HiFiGAN glue kernels (models/vocoder/codehifigan.py:75-101, hifigan.py:180-196).  The convolution stack
// itself runs through sb_gemm (conv taps via TMA row offsets, ConvTranspose1d as a phase-decomposed 3-tap GEMM,
// leaky-relu / residual / resblock-mean fused into the epilogues); only the embedding concat and the final
// C->1 conv + tanh are separate, bandwidth-bound kernels.
#include "common.cuh"

namespace sb {

// x[b][u] = [ lang[lang_idx[b]] | dict[units[b][u]] | spkr[spkr_idx[b]] ]  (codehifigan.py:98-100 channel order)
__global__ void __launch_bounds__(256) vocoder_embed_kernel(const int* __restrict__ units, int U, const elem_t* __restrict__ dict,
                                                            int dict_dim, const elem_t* __restrict__ lang, int lang_dim,
                                                            const int* __restrict__ lang_idx, const elem_t* __restrict__ spkr,
                                                            int spkr_dim, const int* __restrict__ spkr_idx, elem_t* __restrict__ x,
                                                            int x_rows, int x_halo) {
  const int u = blockIdx.x, b = blockIdx.y;
  const int C = lang_dim + dict_dim + spkr_dim;
  elem_t* xp = x + ((long long)b * x_rows + x_halo + u) * C;
  const elem_t* lp = lang + (long long)lang_idx[b] * lang_dim;
  const elem_t* dp = dict + (long long)units[(long long)b * U + u] * dict_dim;
  const elem_t* sp = spkr + (long long)spkr_idx[b] * spkr_dim;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    elem_t v;
    if (c < lang_dim) v = lp[c];
    else if (c < lang_dim + dict_dim) v = dp[c - lang_dim];
    else v = sp[c - lang_dim - dict_dim];
    xp[c] = v;
  }
}

// wav[b][t] = tanh(bias + sum_{j,c} x[b][t + j - k/2][c] * w[j][c]);  x is already leaky-relu'ed, halos are zero.
// With per-sequence lengths, wav[b][t] = 0 for t >= lens[b].
__global__ void __launch_bounds__(256) conv_post_tanh_kernel(const elem_t* __restrict__ x, int x_rows, int x_halo, int T,
                                                             const int* __restrict__ lens, int C, const elem_t* __restrict__ w,
                                                             float bias, int k, float* __restrict__ wav, long long wav_ld) {
  extern __shared__ float sw[];  // [k*C]
  for (int i = threadIdx.x; i < k * C; i += blockDim.x) sw[i] = __half2float(w[i]);
  __syncthreads();
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  if (lens != nullptr && t >= lens[b]) {
    wav[(long long)b * wav_ld + t] = 0.f;
    return;
  }
  const elem_t* xp = x + ((long long)b * x_rows + x_halo + t - k / 2) * C;  // halo >= k/2 guarantees in-bounds zeros
  float acc = bias;
  for (int i = 0; i < k * C; i += 8) {
    uint4 u = *reinterpret_cast<const uint4*>(xp + i);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = __half22float2(h[e]);
      acc += f.x * sw[i + 2 * e] + f.y * sw[i + 2 * e + 1];
    }
  }
  wav[(long long)b * wav_ld + t] = tanhf(acc);
}

}  // namespace sb

extern "C" int sb_vocoder_embed(const int32_t* units, int32_t U, int32_t batch, const void* dict, int32_t dict_dim,
                                const void* lang, int32_t lang_dim, const int32_t* lang_idx, const void* spkr, int32_t spkr_dim,
                                const int32_t* spkr_idx, void* x, int32_t x_rows, int32_t x_halo, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(units && dict && lang && lang_idx && spkr && spkr_idx && x && U > 0 && batch > 0, SB_EINVAL, "sb_vocoder_embed: bad args");
  vocoder_embed_kernel<<<dim3(U, batch), 256, 0, (cudaStream_t)stream>>>(units, U, (const elem_t*)dict, dict_dim, (const elem_t*)lang,
                                                                        lang_dim, lang_idx, (const elem_t*)spkr, spkr_dim, spkr_idx,
                                                                        (elem_t*)x, x_rows, x_halo);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_conv_post_tanh(const void* x, int32_t x_rows, int32_t x_halo, int32_t T, const int32_t* lens, int32_t C,
                                 int32_t batch, const void* w, float bias, int32_t k, float* wav, int64_t wav_ld,
                                 sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && w && wav && T > 0 && batch > 0 && k > 0, SB_EINVAL, "sb_conv_post_tanh: bad args");
  SB_REQUIRE(C % 8 == 0 && x_halo >= k / 2, SB_ENOSUP, "sb_conv_post_tanh: C must be a multiple of 8 and halo >= k/2");
  dim3 grid((T + 255) / 256, batch);
  conv_post_tanh_kernel<<<grid, 256, (size_t)k * C * sizeof(float), (cudaStream_t)stream>>>((const elem_t*)x, x_rows, x_halo, T, lens,
                                                                                          C, (const elem_t*)w, bias, k, wav, wav_ld);
  SB_LAUNCH_OK();
  return SB_OK;
}
