// EMMA monotonic-attention step probability (SeamlessStreaming, SURVEY 8a a17):
//   PChooseLayer.forward (models/monotonic_decoder/p_choose.py:120-148):
//     q = EnergyProjection(seqs)  (4 x Linear+ReLU: sb_gemm),  k = EnergyProjection(AvgPool1d(keys, ratio, ceil))
//     p_choose[h,s,j] = sigmoid((q_h[s] . k_h[j] / sqrt(64) + energy_bias) / temperature)
// The kernels here are the pooling, the energy/sigmoid (one sequence, or the newest position of each stream of a ragged
// batch) and the policy decision of a batch of streams; all are tiny and latency bound.
#include "common.cuh"

namespace sb {

// y[b][j][c] = mean_{t in [j*r, min((j+1)*r, T))} x[b][t][c]      (AvgPool1d(kernel=stride=r, ceil_mode=True))
__global__ void avgpool_time_kernel(const elem_t* __restrict__ x, elem_t* __restrict__ y, int T, int C, int r, int Tp) {
  const int j = blockIdx.x, b = blockIdx.y;
  const int t0 = j * r, t1 = min(t0 + r, T);
  const float inv = 1.f / (float)(t1 - t0);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int t = t0; t < t1; ++t) acc += __half2float(x[((long long)b * T + t) * C + c]);
    y[((long long)b * Tp + j) * C + c] = __float2half_rn(acc * inv);
  }
}

// sigmoid((q_h . k_h / 8 + bias) / temperature) of one head's 64 dims, one warp; the result is valid on every lane.
// Shared by both p_choose kernels so that the ragged entry computes each value exactly as the per-sequence one does.
__device__ __forceinline__ float pchoose_value(const elem_t* __restrict__ q_row, const elem_t* __restrict__ k_row, int lane,
                                               float bias, float inv_temp) {
  const float2 a = __half22float2(reinterpret_cast<const __half2*>(q_row)[lane]);
  const float2 b = __half22float2(reinterpret_cast<const __half2*>(k_row)[lane]);
  const float e = warp_sum(a.x * b.x + a.y * b.y) * 0.125f + bias;
  return 1.f / (1.f + __expf(-e * inv_temp));
}

// one warp per (head, s, j): 64-dim dot product
__global__ void pchoose_kernel(const elem_t* __restrict__ q, const elem_t* __restrict__ k, float* __restrict__ p, int S, int Sp,
                               int heads, float bias, float inv_temp) {
  const int lane = threadIdx.x & 31;
  const long long idx = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)heads * S * Sp;
  if (idx >= total) return;
  const int j = (int)(idx % Sp), s = (int)((idx / Sp) % S), h = (int)(idx / ((long long)Sp * S));
  const int dim = heads * 64;
  const float v = pchoose_value(q + (long long)s * dim + h * 64, k + (long long)j * dim + h * 64, lane, bias, inv_temp);
  if (lane == 0) p[idx] = v;
}

// one warp per (stream b, head h): p[b][h] = p_choose of b's newest target position (q_lens[b] - 1) against its last pooled
// source position (k_lens[b] - 1), the only entry MMATextDecoderAgent's decision reads.  q and k are in sequence layout,
// q_rows / k_rows rows per stream; no other row is read.
__global__ void pchoose_last_kernel(const elem_t* __restrict__ q, int q_rows, const elem_t* __restrict__ k, int k_rows,
                                    const int* __restrict__ q_lens, const int* __restrict__ k_lens, float* __restrict__ p,
                                    int batch, int heads, float bias, float inv_temp) {
  const int lane = threadIdx.x & 31;
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= batch * heads) return;
  const int b = idx / heads, h = idx % heads;
  const int s = q_lens[b] - 1, j = k_lens[b] - 1;
  if (s < 0 || s >= q_rows || j < 0 || j >= k_rows) {  // a length outside the layout: nothing valid to read
    if (lane == 0) p[idx] = __int_as_float(0x7fc00000);
    return;
  }
  const int dim = heads * 64;
  const float v = pchoose_value(q + ((long long)b * q_rows + s) * dim + h * 64, k + ((long long)b * k_rows + j) * dim + h * 64,
                                lane, bias, inv_temp);
  if (lane == 0) p[idx] = v;
}

// (a, ia) ranks before (b, ib) in torch.argmax's order: NaN first (it is the maximum), then larger values, ties to the
// lower index
__device__ __forceinline__ bool argmax_before(float a, int ia, float b, int ib) {
  const bool na = isnan(a), nb = isnan(b);
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

constexpr int DECIDE_THREADS = 256;

// One CTA per stream: the token (argmax over the stream's logits with its blocked ids at -inf) and the decision value
// (min / mean / lower median of p[layer0..layers)[b][0..heads)), written as out[b] = {token, float bits of the value}.
// ctl[b] = {4 blocked ids (-1 = unused), method, layer0}: every stream has its own options.
__global__ void __launch_bounds__(DECIDE_THREADS) policy_decide_kernel(
    const float* __restrict__ logits, long long ld, int vocab, const int* __restrict__ ctl, const float* __restrict__ p,
    int layers, int heads, int batch, int* __restrict__ out) {
  extern __shared__ float vals[];  // the n decision inputs
  __shared__ float red_v[DECIDE_THREADS / 32];
  __shared__ int red_i[DECIDE_THREADS / 32];
  __shared__ float s_prob;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int* c = ctl + b * SB_POLICY_CTL;
  const int method = c[SB_POLICY_MAX_BLOCKED], layer0 = c[SB_POLICY_MAX_BLOCKED + 1];
  if (layer0 < 0 || layer0 >= layers || method < SB_POLICY_MIN || method > SB_POLICY_MEDIAN) {
    if (tid == 0) out[2 * b] = -1, out[2 * b + 1] = 0x7fc00000;  // ops.policy_ctl refuses these; never a valid result
    return;
  }
  const int n = (layers - layer0) * heads;
  int nan_seen = 0;
  for (int i = tid; i < n; i += DECIDE_THREADS) {
    const int l = layer0 + i / heads, h = i % heads;
    vals[i] = p[((long long)l * batch + b) * heads + h];
    nan_seen |= isnan(vals[i]);
  }
  if (tid == 0) s_prob = __int_as_float(0x7fc00000);  // the median of values with a NaN is NaN, as in torch
  int blk[SB_POLICY_MAX_BLOCKED];
#pragma unroll
  for (int i = 0; i < SB_POLICY_MAX_BLOCKED; ++i) blk[i] = c[i];
  // token: every thread scans its strided ids in increasing order, so a strict comparison keeps the lowest tied index
  const float* row = logits + (long long)b * ld;
  float bv = -INFINITY;
  int bi = vocab;
  for (int v = tid; v < vocab; v += DECIDE_THREADS) {
    float x = row[v];
#pragma unroll
    for (int i = 0; i < SB_POLICY_MAX_BLOCKED; ++i)
      if (blk[i] == v) x = -INFINITY;
    if (bi == vocab || argmax_before(x, v, bv, bi)) bv = x, bi = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi < vocab && (bi == vocab || argmax_before(ov, oi, bv, bi))) bv = ov, bi = oi;
  }
  if (lane == 0) red_v[warp] = bv, red_i[warp] = bi;
  const int any_nan = __syncthreads_or(nan_seen);  // also publishes vals and the NaN default of s_prob
  // decision value
  if (method == SB_POLICY_MEDIAN) {
    // torch.median: the lower median, the element of rank (n - 1) / 2 with ties ranked by position; NaN if any is NaN
    const int want = any_nan ? -1 : (n - 1) / 2;
    for (int i = any_nan ? n : tid; i < n; i += DECIDE_THREADS) {
      const float x = vals[i];
      int r = 0;
      for (int j = 0; j < n; ++j) r += (vals[j] < x) || (vals[j] == x && j < i);
      if (r == want) s_prob = x;
    }
  } else if (tid == 0) {
    if (method == SB_POLICY_MIN) {
      float m = vals[0];
      for (int i = 1; i < n; ++i) m = (vals[i] < m || isnan(vals[i])) && !isnan(m) ? vals[i] : m;  // NaN propagates, as in torch
      s_prob = m;
    } else {  // mean: a float64 running sum in layer-major order, rounded once
      double acc = 0.0;
      for (int i = 0; i < n; ++i) acc += (double)vals[i];
      s_prob = (float)(acc / (double)n);
    }
  }
  __syncthreads();
  if (tid == 0) {
    float v = red_v[0];
    int i = red_i[0];
    for (int w = 1; w < DECIDE_THREADS / 32; ++w)
      if (red_i[w] < vocab && (i == vocab || argmax_before(red_v[w], red_i[w], v, i))) v = red_v[w], i = red_i[w];
    out[2 * b] = i;
    out[2 * b + 1] = __float_as_int(s_prob);
  }
}

}  // namespace sb

extern "C" int sb_avgpool_time(const void* x, void* y, int32_t batch, int32_t T, int32_t C, int32_t ratio, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && y && batch > 0 && T > 0 && C > 0 && ratio > 0, SB_EINVAL, "sb_avgpool_time: bad args");
  const int Tp = (T + ratio - 1) / ratio;
  avgpool_time_kernel<<<dim3(Tp, batch), 256, 0, (cudaStream_t)stream>>>((const elem_t*)x, (elem_t*)y, T, C, ratio, Tp);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_pchoose(const void* q_energy, const void* k_energy, float* p, int32_t S, int32_t Sp, int32_t heads,
                          float energy_bias, float temperature, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(q_energy && k_energy && p && S > 0 && Sp > 0 && heads > 0 && temperature > 0.f, SB_EINVAL, "sb_pchoose: bad args");
  const long long total = (long long)heads * S * Sp;
  pchoose_kernel<<<(unsigned)((total + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const elem_t*)q_energy, (const elem_t*)k_energy, p,
                                                                              S, Sp, heads, energy_bias, 1.f / temperature);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_pchoose_ragged(const void* q_energy, int32_t q_rows, const void* k_energy, int32_t k_rows, const int32_t* q_lens,
                                 const int32_t* k_lens, float* p, int32_t batch, int32_t heads, float energy_bias, float temperature,
                                 sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(q_energy && k_energy && q_lens && k_lens && p && q_rows > 0 && k_rows > 0 && batch > 0 && heads > 0 && temperature > 0.f,
             SB_EINVAL, "sb_pchoose_ragged: bad args");
  const int total = batch * heads;
  pchoose_last_kernel<<<(total + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const elem_t*)q_energy, q_rows, (const elem_t*)k_energy,
                                                                         k_rows, q_lens, k_lens, p, batch, heads, energy_bias,
                                                                         1.f / temperature);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_policy_decide(const float* logits, int64_t ld, int32_t vocab, const int32_t* ctl, const float* p,
                                int32_t layers, int32_t heads, int32_t batch, int32_t* out, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(logits && ctl && p && out && vocab > 0 && ld >= vocab && batch > 0 && heads > 0 && layers > 0, SB_EINVAL,
             "sb_policy_decide: bad args");
  const long long n = (long long)layers * heads;
  SB_REQUIRE(n <= SB_POLICY_MAX_VALUES, SB_ENOSUP, "sb_policy_decide: %lld decision values exceed %d", n, SB_POLICY_MAX_VALUES);
  policy_decide_kernel<<<batch, DECIDE_THREADS, n * sizeof(float), (cudaStream_t)stream>>>(logits, ld, vocab, ctl, p, layers,
                                                                                          heads, batch, out);
  SB_LAUNCH_OK();
  return SB_OK;
}
