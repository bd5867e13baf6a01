// Token start times of the transcriber (reference inference/transcriber.py:178-235: _extract_timestamps, generate_lis)
// for every row of a batch in one launch.  The reference moves the attention matrix to the host and runs scipy's
// medfilt2d and an O(F^2) pure-Python longest increasing subsequence one utterance at a time.
//
// One CTA per row.  With n generated tokens, F = len - 2 encoder frames and W[t] the head-summed cross-attention row of
// decoder position t (sb_decode_cross_attn_weights), gathered along the winner's cache slots:
//   1. A[k][j] = W[P-1+k][1+j] in float64 (k < n, j < F);
//   2. each column divided by its float64 sum over k = 0 .. n-1 in that order (numpy's order for an axis-0 sum); a zero
//      column stays 0;
//   3. a w x w median filter with zero padding (the median of w^2 values is one of them: exact);
//   4. per column, the smallest k attaining the filtered maximum;
//   5. the longest strictly increasing subsequence of the pairs (c[j], -j), as generate_lis builds it;
//   6. start[c] = j for every pair of that path, other tokens take the previous token's start (token 0: 0).
// Every step is a comparison or a sum in a fixed order, so the start bins equal a float64 restatement bit for bit.
#include "common.cuh"

namespace sb {

constexpr int TS_THREADS = 256;

// the m-th smallest (m = (W*W-1)/2) of the window: the value v[i] with #{v < v[i]} <= m < #{v <= v[i]}; fully unrolled
// so that the window stays in registers
template <int W>
__device__ __forceinline__ double ts_median(const double* __restrict__ A, int n, int F, int k, int j) {
  constexpr int N = W * W, m = (W * W - 1) / 2, R = W / 2;
  double v[N];
#pragma unroll
  for (int dk = 0; dk < W; ++dk)
#pragma unroll
    for (int dj = 0; dj < W; ++dj) {
      const int kk = k + dk - R, jj = j + dj - R;
      v[dk * W + dj] = (kk >= 0 && kk < n && jj >= 0 && jj < F) ? A[(long long)kk * F + jj] : 0.0;
    }
  double med = 0.0;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    int lt = 0, le = 0;
#pragma unroll
    for (int q = 0; q < N; ++q) {
      lt += v[q] < v[i];
      le += v[q] <= v[i];
    }
    if (lt <= m && m < le) med = v[i];
  }
  return med;
}

template <int W>
__global__ void __launch_bounds__(TS_THREADS, 1) token_timestamps_kernel(const float* __restrict__ hist, int rows, int s_enc,
                                                                      const int* __restrict__ slots, int slots_ld,
                                                                      const int* __restrict__ n_tok, const int* __restrict__ enc_lens,
                                                                      int prefix_len, double* __restrict__ scratch,
                                                                      long long scratch_ld, int* __restrict__ starts, int starts_ld) {
  extern __shared__ int ts_sm[];  // c [F], L [F], prev [F]
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = n_tok[b];
  const int len = enc_lens ? min(enc_lens[b], s_enc) : s_enc;
  const int F = len - 2;
  if (n <= 0 || F < 1 || n > starts_ld || prefix_len - 1 + n > slots_ld || (long long)n * F > scratch_ld) return;
  double* A = scratch + (long long)b * scratch_ld;
  const int* sl = slots + (long long)b * slots_ld;
  int* st = starts + (long long)b * starts_ld;
  // 1-2: gather along the winner's slots, normalise the columns
  for (int j = threadIdx.x; j < F; j += TS_THREADS) {
    double s = 0.0;
    for (int k = 0; k < n; ++k) {
      const int t = prefix_len - 1 + k;
      const double v = (double)hist[((long long)t * rows + sl[t]) * s_enc + 1 + j];
      A[(long long)k * F + j] = v;
      s += v;
    }
    for (int k = 0; k < n; ++k) A[(long long)k * F + j] = s != 0.0 ? A[(long long)k * F + j] / s : 0.0;
  }
  for (int k = threadIdx.x; k < n; k += TS_THREADS) st[k] = -1;
  __syncthreads();
  // 3-4: median filter and the first maximum of every column
  int* c = ts_sm;
  int* L = c + F;
  int* prev = L + F;
  for (int j = threadIdx.x; j < F; j += TS_THREADS) {
    double best = -INFINITY;  // the filtered values are >= 0
    int bk = 0;
    for (int k = 0; k < n; ++k) {
      const double v = ts_median<W>(A, n, F, k, j);
      if (v > best) { best = v; bk = k; }
    }
    c[j] = bk;
  }
  __syncthreads();
  if (warp != 0) return;
  // 5: for j < i, (c[j], -j) < (c[i], -i) exactly when c[j] < c[i].  L[i] = 1 + the largest L[j] over those j, prev[i] the
  // first j attaining it (generate_lis updates on strict improvement only), i when there is none.
  for (int i = 0; i < F; ++i) {
    const int ci = c[i];
    int bl = 0, bj = i;
    for (int j = lane; j < i; j += 32)
      if (c[j] < ci && L[j] > bl) { bl = L[j]; bj = j; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int ol = __shfl_xor_sync(0xffffffffu, bl, o), oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ol > bl || (ol == bl && oj < bj)) { bl = ol; bj = oj; }
    }
    if (lane == 0) {
      L[i] = bl + 1;
      prev[i] = bl > 0 ? bj : i;
    }
    __syncwarp();
  }
  if (lane != 0) return;
  // the path ends at the first i with the largest L
  int idx = 0;
  for (int i = 1; i < F; ++i)
    if (L[i] > L[idx]) idx = i;
  // 6: starts along the path, then carried forward
  st[c[idx]] = idx;
  while (prev[idx] != idx) {
    idx = prev[idx];
    st[c[idx]] = idx;
  }
  int last = 0;
  for (int k = 0; k < n; ++k) {
    if (st[k] < 0) st[k] = last;
    last = st[k];
  }
}

template <int W>
static int launch_timestamps(const float* hist, int rows, int s_enc, const int* slots, int slots_ld, const int* n_tok,
                             const int* enc_lens, int prefix_len, int batch, double* scratch, long long scratch_ld, int* starts,
                             int starts_ld, cudaStream_t stream) {
  const int F_max = s_enc - 2;
  const size_t smem = (size_t)3 * F_max * sizeof(int);
  token_timestamps_kernel<W><<<batch, TS_THREADS, smem, stream>>>(hist, rows, s_enc, slots, slots_ld, n_tok, enc_lens, prefix_len,
                                                                   scratch, scratch_ld, starts, starts_ld);
  SB_LAUNCH_OK();
  return SB_OK;
}

}  // namespace sb

extern "C" int sb_token_timestamps(const float* hist, int32_t rows, int32_t s_enc, const int32_t* slots, int32_t slots_ld,
                                   const int32_t* n_tok, const int32_t* enc_lens, int32_t prefix_len, int32_t batch,
                                   int32_t width, double* scratch, int64_t scratch_ld, int32_t* starts, int32_t starts_ld,
                                   sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(hist && slots && n_tok && scratch && starts && rows > 0 && batch > 0 && s_enc > 0 && prefix_len >= 1 &&
                 slots_ld > 0 && scratch_ld > 0 && starts_ld > 0,
             SB_EINVAL, "sb_token_timestamps: bad args");
  SB_REQUIRE(width >= 1 && width % 2 == 1, SB_EINVAL, "sb_token_timestamps: the filter width must be odd and >= 1");
  SB_REQUIRE(width <= SB_TS_MAX_WIDTH, SB_ENOSUP, "sb_token_timestamps: filter width %d above %d", width, SB_TS_MAX_WIDTH);
  SB_REQUIRE(s_enc - 2 <= SB_TS_MAX_FRAMES, SB_ENOSUP, "sb_token_timestamps: %d encoder frames above %d", s_enc - 2,
             SB_TS_MAX_FRAMES);
  if (s_enc < 3) return SB_OK;  // F < 1 on every row: nothing to write
  const cudaStream_t st = (cudaStream_t)stream;
  switch (width) {
    case 1: return launch_timestamps<1>(hist, rows, s_enc, slots, slots_ld, n_tok, enc_lens, prefix_len, batch, scratch, scratch_ld, starts, starts_ld, st);
    case 3: return launch_timestamps<3>(hist, rows, s_enc, slots, slots_ld, n_tok, enc_lens, prefix_len, batch, scratch, scratch_ld, starts, starts_ld, st);
    case 5: return launch_timestamps<5>(hist, rows, s_enc, slots, slots_ld, n_tok, enc_lens, prefix_len, batch, scratch, scratch_ld, starts, starts_ld, st);
    default: return launch_timestamps<7>(hist, rows, s_enc, slots, slots_ld, n_tok, enc_lens, prefix_len, batch, scratch, scratch_ld, starts, starts_ld, st);
  }
}
