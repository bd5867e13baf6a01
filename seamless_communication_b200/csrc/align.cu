// UnitY2 forced aligner (models/aligner/model.py:146-277): the distance log-softmax and the monotonic alignment search.
//
// sb_align_lprob never forms the (B, T_feat, T_text, dim) difference tensor the reference builds for torch.norm: a CTA owns
// 64 frames of one row and walks the row's tokens in tiles of 32, accumulating sum_c (f - t)^2 in fp32 from shared-memory
// tiles of 32 channels (4 frames x 2 tokens per thread).  Direct differences, not |f|^2 + |t|^2 - 2 f.t: the expanded form
// cancels exactly at the best-matching token, where f ~ t.  Scores go to the output as they are made, with an online
// (max, sum exp) per frame; a second pass over the same values (each thread re-reads what it wrote) subtracts the
// log-sum-exp.  Every output element's arithmetic depends only on its own row, so a row gives the same bits in any batch.
//
// sb_monotonic_align runs the dynamic programme of _monotonic_alignment_search with one warp per row: lane l owns the
// contiguous rows [l*chunk, (l+1)*chunk) of Q, kept in shared memory interleaved by lane (conflict-free), and updates them
// column by column in descending order, so the only value crossing lanes per column is the neighbour's last Q of the
// previous column (one shuffle, no barrier).  The comparison that selects max(Q[i-1][j-1], Q[i][j-1]) is the backtrack's
// decision bit of column j-1; the bits are gathered 32 columns to a word and stored, and lane 0 walks them back.
#include "common.cuh"

namespace sb {

constexpr int AL_TJ = 64, AL_TI = 32, AL_TC = 32;  // frames x tokens per CTA tile, channels per shared-memory chunk
constexpr int MAS_MAX_TEXT = 8192;
constexpr int MAS_PRE = 8;  // rows per lane whose next-column log-probabilities are loaded one column ahead

__global__ void __launch_bounds__(256) align_lprob_kernel(const float* __restrict__ f, long long f_ld, int f_rows, int f_halo,
                                                          const int* __restrict__ feat_lens, const float* __restrict__ t,
                                                          long long t_ld, int t_rows, int t_halo, const int* __restrict__ text_lens,
                                                          int dim, int T_feat, int T_text, float temperature,
                                                          float* __restrict__ out, long long out_ld) {
  // Row-major tiles ([frame][channel], [token][channel]): a warp stores 32 consecutive channels of one row (no bank
  // conflict) and the compute loop reads 4 channels per 16-byte load.  The 36-float row stride keeps those loads aligned,
  // and with tokens tx and tx + 16 per thread the 8 lanes of each 16-byte load phase hit 8 distinct bank quads.
  __shared__ __align__(16) float fs[AL_TJ][AL_TC + 4];
  __shared__ __align__(16) float ts[AL_TI][AL_TC + 4];
  const int b = blockIdx.y, j0 = blockIdx.x * AL_TJ, tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // tokens tx, tx + 16 and frames 4ty .. 4ty+3 of the tile
  const int F = min(feat_lens[b], T_feat), N = min(text_lens[b], T_text);
  float* ob = out + (long long)b * T_feat * out_ld;
  if (j0 >= F || N <= 0) {  // nothing of this tile is a valid frame: padding rows are 0
    for (long long e = tid; e < (long long)AL_TJ * T_text; e += blockDim.x) {
      const int j = j0 + (int)(e / T_text), i = (int)(e % T_text);
      if (j < T_feat) ob[(long long)j * out_ld + i] = 0.f;
    }
    return;
  }
  const float* fb = f + ((long long)b * f_rows + f_halo) * f_ld;
  const float* tb = t + ((long long)b * t_rows + t_halo) * t_ld;
  float m[4], s[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) { m[r] = -INFINITY; s[r] = 0.f; }
  const int n_tiles = (N + AL_TI - 1) / AL_TI;
  for (int it = 0; it < n_tiles; ++it) {
    const int i0 = it * AL_TI;
    float acc[4][2] = {};
    for (int c0 = 0; c0 < dim; c0 += AL_TC) {
      const int cl = tid & 31, c = c0 + cl;
      for (int r = tid >> 5; r < AL_TJ; r += 8) {
        const int j = j0 + r;
        fs[r][cl] = (j < F && c < dim) ? fb[(long long)j * f_ld + c] : 0.f;
      }
      for (int r = tid >> 5; r < AL_TI; r += 8) {
        const int i = i0 + r;
        ts[r][cl] = (i < N && c < dim) ? tb[(long long)i * t_ld + c] : 0.f;
      }
      __syncthreads();
#pragma unroll 2
      for (int cc = 0; cc < AL_TC; cc += 4) {
        float fv[4][4], tv[2][4];
#pragma unroll
        for (int r = 0; r < 4; ++r) *reinterpret_cast<float4*>(fv[r]) = *reinterpret_cast<const float4*>(&fs[4 * ty + r][cc]);
#pragma unroll
        for (int q = 0; q < 2; ++q) *reinterpret_cast<float4*>(tv[q]) = *reinterpret_cast<const float4*>(&ts[tx + 16 * q][cc]);
#pragma unroll
        for (int k = 0; k < 4; ++k)  // channels in ascending order, as before the 16-byte loads
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const float d = fv[r][k] - tv[q][k];
              acc[r][q] = fmaf(d, d, acc[r][q]);
            }
      }
      __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int j = j0 + 4 * ty + r;
      float sc[2], tmax = -INFINITY;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int i = i0 + tx + 16 * q;
        sc[q] = i < N ? -temperature * sqrtf(acc[r][q]) : -INFINITY;
        tmax = fmaxf(tmax, sc[q]);
        if (j < F && i < T_text) ob[(long long)j * out_ld + i] = sc[q];
      }
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
      float ts_ = 0.f;
#pragma unroll
      for (int q = 0; q < 2; ++q) ts_ += sc[q] == -INFINITY ? 0.f : expf(sc[q] - tmax);
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) ts_ += __shfl_xor_sync(0xffffffffu, ts_, o);
      // every tile holds at least one token i < N, so tmax is finite
      const float mn = fmaxf(m[r], tmax);
      s[r] = s[r] * expf(m[r] - mn) + ts_ * expf(tmax - mn);
      m[r] = mn;
    }
  }
  // second pass: thread tx re-reads the tokens i = tx (mod 16) it wrote above
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int j = j0 + 4 * ty + r;
    if (j >= T_feat) continue;
    float* orow = ob + (long long)j * out_ld;
    if (j >= F) {
      for (int i = tx; i < T_text; i += 16) orow[i] = 0.f;
      continue;
    }
    const float lse = m[r] + logf(s[r]);
    for (int i = tx; i < T_text; i += 16) orow[i] = i < N ? orow[i] - lse : -INFINITY;
  }
}

// One warp per row.  Q[i] of lane l's k-th row (i = l*chunk + k) lives at qs[k*32 + l]; acc[k*32 + l] gathers its decision
// bits for the current word of 32 columns.
__global__ void __launch_bounds__(32) monotonic_align_kernel(const float* __restrict__ lp, long long lp_ld, int T_feat,
                                                             int T_text, const int* __restrict__ feat_lens,
                                                             const int* __restrict__ text_lens, int chunk,
                                                             uint32_t* __restrict__ bits, int words, int* __restrict__ dur,
                                                             int* __restrict__ path) {
  extern __shared__ double qs[];
  uint32_t* acc = reinterpret_cast<uint32_t*>(qs + (size_t)chunk * 32);
  const int b = blockIdx.x, lane = threadIdx.x;
  const int F = min(feat_lens[b], T_feat), N = min(text_lens[b], T_text);
  int* db = dur + (long long)b * T_text;
  for (int i = lane; i < T_text; i += 32) db[i] = 0;
  if (path != nullptr)
    for (int j = lane; j < T_feat; j += 32) path[(long long)b * T_feat + j] = -1;
  if (F <= 0 || N <= 0) return;
  const float* lb = lp + (long long)b * T_feat * lp_ld;
  uint32_t* bb = bits + (long long)b * T_text * words;
  const int i0 = lane * chunk;
  const int kn = max(0, min(chunk, N - i0));  // rows this lane owns
  for (int k = 0; k < chunk; ++k) {
    qs[k * 32 + lane] = -INFINITY;
    acc[k * 32 + lane] = 0u;
  }
  if (lane == 0) qs[0] = (double)lb[0];
  float pre[MAS_PRE];
#pragma unroll
  for (int k = 0; k < MAS_PRE; ++k) pre[k] = (F > 1 && k < kn && i0 + k <= 1) ? lb[lp_ld + i0 + k] : 0.f;
  for (int j = 1; j < F; ++j) {
    const float* col = lb + (long long)j * lp_ld;
    const double last_old = qs[(chunk - 1) * 32 + lane];
    const double prev = __shfl_up_sync(0xffffffffu, last_old, 1);  // Q[i0 - 1][j - 1]
    const int khi = min(kn - 1, j - i0);                           // rows i <= min(j, N - 1)
    float cur[MAS_PRE];
#pragma unroll
    for (int k = 0; k < MAS_PRE; ++k) cur[k] = pre[k];
    if (j + 1 < F) {
      const float* nxt = col + lp_ld;
#pragma unroll
      for (int k = 0; k < MAS_PRE; ++k) pre[k] = (k < kn && i0 + k <= j + 1) ? nxt[i0 + k] : 0.f;
    }
    const uint32_t bit = 1u << ((j - 1) & 31);
    for (int k = khi; k >= 0; --k) {
      const int i = i0 + k;
      double v;
      float l = 0.f;
      if (k < MAS_PRE) {
#pragma unroll
        for (int q = 0; q < MAS_PRE; ++q)
          if (q == k) l = cur[q];
      } else {
        l = col[i];
      }
      const double qi = qs[k * 32 + lane];
      if (i == 0) {
        v = qi + (double)l;
      } else {
        const double qm = k > 0 ? qs[(k - 1) * 32 + lane] : prev;
        const bool up = qm >= qi;  // backtrack decision of column j - 1: Q[i-1][j-1] >= Q[i][j-1]
        if (up) acc[k * 32 + lane] |= bit;
        v = (up ? qm : qi) + (double)l;
      }
      qs[k * 32 + lane] = v;
    }
    if (((j - 1) & 31) == 31) {
      const int w = (j - 1) >> 5;
      for (int k = 0; k < kn; ++k) {
        bb[(long long)(i0 + k) * words + w] = acc[k * 32 + lane];
        acc[k * 32 + lane] = 0u;
      }
    }
  }
  if (F >= 2 && ((F - 2) & 31) != 31) {
    const int w = (F - 2) >> 5;
    for (int k = 0; k < kn; ++k) bb[(long long)(i0 + k) * words + w] = acc[k * 32 + lane];
  }
  __syncwarp();
  if (lane != 0) return;
  // A[F-1] = N-1; A[j] = A[j+1] - 1 when Q[A[j+1]-1][j] >= Q[A[j+1]][j] (always so when A[j+1] > j: Q[A[j+1]][j] is -inf
  // there and no bit is stored), else A[j+1]; 0 once A[j+1] == 0.  Durations are the run lengths of A.
  int a = N - 1, run = 1;
  long long cached = -1;
  uint32_t word = 0;
  if (path != nullptr) path[(long long)b * T_feat + F - 1] = a;
  for (int j = F - 2; j >= 0; --j) {
    int na = a;
    if (a > 0) {
      if (a > j) {
        na = a - 1;
      } else {
        const long long widx = (long long)a * words + (j >> 5);
        if (widx != cached) { word = bb[widx]; cached = widx; }
        if ((word >> (j & 31)) & 1u) na = a - 1;
      }
    }
    if (na != a) {
      db[a] = run;
      run = 0;
      a = na;
    }
    ++run;
    if (path != nullptr) path[(long long)b * T_feat + j] = a;
  }
  db[a] = run;
}

}  // namespace sb

extern "C" int sb_align_lprob(const float* f, int64_t f_ld, int32_t f_rows, int32_t f_halo, const int32_t* feat_lens, const float* t,
                              int64_t t_ld, int32_t t_rows, int32_t t_halo, const int32_t* text_lens, int32_t dim, int32_t batch,
                              int32_t T_feat, int32_t T_text, float temperature, float* out, int64_t out_ld, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(f && t && feat_lens && text_lens && out && dim > 0 && batch > 0 && T_feat > 0 && T_text > 0, SB_EINVAL,
             "sb_align_lprob: bad args");
  SB_REQUIRE(batch <= 65535 && out_ld >= T_text && f_ld >= dim && t_ld >= dim, SB_EINVAL,
             "sb_align_lprob: batch above 65535 or a row stride below its width");
  dim3 grid((T_feat + AL_TJ - 1) / AL_TJ, batch);
  align_lprob_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(f, (long long)f_ld, f_rows, f_halo, feat_lens, t, (long long)t_ld, t_rows,
                                                             t_halo, text_lens, dim, T_feat, T_text, temperature, out,
                                                             (long long)out_ld);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_monotonic_align(const float* lprob, int64_t lp_ld, int32_t batch, int32_t T_feat, int32_t T_text,
                                  const int32_t* feat_lens, const int32_t* text_lens, uint32_t* bits, int32_t* durations,
                                  int32_t* path, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(lprob && feat_lens && text_lens && bits && durations && batch > 0 && T_feat > 0 && T_text > 0 && lp_ld >= T_text,
             SB_EINVAL, "sb_monotonic_align: bad args");
  SB_REQUIRE(T_text <= MAS_MAX_TEXT, SB_ENOSUP, "sb_monotonic_align: T_text %d exceeds %d", T_text, MAS_MAX_TEXT);
  const int chunk = (T_text + 31) / 32;
  const size_t smem = (size_t)chunk * 32 * (sizeof(double) + sizeof(uint32_t));
  SB_CUDA_OK(cudaFuncSetAttribute(monotonic_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  monotonic_align_kernel<<<batch, 32, smem, (cudaStream_t)stream>>>(lprob, (long long)lp_ld, T_feat, T_text, feat_lens, text_lens,
                                                                     chunk, bits, (T_feat + 31) / 32, durations, path);
  SB_LAUNCH_OK();
  return SB_OK;
}
