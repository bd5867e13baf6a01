// Device versions of the NAR text-to-unit frontend glue.  The reference does this with Python loops and .item()
// syncs (models/unity/nar_decoder_frontend.py:130-259, length_regulator.py:24-39); at 200 utt/s those loops would
// dominate, so subword->char expansion, duration rounding and hard upsampling are small kernels here.
#include "common.cuh"

namespace sb {

// one CTA per sentence; the subword loop is sequential (<= a few hundred items)
__global__ void text_to_chars_kernel(const int* __restrict__ text_seqs, int L, const uint8_t* __restrict__ tok_len,
                                     const uint8_t* __restrict__ tok_flags, const int* __restrict__ tok_chars, int max_chars,
                                     int pad_idx, int unk_idx, int eos_idx, int* __restrict__ char_lens,
                                     int* __restrict__ char_seqs, int max_c, int* __restrict__ char_seq_lens) {
  const int b = blockIdx.x;
  const int* ts = text_seqs + (long long)b * L;
  int* cl = char_lens + (long long)b * L;
  int* cs = char_seqs + (long long)b * max_c;
  for (int i = threadIdx.x; i < max_c; i += blockDim.x) cs[i] = pad_idx;
  for (int i = threadIdx.x; i < L; i += blockDim.x) cl[i] = 0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  // TagManager.preprocess_text_seqs: drop the 2 prefix tokens, EOS -> PAD (nar_decoder_frontend.py:35-42)
  const int n = L - 2;
  auto tokat = [&](int i) { int t = ts[2 + i]; return t == eos_idx ? pad_idx : t; };
  int n_sub = 0;  // subword_lens = text_seqs.ne(pad).sum()  (a count, as in the reference)
  for (int i = 0; i < n; ++i) n_sub += (tokat(i) != pad_idx);
  int total = 0;
  bool stopped = false;
  for (int i = 0; i < n_sub; ++i) {
    const int t = tokat(i);
    // char ids (get_char_seqs :227-259) are appended for every one of the first n_sub subwords
    if (t == unk_idx) {
      if (total < max_c) cs[total] = unk_idx;
      total += 1;
    } else {
      const int len = tok_len[t];
      for (int c = 0; c < len; ++c)
        if (total + c < max_c) cs[total + c] = tok_chars[(long long)t * max_chars + c];
      total += len;
    }
    // char lengths (count_character_length_in_subword :158-225): the loop breaks at the first PAD
    if (stopped) continue;
    if (t == pad_idx) { stopped = true; continue; }
    int len;
    if (t == unk_idx) {
      len = 1;
    } else {
      len = tok_len[t];
      const bool nss_i = (i < n_sub - 1) && (tok_flags[tokat(i + 1)] & 2);
      const bool punc_i = tok_flags[t] & 1;
      if (punc_i && nss_i) len += 1;
      else if (i > 0 && (tok_flags[tokat(i - 1)] & 1) && (tok_flags[t] & 2)) len -= 1;
    }
    cl[1 + i] = len;  // postprocess_dur_or_len pads one zero on each side (:44-50)
  }
  char_seq_lens[b] = total;
}

// y[b][u] = x[b][src(u)] (+ alpha*pos[u]) (+ emb[ids[b][u]]*emb_scale); src from an in-block scan of the durations
__global__ void __launch_bounds__(256) upsample_add_kernel(const elem_t* __restrict__ x, int x_rows, int x_halo, int S,
                                                           const int* __restrict__ dur, elem_t* __restrict__ y, int y_rows,
                                                           int y_halo, int U, int dim, const float* __restrict__ pos,
                                                           const float* __restrict__ alpha, const elem_t* __restrict__ emb,
                                                           const int* __restrict__ ids, int ids_ld, float emb_scale,
                                                           int* __restrict__ out_lens) {
  extern __shared__ int cum[];  // [S] inclusive prefix sums
  const int b = blockIdx.y;
  const int* d = dur + (long long)b * S;
  // block scan (S is small: <= a few thousand)
  __shared__ int warp_tot[8];
  int carry = 0;
  for (int base = 0; base < S; base += 256) {
    int i = base + threadIdx.x;
    int v = i < S ? d[i] : 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += n;
    }
    if (lane == 31) warp_tot[warp] = v;
    __syncthreads();
    int off = 0;
    for (int w = 0; w < warp; ++w) off += warp_tot[w];
    int tot = 0;
    for (int w = 0; w < 8; ++w) tot += warp_tot[w];
    if (i < S) cum[i] = carry + off + v;
    carry += tot;
    __syncthreads();
  }
  const int total = carry;
  if (blockIdx.x == 0 && threadIdx.x == 0 && out_lens != nullptr) out_lens[b] = total;
  const float a = alpha ? alpha[0] : 0.f;
  const int u0 = blockIdx.x * 16;
  for (int uu = 0; uu < 16; ++uu) {
    const int u = u0 + uu;
    if (u >= U) break;
    int src = -1;
    if (u < total) {  // first index with cum > u
      int lo = 0, hi = S - 1;
      while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (cum[mid] > u) hi = mid; else lo = mid + 1;
      }
      src = lo;
    }
    const elem_t* xp = src >= 0 ? x + ((long long)b * x_rows + x_halo + src) * dim : nullptr;
    const elem_t* ep = emb ? emb + (long long)ids[(long long)b * ids_ld + u] * dim : nullptr;
    const float* pp = pos ? pos + (long long)u * dim : nullptr;
    elem_t* yp = y + ((long long)b * y_rows + y_halo + u) * dim;
    for (int c = threadIdx.x * 2; c < dim; c += 512) {
      float v0 = 0.f, v1 = 0.f;
      if (xp) { float2 f = __half22float2(*reinterpret_cast<const __half2*>(xp + c)); v0 = f.x; v1 = f.y; }
      // the reference adds in model precision: seqs (+)= alpha*pos (+ emb*scale); mirror the association order
      float p0 = 0.f, p1 = 0.f;
      // rows past the upsampled length stay zero (the reference leaves pos/emb garbage there, but every consumer
      // masks those rows; zero rows double as the conv padding mask of the next module)
      if (pp && xp) { p0 = a * pp[c]; p1 = a * pp[c + 1]; }
      if (ep && xp) { float2 f = __half22float2(*reinterpret_cast<const __half2*>(ep + c)); p0 += f.x * emb_scale; p1 += f.y * emb_scale; }
      *reinterpret_cast<__half2*>(yp + c) = __floats2half2_rn(v0 + p0, v1 + p1);
    }
  }
}

// one warp per (b, s): logd = hidden . w + bias; dur = clamp(round((exp(logd)-1)*factor), 1) masked
__global__ void durations_kernel(const elem_t* __restrict__ hidden, int rows_ld, int halo, const elem_t* __restrict__ w,
                                 float bias, int dim, const int* __restrict__ lens, int batch, int S, float factor,
                                 int* __restrict__ dur) {
  const int lane = threadIdx.x & 31;
  const long long idx = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= (long long)batch * S) return;
  const int b = (int)(idx / S), s = (int)(idx - (long long)b * S);
  const elem_t* hp = hidden + ((long long)b * rows_ld + halo + s) * dim;
  float acc = 0.f;
  for (int c = lane * 2; c < dim; c += 64) {
    float2 hv = __half22float2(*reinterpret_cast<const __half2*>(hp + c));
    float2 wv = __half22float2(*reinterpret_cast<const __half2*>(w + c));
    acc += hv.x * wv.x + hv.y * wv.y;
  }
  acc = warp_sum(acc) + bias;
  if (lane == 0) {
    const float logd = acc;
    // float -> s64 saturates; durations past INT32_MAX are clamped to it rather than wrapped to their low 32 bits, so
    // that the callers' length checks see them as too long
    long long d = (long long)rintf((expf(logd) - 1.f) * factor);
    if (d < 1) d = 1;
    if (lens != nullptr && s >= lens[b]) d = 0;
    dur[idx] = (int)min(d, (long long)INT_MAX);
  }
}

// one CTA per (b, u) row: argmax over vocab (first max wins) + UnitTokenDecoder transform
__global__ void __launch_bounds__(256) unit_argmax_kernel(const float* __restrict__ logits, long long ld, int rows_per_seq,
                                                          int halo, int U, int vocab, const int* __restrict__ lens, int pad_idx,
                                                          int eos_idx, int* __restrict__ units) {
  const int u = blockIdx.x, b = blockIdx.y;
  int tok;
  if (lens != nullptr && u >= lens[b]) {
    tok = pad_idx;  // apply_padding_mask(unit_seqs, mask, pad_idx) generator.py:348-350
  } else {
    const float* row = logits + ((long long)b * rows_per_seq + halo + u) * ld;
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < vocab; i += blockDim.x) {
      float v = row[i];
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    __shared__ float sv[8];
    __shared__ int si[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
      int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (v2 > bv || (v2 == bv && i2 < bi)) { bv = v2; bi = i2; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    bv = sv[0]; bi = si[0];
    for (int w = 1; w < 8; ++w)
      if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
    tok = bi;
  }
  if (threadIdx.x == 0) {
    // UnitTokenDecoder (NAR): eos->pad, pad->pad+4, then -4  (unit_tokenizer.py:231-241)
    if (tok == eos_idx) tok = pad_idx;
    if (tok == pad_idx) tok = pad_idx + 4;
    units[(long long)b * U + u] = tok - 4;
  }
}

}  // namespace sb

extern "C" int sb_text_to_chars(const int32_t* text_seqs, int32_t L, int32_t batch, const uint8_t* tok_len,
                                const uint8_t* tok_flags, const int32_t* tok_chars, int32_t max_chars, int32_t pad_idx,
                                int32_t unk_idx, int32_t eos_idx, int32_t* char_lens, int32_t* char_seqs, int32_t max_c,
                                int32_t* char_seq_lens, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(text_seqs && tok_len && tok_flags && tok_chars && char_lens && char_seqs && char_seq_lens && L >= 2 && batch > 0,
             SB_EINVAL, "sb_text_to_chars: bad args");
  text_to_chars_kernel<<<batch, 128, 0, (cudaStream_t)stream>>>(text_seqs, L, tok_len, tok_flags, tok_chars, max_chars, pad_idx,
                                                                unk_idx, eos_idx, char_lens, char_seqs, max_c, char_seq_lens);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_upsample_add(const void* x, int32_t x_rows, int32_t x_halo, int32_t S, const int32_t* dur, void* y,
                               int32_t y_rows, int32_t y_halo, int32_t U, int32_t batch, int32_t dim, const void* pos_table,
                               const float* alpha, const void* emb, const int32_t* ids, int32_t ids_ld, float emb_scale,
                               int32_t* out_lens, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(x && dur && y && S > 0 && U > 0 && batch > 0 && dim % 2 == 0, SB_EINVAL, "sb_upsample_add: bad args");
  SB_REQUIRE((size_t)S * 4 <= 40 * 1024, SB_ENOSUP, "sb_upsample_add: S=%d too large", S);
  dim3 grid((U + 15) / 16, batch);
  upsample_add_kernel<<<grid, 256, (size_t)S * 4, (cudaStream_t)stream>>>((const elem_t*)x, x_rows, x_halo, S, dur, (elem_t*)y,
                                                                         y_rows, y_halo, U, dim, (const float*)pos_table, alpha,
                                                                         (const elem_t*)emb, ids, ids_ld, emb_scale, out_lens);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_durations(const void* hidden, int32_t rows_ld, int32_t halo, const void* proj_w, float proj_b, int32_t dim,
                            const int32_t* lens, int32_t batch, int32_t S, float factor, int32_t* dur, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(hidden && proj_w && dur && batch > 0 && S > 0 && dim % 2 == 0, SB_EINVAL, "sb_durations: bad args");
  long long rows = (long long)batch * S;
  durations_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const elem_t*)hidden, rows_ld, halo,
                                                                               (const elem_t*)proj_w, proj_b, dim, lens, batch, S,
                                                                               factor, dur);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_unit_argmax(const float* logits, int64_t ld, int32_t rows_per_seq, int32_t halo, int32_t U, int32_t batch,
                              int32_t vocab, const int32_t* lens, int32_t pad_idx, int32_t eos_idx, int32_t* units,
                              sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(logits && units && U > 0 && batch > 0 && vocab > 0, SB_EINVAL, "sb_unit_argmax: bad args");
  unit_argmax_kernel<<<dim3(U, batch), 256, 0, (cudaStream_t)stream>>>(logits, ld, rows_per_seq, halo, U, vocab, lens, pad_idx,
                                                                      eos_idx, units);
  SB_LAUNCH_OK();
  return SB_OK;
}
