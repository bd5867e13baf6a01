/*
 * seamless_b200.h - C ABI of the H100-native SeamlessM4T-v2 S2ST hot path.
 *
 * Convention (SURVEY.md 8b): one `extern "C" int sb_<op>(...)` per module of the path, plain device pointers and
 * sizes, a CUDA stream, an int return code (0 = ok, otherwise a negative SB_E* code; sb_last_error() gives text).
 * Nothing here allocates device memory or synchronises; the caller owns every buffer.  This mirrors the reference's
 * own native convention of one `extern "C" <Module>_forward(model, prefix, tensors...)` per module
 * (ggml/examples/unity/fairseq2.h:153-250) loaded through ctypes (ggml/ggml.py:384-398).
 *
 * Activations are fp16, channels-last: a (B,T,C) tensor is a matrix of B*Tp rows by C columns where each sequence
 * owns Tp = T + halos rows ("sequence layout": data row t of sequence b lives at row b*Tp + PH + t; halo rows are
 * zero).  A dense tensor is the special case Tp = T, PH = 0.  Weights keep the reference's tensor layouts
 * (nn.Linear (out,in); Conv1d repacked once by the host to (out, k, in)).
 */
#ifndef SEAMLESS_B200_H_
#define SEAMLESS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* sb_stream_t; /* cudaStream_t */

enum {
  SB_OK = 0,
  SB_EINVAL = -1,  /* bad argument */
  SB_ECUDA = -2,   /* CUDA runtime / driver error */
  SB_ENOSUP = -3   /* shape not supported by the kernels */
};

enum { SB_ACT_NONE = 0, SB_ACT_RELU = 1, SB_ACT_SILU = 2, SB_ACT_LRELU = 3, SB_ACT_TANH = 4 };

const char* sb_last_error(void);
int sb_version(void);
/* number of kernels launched by this library since load (bench.py reports it as gpu_launches) */
int64_t sb_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_gemm - fused Linear / Conv1d-as-GEMM on Hopper tensor cores (TMA -> smem -> wgmma -> registers -> epilogue).
 *   acc[m, n] = sum_{tap, c} A[a_row0 + m + tap*dil, c] * W[n, tap*c_in + c]
 *   v   = act(acc + bias[n])            (glu: v[j] = (acc[2j]+b[2j]) * sigmoid(acc[2j+1]+b[2j+1]), N/2 outputs)
 *   out[q, n] = gamma * (alpha * v + res1[q, n] + res2[q, n]),  q = m + out_row0
 *   out2[q, n] = leaky_relu(out[q, n], out2_slope)                         (optional second output)
 *   rows q whose sequence position is outside [0, len) are written as zeros (when seq_rows > 0).
 * Replaces: fairseq2 Linear / torch Conv1d / ConvTranspose1d call sites of the path, e.g. Linear_forward
 * (ggml/examples/unity/fairseq2.cpp:251), ggml_conv_1d in ConvModule_forward (fairseq2.cpp:698-731),
 * Conv1dBlock.forward (models/unity/fft_decoder_layer.py:75-101), hifigan.py:114-121,180-196.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* a;       /* fp16 activations, row-major, row stride a_ld elements */
  int64_t a_rows;      /* rows addressable from `a` (TMA bound; reads outside are zero) */
  int64_t a_ld;        /* elements between rows (multiple of 8) */
  int32_t c_in;        /* channels per tap */
  int32_t taps;        /* 1 for Linear */
  int32_t dil;         /* row step between taps */
  int32_t a_row0;      /* window start of output row m=0 (may be negative) */
  const void* w;       /* fp16 [n][taps*c_in] */
  int32_t n;           /* output features before GLU */
  int32_t m;           /* output rows */
  const float* bias;   /* fp32 [n] or NULL */
  int32_t act;         /* SB_ACT_* */
  float act_slope;     /* leaky-relu slope */
  int32_t glu;         /* 1: pairs (2j,2j+1) -> a*sigmoid(b) */
  float alpha, gamma;
  const void* res1; int64_t res1_ld;
  const void* res2; int64_t res2_ld;
  void* out; int64_t out_ld; int32_t out_f32;
  void* out2; int64_t out2_ld; float out2_slope;
  int64_t out_row0;
  int32_t seq_rows;    /* Tp (0: no masking) */
  int32_t seq_halo;    /* PH */
  int32_t seq_len;     /* T when seq_lens == NULL */
  const int32_t* seq_lens; /* per-sequence valid lengths or NULL */
  const void* prefetch;    /* optional: a device range (e.g. the next layer's weights) to pull into L2 while this GEMM runs */
  int64_t prefetch_bytes;
  float* tile_stats;       /* optional fp32 [ceil(n/128)][m][2]: per output row and 128-column tile (max, sum exp(x - max)) of
                              the stored values - log-softmax statistics fused into the projection (sb_logits_topk_tiles) */
} sb_gemm_t;

int sb_gemm(const sb_gemm_t* g, sb_stream_t stream);
/* split-K variant for skinny-M / large-K products (the decoder's residual GEMMs at M = batch*beam rows): the K range is
 * cut into `splits` slices computed by different CTAs so every SM streams weights; slice z writes its raw fp32 partial
 * products to rows [z*slice_rows, z*slice_rows + m) of `partials` (row stride n; slice_rows a multiple of 128 enables
 * the TMA-store epilogue).  Only a/w/shape fields of `g` are used. */
int sb_gemm_splitk(const sb_gemm_t* g, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream);
/* The same products for at most 256 rows in TRANSPOSED form on wgmma (decode_gemm.cu): a 128-feature weight tile is the
 * MMA A operand and all rows are the B operand, so a CTA reads its weights once and the activations once per k-block
 * (the row-major kernel re-reads a 128-row activation tile for every 64 features and is L2 -> SM bound at 160 rows).
 * partials != NULL: split-K mode, same output contract as sb_gemm_splitk (splits need not divide the k-blocks).
 * partials == NULL (splits must be 1): out = act(a . w^T + bias) in fp16, act in {none, relu}.  At splits that divide
 * the k-blocks the partials are bit-identical to sb_gemm_splitk's on the H100 (same k-blocks in the same m64 x k16
 * steps; tests/test_decode_gemm.py checks it), so the decoder step's outputs do not depend on the path. */
int sb_gemm_decode_supported(const sb_gemm_t* g, int32_t splits);
int sb_gemm_decode(const sb_gemm_t* g, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream);
/* consumer of the partials: x += bias + sum_z partial[z] (x fp16 [rows][dim], updated in place) and h = LayerNorm(x).
 * Fuses the reduction into the LayerNorm that follows every residual GEMM of a pre-LN decoder layer
 * (StandardTransformerDecoderLayer, fairseq2.cpp:979-1060). */
int sb_splitk_reduce_ln(const float* partials, int32_t splits, int32_t rows, int64_t slice_rows, int32_t dim,
                        const float* bias, void* x,
                        const float* ln_w, const float* ln_b, void* h, sb_stream_t stream);
/* same contract on CUDA cores (fp32 accumulate); a debugging cross-check, never used by the product path */
int sb_gemm_ref(const sb_gemm_t* g, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_fbank - WaveformToFbankConverter(num_mel_bins=80, waveform_scale=2**15, standardize=...) on device.
 * Replaces inference/translator.py:136-143,293 (fairseq2n knf path; arithmetic
 * ggml/examples/kaldi-native-fbank/csrc/feature-window.cc:76-232, feature-fbank.cc:73-120).
 *   wave  : fp32 [batch][wave_ld], num_samples[b] valid samples each
 *   out   : fp16 [batch][out_frames_ld][80]; frames beyond the utterance are zero (Collater pad_value 0)
 *   work  : fp32 [batch][out_frames_ld][80] scratch
 *   frames_out : int32 [batch] number of frames per utterance (may be NULL)
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_fbank(const float* wave, int64_t wave_ld, const int32_t* num_samples, int32_t batch, void* out,
             int32_t out_frames_ld, float* work, int32_t* frames_out, int32_t standardize, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_layernorm - y = LN(x (+ res)) * w + b over the last dim (eps 1e-5), fp16 io, fp32 statistics.
 * Rows are addressed in sequence layout on both sides; rows at positions >= len are written as zeros when
 * mask_out != 0.  res (optional) has x's layout and is added to x in fp32 before the statistics, without rounding;
 * sum_out (optional, used only with res) receives x + res rounded to fp16 in the OUT layout (out_rows / out_halo).
 * SB_ENOSUP unless dim is a multiple of 8 and at most 2048.  Replaces LayerNorm_forward (fairseq2.cpp:266).
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_layernorm(const void* x, const void* res, void* y, void* sum_out, const float* w, const float* b, int32_t dim,
                 int32_t batch, int32_t T, int32_t in_rows, int32_t in_halo, int32_t out_rows, int32_t out_halo,
                 const int32_t* lens, int32_t mask_out, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_attention - multi-head scaled dot-product attention, head_dim 64, fp16 io, fp32 softmax, flash-style.
 *   scores = (q.k^T + q.rel_k[clamp(j-i,-left,right)+left]) / 8, key mask j < kv_lens[b] (kv_lens NULL: j < sk);
 *   causal != 0 also masks j > i + sk - sq (aligned bottom-right: the last query row sees every key).
 *   A row with no admissible key (kv_lens[b] == 0, or a causal row i < sq - sk) is written as 0.
 * q/k/v/out pointers address row 0 of sequence 0 (sequence layout given by the x_rows / x_halo arguments; out uses q's),
 * x_ld = row stride.  Only rows [q_halo, q_halo + sq) x columns [0, heads*64) of each sequence of out are written.
 * SB_ENOSUP, before anything is launched: q_ld, k_ld or v_ld not a multiple of 8 elements, out_ld odd, or rel_k != NULL
 * with left + right + 1 > 80.
 * Replaces MultiheadAttention_forward (fairseq2.cpp:399-499) and ShawRelativePositionSDPA
 * (models/conformer_shaw/builder.py:127-146).
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_attention(const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, void* out,
                 int64_t out_ld, int32_t batch, int32_t heads, int32_t sq, int32_t sk, int32_t q_rows, int32_t q_halo,
                 int32_t kv_rows, int32_t kv_halo, const int32_t* kv_lens, int32_t causal, const void* rel_k,
                 int32_t rel_left, int32_t rel_right, sb_stream_t stream);
/* sb_attention_relpos - Transformer-XL relative-position self-attention of w2v-BERT v1 (RelativePositionSDPA, mirrored
 * fairseq2.cpp:605-696), same layouts and key mask as sb_attention, sq = sk = s, no causal mode:
 *   scores[i][j] = ((q_i + u) . k_j + (q_i + v) . R[s-1+j-i]) / 8
 * r: fp16 [2s-1][r_ld], head h in columns h*64..h*64+63 (R = r_proj(pos table rows n_ctx-s .. n_ctx+s-2)); u, v: fp32
 * [heads][64] or NULL (= 0); q + u and q + v are summed in fp32 and rounded once to fp16.  SB_ENOSUP for s > 4096 (the
 * relative position table covers distances up to 4095), before anything is launched.
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_attention_relpos(const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, void* out,
                        int64_t out_ld, int32_t batch, int32_t heads, int32_t s, int32_t q_rows, int32_t q_halo,
                        int32_t kv_rows, int32_t kv_halo, const int32_t* kv_lens, const void* r, int64_t r_ld,
                        const float* u, const float* v_bias, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_dwconv_ln_silu - Conformer conv module middle: causal depthwise Conv1d(k) -> LayerNorm(C) -> SiLU.
 * Replaces ConformerConvolution's depthwise_conv/layer_norm/activation (conformer_shaw/builder.py:148-156;
 * op order fairseq2.cpp:698-731 with the v2 causal + LayerNorm variant).  x,y dense (B,T,C) fp16; w [C][k] fp16.
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_dwconv_ln_silu(const void* x, void* y, const void* w, const float* ln_w, const float* ln_b, int32_t batch,
                      int32_t T, int32_t C, int32_t k, sb_stream_t stream);
/* sb_dwconv_bias_silu - the w2v-BERT v1 form: depthwise Conv1d(k = 31, pad 15 on both sides) -> + bias[c] -> SiLU, with
 * BatchNorm's scale already folded into w (fairseq2.cpp:698-731).  Frames outside [0, T) read as zero.  C % 64 == 0, C <= 1024. */
int sb_dwconv_bias_silu(const void* x, void* y, const void* w, const float* bias, int32_t batch, int32_t T, int32_t C,
                        int32_t k, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Text decoder step pieces (KV cache with beam-ancestor indirection instead of the reference's per-step
 * index_select copies, fairseq2.cpp:170-198).
 * ---------------------------------------------------------------------------------------------------------------- */
/* The step index of the incremental decoder lives in device memory (*step_ptr) so that ONE captured CUDA graph of a
 * decoder step can be replayed for every position; sb_step_advance increments it at the end of the graph.
 * x[r] = embed[tok[r]] * scale + pos[step]; tok = seqs[r*seq_ld + step]  (fairseq2.cpp:917-953); pos_table fp32. */
int sb_embed_step(const int32_t* seqs, int32_t seq_ld, const int32_t* step_ptr, const void* embed, const void* pos_table,
                  float scale, void* x, int32_t rows, int32_t dim, sb_stream_t stream);
int sb_step_advance(int32_t* step_ptr, sb_stream_t stream);
/* hist[*step_ptr] = h (bytes_per_step each): records the decoder output state of every search step */
int sb_store_step(const void* h, void* hist, const int32_t* step_ptr, int64_t bytes_per_step, sb_stream_t stream);
/* embeds a full (rows, L) id matrix (teacher-forced pass): x[(r*L+t)] = embed[ids[r*ids_ld+t]]*scale + pos[t] */
int sb_embed_seq(const int32_t* ids, int32_t ids_ld, int32_t L, const void* embed, const void* pos_table, float scale,
                 void* x, int32_t rows, int32_t dim, sb_stream_t stream);
/* self-attention of one new token per row against the cache.
 *   qkv: fp16 [rows][3*dim] (q|k|v of the new token); kcache/vcache: fp16 [max_len][rows][dim];
 *   anc: int32 [rows][anc_ld], anc[r][t] = cache slot holding position t of row r's history (t < step);
 *   the new k/v are stored to slot r at position `step`.  out: fp16 [rows][dim]. */
/* q|k|v of the new token come either as fp16 `qkv` or (qkv == NULL) as split-K partials of the qkv projection
 * ([splits][slice_rows][3*dim] fp32 + the fp32 projection bias), reduced on the fly. */
int sb_decode_self_attn(const void* qkv, const float* qkv_partials, int32_t splits, int64_t slice_rows,
                        const float* qkv_bias, void* kcache, void* vcache, const int32_t* anc, int32_t anc_ld,
                        const int32_t* step_ptr, int32_t max_len, void* out, int32_t rows, int32_t heads,
                        sb_stream_t stream);
/* cross-attention of one token per row against per-utterance static K/V: k/v fp16 [batch][s_enc][dim] (row stride
 * kv_ld), row r attends utterance r / beam. */
int sb_decode_cross_attn(const void* q, const float* q_partials, int32_t splits, int64_t slice_rows, const float* q_bias,
                         const void* k, const void* v, int64_t kv_ld, const int32_t* enc_lens, int32_t s_enc, void* out,
                         int32_t rows, int32_t beam, int32_t heads, sb_stream_t stream);
/* per row: log-softmax statistics and the top-K candidates of an fp32 logit row.
 *   cand_val [rows][K] = lprob, cand_idx [rows][K]; eos_lprob[rows] = lprob of eos; pad is never a candidate. */
int sb_logits_topk(const float* logits, int64_t ld, int32_t rows, int32_t vocab, int32_t pad_idx, int32_t eos_idx,
                   int32_t unk_idx, float unk_penalty, int32_t K, float* cand_val, int32_t* cand_idx, float* eos_lprob,
                   sb_stream_t stream);

/* Same contract as sb_logits_topk, for logits written by sb_gemm with `tile_stats`: the log-sum-exp comes from the tile
 * statistics and only the tiles whose maximum reaches the (K+2)-th largest tile maximum are read back (a lower bound of the
 * K-th best candidate even if PAD and UNK head two of them), i.e. ~K x 512 B per row instead of two passes over the row.
 * Replaces log_softmax + topk over the vocabulary (fairseq2.cpp:1463-1516) without the 164 MB round trips per step. */
int sb_logits_topk_tiles(const float* logits, int64_t ld, const float* tile_stats, int32_t rows, int32_t vocab, int32_t pad_idx,
                         int32_t eos_idx, int32_t unk_idx, float unk_penalty, int32_t K, float* cand_val, int32_t* cand_idx,
                         float* eos_lprob, sb_stream_t stream);

/* one beam-search step for every sentence (BeamSearchSeq2SeqGenerator step, mirrored fairseq2.cpp:1463-1594).
 * State (all device, int32/fp32):
 *   seqs [B*beam][max_len], scores [B*beam][max_len], anc [B*beam][max_len],
 *   fin_count [B], fin_score [B][beam], fin_len [B][beam], fin_seqs [B][beam][max_len], active [B] */
typedef struct {
  int32_t batch, beam, max_len, vocab, K;
  const int32_t* step_ptr; /* position being consumed; the new token goes to step+1 */
  int32_t prefix_len;      /* at step == prefix_len-1 only beam 0 of each sentence is a candidate source */
  int32_t eos_idx;
  int32_t min_len;     /* EOS forbidden while step < min_len */
  float len_penalty;
  const float* cand_val; const int32_t* cand_idx; const float* eos_lprob;
  int32_t* seqs; float* scores; int32_t* anc;  /* reordered in place */
  int32_t* fin_count; float* fin_score; int32_t* fin_len; int32_t* fin_seqs; int32_t* active;
  int32_t* fin_anc;    /* [B][beam][max_len] or NULL: per finished hypothesis, the cache slot of every position */
  int32_t* n_active;   /* [1] number of sentences still searching (written every step) */
  const int32_t* len_budget; /* [1] on the device or NULL: the search's length budget (<= max_len; EOS forced at step
                                budget-2, no step past budget-1), so one captured step serves every budget up to the
                                allocated max_len, which stays the row stride of the arrays above.  NULL: max_len */
} sb_beam_t;
int sb_beam_step(const sb_beam_t* p, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * sb_decoder_step - module-level entry: ONE persistent kernel for a whole incremental decoder step over `rows`
 * hypotheses (embedding frontend -> every pre-LN decoder layer with KV cache -> final LayerNorm).
 * Replaces: TransformerEmbeddingFrontend + StandardTransformerDecoder.forward with an IncrementalStateBag as driven by
 * UnitYX2TModel.decode (models/unity/model.py:233-252); C++ mirror StandardTransformerDecoderLayer_forward
 * (ggml/examples/unity/fairseq2.cpp:979-1094), TransformerEmbeddingFrontend_forward (:917-953).
 * Workspace convention of SURVEY 8(b): sb_decoder_plan_query() reports every size, the caller allocates, then
 * sb_decoder_plan_init() fills the POD launch descriptor (shapes, pointers and TMA descriptors travel as kernel
 * parameters; no device allocation, no copy) that sb_decoder_step() replays (graph-capturable: a memset node + one
 * kernel).  At most 32 layers.
 * Weights keep the reference layouts (Linear (out,in) fp16) but are STACKED into two tensors so that one TMA descriptor
 * serves all layers: w_dim_stack [layers][3*dim (q|k|v) + dim (self out) + dim (cross q) + dim (cross out) + ffn_dim
 * (FFN inner)][dim] and w_ffn_stack [layers][dim][ffn_dim] (FFN out); biases / LayerNorm fp32 per layer.
 * State per call: x (residual stream), h (= LN of x, at the end: the decoder output of this step), both [rows][dim].
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  /* biases of: self qkv, self out, cross q, cross out, FFN inner, FFN out */
  const float *qkv_b, *out_b, *cq_b, *co_b, *ffn1_b, *ffn2_b;
  const float *ca_ln_w, *ca_ln_b;     /* encoder_decoder_attn_layer_norm */
  const float *ffn_ln_w, *ffn_ln_b;   /* ffn_layer_norm */
  const float *next_ln_w, *next_ln_b; /* next layer's self_attn_layer_norm, or the decoder's final layer_norm */
  void *k_cache, *v_cache;            /* fp16 [rows (slots)][heads][max_len][64]: position `step` is written at slot = row */
  const void *cross_k, *cross_v;      /* fp16 [batch][heads][s_enc][64] static encoder K / V of this layer (sb_kv_heads_major) */
} sb_decoder_layer_t;

typedef struct {
  int32_t layers, dim, ffn_dim, heads, rows, beam, groups /* 0 = auto */, max_len, s_enc;
  const sb_decoder_layer_t* layer;    /* [layers] (host array) */
  const void *w_dim_stack, *w_ffn_stack; /* stacked fp16 weights, see above */
  const float *ln0_w, *ln0_b;         /* layer 0 self_attn_layer_norm */
  const void* embed;                  /* fp16 [vocab][dim] */
  const float* pos;                   /* fp32 [>= max_len][dim] sinusoid table (position index = step) */
  float embed_scale;
  const int32_t* seqs; int32_t seqs_ld;   /* token of row r at position *step_ptr: seqs[r*seqs_ld + step] */
  const int32_t* anc; int32_t anc_ld;     /* cache slot of row r at position t < step: anc[r*anc_ld + t] */
  const int32_t* step_ptr;
  const int32_t* enc_lens;            /* [batch] or NULL */
  void *x, *h, *att, *ffn_act;        /* fp16 [rows][dim] x3, [rows][ffn_dim] */
  float* part_qkv; int64_t part_qkv_floats;
  float* part; int64_t part_floats;
  void* hist;                         /* fp16 [max_len][rows][dim] or NULL: h of every step */
  uint32_t* counters; int64_t counters_len;
  uint64_t* timeline;                 /* NULL, or [groups][n_phases][8] ns stamps of CTA 0 (profiling) */
} sb_decoder_plan_desc_t;

typedef struct {
  int64_t part_qkv_floats, part_floats, counters_len;
  int32_t groups, rows_per_group, npad, ctas_per_group, stages, smem_bytes, n_phases;
  int32_t splits[6];                  /* split-K of qkv, out, cq, co, ffn1 (always 1), ffn2 */
} sb_decoder_plan_info_t;

typedef struct {
  uint32_t* counters; int64_t counters_len;
  int32_t grid, block, smem_bytes, cooperative, npad, reserved;
  uint64_t params[768];               /* opaque: the kernel's parameter block (shapes, pointers, 5 TMA descriptors) */
} sb_decoder_launch_t;

/* kv [batch*s_enc][ld] with K | V concatenated along the features (the output of the cross-attention k/v projection)
 * -> head-major k_out, v_out [batch][heads][s_enc][64]: the keys of one (utterance, head) become consecutive rows */
int sb_kv_heads_major(const void* kv, int64_t ld, int32_t batch, int32_t s_enc, int32_t heads, void* k_out, void* v_out,
                      sb_stream_t stream);
int sb_decoder_plan_query(int32_t layers, int32_t dim, int32_t ffn_dim, int32_t rows, int32_t beam, int32_t groups,
                          sb_decoder_plan_info_t* info);
int sb_decoder_plan_init(const sb_decoder_plan_desc_t* desc, sb_decoder_launch_t* launch);
int sb_decoder_step(const sb_decoder_launch_t* launch, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * NAR T2U frontend (models/unity/nar_decoder_frontend.py:130-334, length_regulator.py:24-39,275-321) on device.
 * ---------------------------------------------------------------------------------------------------------------- */
/* text ids -> per-subword char lengths + char id sequence, using per-token tables built once from the vocab:
 *   tok_len[v] (chars in piece), tok_flags[v] (bit0 punct, bit1 starts-with-space-and-longer-than-1),
 *   tok_chars[v][max_chars] char ids.  text_seqs [B][L] (already [:, :-1]-trimmed, generator.py:287).
 *   char_lens [B][L] (incl. the two zero pads of TagManager), char_seqs [B][max_c] (filled with text pad),
 *   char_seq_lens [B]. */
int sb_text_to_chars(const int32_t* text_seqs, int32_t L, int32_t batch, const uint8_t* tok_len,
                     const uint8_t* tok_flags, const int32_t* tok_chars, int32_t max_chars, int32_t pad_idx,
                     int32_t unk_idx, int32_t eos_idx, int32_t* char_lens, int32_t* char_seqs, int32_t max_c,
                     int32_t* char_seq_lens, sb_stream_t stream);
/* HardUpsampling + additive terms: y[b][u] = x[b][src(u)] + alpha*pos[u] + (emb ? emb[ids[b][u]]*emb_scale : 0)
 * for u < sum(dur[b]), and exact zeros for sum(dur[b]) <= u < U: pos / emb are not added there, so those rows are the
 * zero padding the next conv reads (the reference adds them to padded rows too; every consumer masks those rows).
 *   x in sequence layout (x_rows,x_halo), y in sequence layout (y_rows,y_halo), U = y logical length; pos_table fp32
 *   [U][dim] or NULL, alpha a device fp32 scalar or NULL (0), emb fp16 or NULL; out_lens[b] = sum(dur[b]) if given.
 *   SB_ENOSUP for S > 10240 (the prefix sums of the durations live in 40 KB of shared memory). */
int sb_upsample_add(const void* x, int32_t x_rows, int32_t x_halo, int32_t S, const int32_t* dur, void* y,
                    int32_t y_rows, int32_t y_halo, int32_t U, int32_t batch, int32_t dim, const void* pos_table,
                    const float* alpha, const void* emb, const int32_t* ids, int32_t ids_ld, float emb_scale,
                    int32_t* out_lens, sb_stream_t stream);
/* durations = clamp(round((exp(logd)-1)*factor), min 1) * mask  (length_regulator.py:286-293) */
int sb_durations(const void* hidden, int32_t rows_ld, int32_t halo, const void* proj_w, float proj_b, int32_t dim,
                 const int32_t* lens, int32_t batch, int32_t S, float factor, int32_t* dur, sb_stream_t stream);
/* unit logits argmax with the tied projection done by sb_gemm into fp32: units = decode(argmax) (generator.py:346-353,
 * unit_tokenizer.py:231-241): pad beyond lens, eos->pad, pad->pad+4, -4.  units int32 [B][U] */
int sb_unit_argmax(const float* logits, int64_t ld, int32_t rows_per_seq, int32_t halo, int32_t U, int32_t batch,
                   int32_t vocab, const int32_t* lens, int32_t pad_idx, int32_t eos_idx, int32_t* units,
                   sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Vocoder glue (models/vocoder/codehifigan.py:75-101): x[b][u] = [lang | dict[unit] | spkr] into a sequence-layout
 * buffer; everything else of the HiFi-GAN generator is sb_gemm with fused epilogues.
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_vocoder_embed(const int32_t* units, int32_t U, int32_t batch, const void* dict, int32_t dict_dim,
                     const void* lang, int32_t lang_dim, const int32_t* lang_idx, const void* spkr, int32_t spkr_dim,
                     const int32_t* spkr_idx, void* x, int32_t x_rows, int32_t x_halo, sb_stream_t stream);
/* One whole HiFi-GAN ResBlock (models/vocoder/hifigan.py:33-121: three (convs1[d], convs2) pairs with leaky-relu and
 * residual adds) on a sequence-layout activation with 16 or 32 channels, fused in shared memory:
 *   out  = (resblock(x) + res2) * gamma        res2 = running sum over the generator's ResBlocks or NULL
 *   out2 = leaky_relu(out, out2_slope)         optional (the activation that feeds the next stage, hifigan.py:183/192)
 * Weights are the folded weight-norm kernels in sb_gemm conv layout (C, kernel_size * C), biases fp32.
 * Every row of `out` / `out2` that belongs to a sequence or its halo is written (halo rows with zeros).
 * lens (optional, int32 [batch], each <= T): sequence b has lens[b] rows; every conv sees rows >= lens[b] as zero
 * padding, as it would for that sequence alone, and those rows of `out` / `out2` are written as 0. */
typedef struct {
  const void* x; const void* res2; void* out; void* out2;
  const void* w1[3]; const float* b1[3];   /* convs1: dilation[i] */
  const void* w2[3]; const float* b2[3];   /* convs2: dilation 1 */
  int32_t dilation[3];
  int32_t channels, kernel_size;
  int32_t batch, T, rows_per_seq, halo;    /* sequence layout: data rows [halo, halo + T) of each rows_per_seq block */
  float slope;                             /* leaky-relu slope inside the block (hifigan.py:12 LRELU_SLOPE) */
  float gamma, out2_slope;
  const int32_t* lens;                     /* optional per-sequence lengths (NULL: every sequence has T rows) */
} sb_resblock_t;
int sb_hifigan_resblock(const sb_resblock_t* r, sb_stream_t stream);
/* final conv_post (C->1, k7) + tanh on CUDA cores: wav fp32 [B][T] from lrelu'ed activations in sequence layout;
 * lens (optional, int32 [B]): wav[b][t] = 0 for t >= lens[b] */
int sb_conv_post_tanh(const void* x, int32_t x_rows, int32_t x_halo, int32_t T, const int32_t* lens, int32_t C, int32_t batch,
                      const void* w, float bias, int32_t k, float* wav, int64_t wav_ld, sb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * SeamlessStreaming monotonic (EMMA) decoder pieces: PChooseLayer.forward (models/monotonic_decoder/p_choose.py:120-148).
 * The energy projections are sb_gemm calls (Linear+ReLU x4); these two cover the pooling and the step probability.
 *   sb_avgpool_time: y[b][j] = mean of x[b][j*ratio .. min((j+1)*ratio, T))   (AvgPool1d, ceil_mode=True), fp16
 *   sb_pchoose:      p[h][s][j] = sigmoid((q_h[s].k_h[j]/8 + energy_bias)/temperature), q (S, H*64), k (Sp, H*64), p fp32
 * ---------------------------------------------------------------------------------------------------------------- */
int sb_avgpool_time(const void* x, void* y, int32_t batch, int32_t T, int32_t C, int32_t ratio, sb_stream_t stream);
int sb_pchoose(const void* q_energy, const void* k_energy, float* p, int32_t S, int32_t Sp, int32_t heads,
               float energy_bias, float temperature, sb_stream_t stream);

/* small utilities */
int sb_cast_f32_to_f16(const float* src, void* dst, int64_t n, sb_stream_t stream);
int sb_fill_zero(void* dst, int64_t bytes, sb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SEAMLESS_B200_H_ */
