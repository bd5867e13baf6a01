// sb_decoder_step: ONE persistent kernel for a whole incremental text-decoder step (embedding frontend + every
// pre-LN decoder layer: self-attention over the KV cache, cross-attention over the static encoder K/V, FFN, final
// LayerNorm).  Replaces the ~280 dependent launches per step of round 1 (fairseq2 StandardTransformerDecoder with an
// IncrementalStateBag; C++ mirror ggml/examples/unity/fairseq2.cpp:979-1094 layer, :917-953 frontend).
//
// The step is HBM / latency bound: R = batch * beam rows (160 at the BASELINE config) against 1.2 GB of weights.
// Design:
//   * grid = G groups x NC CTAs, all co-resident (NC = #SMs, G CTAs per SM).  A group owns a contiguous slice of the
//     rows and walks the layer stack on its own: 11 phases per layer separated by group-wide barriers (one counter per
//     phase in global memory: arrive = fence + atomicAdd, wait = one polling lane per CTA).  Two groups per SM hide each
//     other's barrier / L2 round trips; the second group's weight tiles hit L2.
//   * GEMM phases (qkv, attention out, cross q, cross out, FFN inner, FFN out) run "transposed": a 128-feature weight
//     tile is the wgmma A operand (two m64 halves), the group's rows are the B operand (N = rows padded to 16),
//     accumulators in the registers of warpgroup 0, both operands staged by TMA (128B swizzle) through one smem ring.  The producer warp runs ahead of the
//     barriers: the weight tile of a stage is requested as soon as the stage is free, the activation tile only once
//     the previous phase has completed, so weights stream from HBM while the group waits.
//     Narrow products split K across CTAs (fp32 partials, reduced in fixed order by the consuming phase).
//   * SIMT phases run on all 8 warps: single-token attention (one warp per (row, head), online softmax, beam ancestry
//     through the `anc` slot table, K/V written once) and split-K reduce + bias + residual + LayerNorm (one row per CTA).
//   * Everything the kernel needs (pointers, shapes, the 5 TMA descriptors) travels as ONE __grid_constant__ parameter:
//     constant-bank reads survive the L1 invalidation that every gpu-scope fence / acquire performs, whereas a plan in
//     global memory (first version) had to be re-fetched from L2 at every phase, field by field, on the critical path.
//     Weights are TWO stacked tensors (all matrices with K = dim, all with K = ffn) so that 5 descriptors serve all
//     layers.  Each phase kind exists once in the instruction stream (loop + switch, single call site): the per-layer
//     hot code must stay in the SM's instruction cache, every phase runs it only once per layer.
// Every spin is bounded (trap + message instead of a hung GPU).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace sb {
namespace {

constexpr int DS_BK = 64;
constexpr int DS_TM = 128;
constexpr int DS_W_BYTES = DS_TM * DS_BK * 2;  // 16 KB weight tile per k-block
constexpr int DS_WORKERS = 8;
constexpr int DS_THREADS = 256;                // 8 warps, all SIMT workers; 0-3 also MMA + epilogue, 5 TMA producer
constexpr int DS_PPL = 11;                     // phases per layer
constexpr int DS_HD = 64;
constexpr int DS_MAX_STAGES = 8;
constexpr int DS_MAX_LAYERS = 32;
constexpr int DS_MISC_BYTES = 4096;            // barriers, LN scratch, attention staging (8 x 384 B)
constexpr int DS_MAX_NPAD = 128;               // rows per group: the wgmma N of the GEMM phases (npad accumulators per thread)

enum { G_QKV = 0, G_OUT = 1, G_CQ = 2, G_CO = 3, G_W1 = 4, G_W2 = 5 };
// phase offsets inside a layer: GEMM phases are 0,2,4,6,8,9; attention 1,5; reduce + LayerNorm 3,7,10
enum { PH_QKV = 0, PH_SELF = 1, PH_OUT = 2, PH_RED1 = 3, PH_CQ = 4, PH_CROSS = 5, PH_CO = 6, PH_RED2 = 7, PH_W1 = 8, PH_W2 = 9, PH_RED3 = 10 };

struct DsLayer {
  const float* bias[6];  // qkv, out, cq, co, w1, w2
  const float* ln_w[3];  // LayerNorm that follows the self-attn block / the cross-attn block / the FFN block
  const float* ln_b[3];
  elem_t* kc;             // self-attention K cache [rows (slots)][heads][max_len][64]
  elem_t* vc;
  const elem_t* cross_k;  // encoder K [batch][heads][s_enc][64]
  const elem_t* cross_v;
};

struct DsParams {
  CUtensorMap w_dim;  // fp16 [layers * (6*dim + ffn)][dim]: per layer qkv (3*dim rows), out, cq, co (dim rows each), ffn1 (ffn rows); box 64 x 128
  CUtensorMap w_ffn;  // fp16 [layers * dim][ffn]: ffn2; box 64 x 128
  CUtensorMap h, att, t;  // activations [rows][dim | dim | ffn]; box 64 x npad
  int layers, dim, ffn, heads;
  int R, G, rg, npad, NC, stages;
  int splits[6];
  int beam, s_enc, max_len, seqs_ld, anc_ld, n_phases;
  int pre_max;  // weight tiles a CTA may request ahead of a phase barrier (<= stages)
  int flags;  // debugging switches (SB_DS_FLAGS): 1 no proxy fence at arrive, 2 none at the producer, 4 no early weight prefetch, 8 no gpu fence at arrive
  float embed_scale;
  const int* seqs;
  const int* anc;
  const int* step_ptr;
  const int* enc_lens;
  const elem_t* embed;
  const float* pos;
  const float* ln0_w;
  const float* ln0_b;
  elem_t* x;
  elem_t* h_buf;
  elem_t* att_buf;
  elem_t* t_buf;
  float* part_qkv;
  float* part;
  elem_t* hist;
  unsigned int* counters;        // [G][n_phases]
  unsigned long long* timeline;  // optional [G][n_phases][8] SM-cycle stamps of CTA 0 of each group
  DsLayer layer[DS_MAX_LAYERS];
};

__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// slow path of wait_counter, out of line: the kernel's hot code has to stay small (instruction cache, see header)
__device__ __noinline__ void ds_poll(const unsigned* p, unsigned target) {
  unsigned long long t0 = 0;
  unsigned polls = 0;
  while (ld_relaxed_u32(p) < target) {
    __nanosleep(20);
    if ((++polls & 4095u) == 0) {  // %globaltimer is slow to read: the watchdog looks at it every 4096 polls
      const unsigned long long now = gtime_ns();
      if (t0 == 0) t0 = now;
      // a phase barrier that has not completed in 4 s traps (no printf: a call anywhere in the kernel makes ptxas
      // serialise the wgmma pipeline of the GEMM phases)
      if (now - t0 > 4000000000ull) asm volatile("trap;");
    }
  }
}
// Wait until *p >= target.  ONE lane polls (relaxed loads with back-off, then a gpu-scope fence); callers fan the result
// out with a warp / CTA barrier.
__device__ __forceinline__ void wait_counter(const unsigned* p, unsigned target) {
  if ((threadIdx.x & 31) == 0) {
    if (ld_relaxed_u32(p) < target) ds_poll(p, target);
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncwarp();
}
__device__ __forceinline__ void arrive_counter(unsigned* p, int flags) {
  if (!(flags & 1)) asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy stores of this CTA vs. remote TMA (async proxy) reads
  if (!(flags & 8)) asm volatile("fence.acq_rel.gpu;" ::: "memory");
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}

// stamps are SM cycle counts (clock64): all of them come from CTA 0 of a group, i.e. one SM
#define DS_TL(phase, k) do { if (tl != nullptr) tl[8 * (phase) + (k)] = (unsigned long long)clock64(); } while (0)

struct GemmPhase {
  const CUtensorMap* tmW;
  const CUtensorMap* tmX;
  int w_row0;  // first row of this matrix inside the stacked weight tensor
  int n_out, kb_total, splits, relu_f16;
  void* out;
  int phase;   // global phase index
};

__device__ __forceinline__ GemmPhase gemm_phase(const DsParams& P, int layer, int which) {
  GemmPhase g;
  g.tmW = &P.w_dim;
  g.splits = P.splits[which];
  g.relu_f16 = 0;
  const int base = 1 + DS_PPL * layer;
  const int lrow = layer * (6 * P.dim + P.ffn);
  g.kb_total = P.dim / DS_BK;
  g.n_out = P.dim;
  g.out = P.part;
  g.tmX = (which & 1) ? &P.att : &P.h;  // out / co read the attention output, qkv / cq / w1 the normalised stream
  switch (which) {
    case G_QKV: g.w_row0 = lrow; g.n_out = 3 * P.dim; g.out = P.part_qkv; g.phase = base + PH_QKV; break;
    case G_OUT: g.w_row0 = lrow + 3 * P.dim; g.phase = base + PH_OUT; break;
    case G_CQ: g.w_row0 = lrow + 4 * P.dim; g.phase = base + PH_CQ; break;
    case G_CO: g.w_row0 = lrow + 5 * P.dim; g.phase = base + PH_CO; break;
    case G_W1: g.w_row0 = lrow + 6 * P.dim; g.n_out = P.ffn; g.out = P.t_buf; g.relu_f16 = 1; g.phase = base + PH_W1; break;
    default: g.tmW = &P.w_ffn; g.tmX = &P.t; g.w_row0 = layer * P.dim; g.kb_total = P.ffn / DS_BK; g.phase = base + PH_W2; break;
  }
  return g;
}

// unit u of a GEMM phase -> (tile, split, first k-block, end k-block); out of line (three integer divisions, four call sites)
struct UnitRange { int tile, split, kb0, kb1; };
__device__ __noinline__ UnitRange unit_range(int u, int splits, int kb_total) {
  UnitRange r;
  r.tile = u / splits;
  r.split = u - r.tile * splits;
  r.kb0 = (kb_total * r.split) / splits;
  r.kb1 = (kb_total * (r.split + 1)) / splits;
  return r;
}

// Single-query attention of one warp, keys staged in SHARED memory.  A decoder step is a chain of dependent round trips
// (each a full memory latency under load): reading K/V in register-sized slices put 7+ of them into every attention item.  Here
// the keys of a pass arrive with one batch of asynchronous copies (cp.async: no registers held) and the arithmetic runs
// from shared memory: scores -> probabilities (kept in shared memory) -> values, i.e. one round trip for K and one for V.
// Lane = (key group kg = lane/8, dim chunk dc = lane%8): 4 keys x 128 B per instruction, conflict-free.
// A pass covers up to `cap` keys; longer sequences take several passes with the running (max, sum, output) carried along.
struct AttnState { float m, l, o[8]; };

// scores of keys [0, n) against q -> p_s[t] = exp(score - new running max); updates m, l and rescales o
__device__ __noinline__ void attn_scores(AttnState& st, const elem_t* q_s, int n, const elem_t* k_s, float* p_s) {
  const int lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
  float q[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(q_s + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); q[2 * e] = f.x; q[2 * e + 1] = f.y; }
  }
  float mx = -INFINITY;
#pragma unroll 2
  for (int t0 = 0; t0 < n; t0 += 4) {  // warp-uniform trip count: the shuffles below name the full warp
    const int t = t0 + kg;
    const bool ok = t < n;
    const uint4 u = ok ? *reinterpret_cast<const uint4*>(k_s + t * DS_HD + dc * 8) : make_uint4(0, 0, 0, 0);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); a += q[2 * e] * f.x + q[2 * e + 1] * f.y; }
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    a += __shfl_xor_sync(0xffffffffu, a, 4);
    a *= 0.125f;
    if (ok) {
      if (dc == 0) p_s[t] = a;
      mx = fmaxf(mx, a);
    }
  }
  mx = warp_max(mx);
  const float m_new = fmaxf(st.m, mx);
  const float scale = __expf(st.m - m_new);
  st.m = m_new;
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < n; t += 32) {
    const float pw = __expf(p_s[t] - m_new);
    p_s[t] = pw;
    sum += pw;
  }
  st.l = st.l * scale + warp_sum(sum);
#pragma unroll
  for (int e = 0; e < 8; ++e) st.o[e] *= scale;
  __syncwarp();
}
// o += sum_t p_s[t] * v[t] (per lane: the partial sum of its key group for its 8 dims)
__device__ __noinline__ void attn_values(AttnState& st, int n, const elem_t* v_s, const float* p_s) {
  const int lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
#pragma unroll 2
  for (int t = kg; t < n; t += 4) {
    const float pw = p_s[t];
    const uint4 u = *reinterpret_cast<const uint4*>(v_s + t * DS_HD + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); st.o[2 * e] += pw * f.x; st.o[2 * e + 1] += pw * f.y; }
  }
}
__device__ __forceinline__ void attn_init(AttnState& st) {
  st.m = -INFINITY; st.l = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) st.o[e] = 0.f;
}
__device__ __noinline__ void attn_finish(AttnState& st, elem_t* __restrict__ outp) {
  const int lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    st.o[e] += __shfl_xor_sync(0xffffffffu, st.o[e], 8);
    st.o[e] += __shfl_xor_sync(0xffffffffu, st.o[e], 16);
  }
  if (kg == 0) {
    const float inv = st.l > 0.f ? 1.f / st.l : 0.f;
    uint4 w;
    __half2* hh = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) hh[e] = __floats2half2_rn(st.o[2 * e] * inv, st.o[2 * e + 1] * inv);
    *reinterpret_cast<uint4*>(outp + dc * 8) = w;
  }
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// sum of the split-K slices (+bias) of 64 consecutive features of one row -> fp16 in shared memory
__device__ __forceinline__ void gather_head(const float* __restrict__ part, int splits, long long R, long long ld,
                                            const float* __restrict__ bias, long long row, int col0, elem_t* dst) {
  const int lane = threadIdx.x & 31;
  float2 acc = *reinterpret_cast<const float2*>(bias + col0 + 2 * lane);
  const float* pp = part + row * ld + col0 + 2 * lane;
  const long long zs = R * ld;
#pragma unroll 8
  for (int z = 0; z < splits; ++z) {
    const float2 p = __ldcg(reinterpret_cast<const float2*>(pp + z * zs));
    acc.x += p.x; acc.y += p.y;
  }
  reinterpret_cast<__half2*>(dst)[lane] = __floats2half2_rn(acc.x, acc.y);
}

// ------------------------------------------------------------------------------------------------ the kernel
// Warp roles: every warp is a SIMT worker; in GEMM phases warps 0-3 (warpgroup 0) issue the MMAs and run the epilogue
// from their accumulator registers, warp 5 is the TMA producer (it requests the next GEMM phase's weight tiles at the
// tail of the SIMT phase before it, i.e. before that phase's barrier).  8 warps x <= 128 registers keep two CTAs on an
// SM.  NP (= npad, the wgmma N) is a compile-time constant.  The NP accumulators per warpgroup-0 thread do not fit that
// budget beside the rest of the kernel for NP >= 64: the sm_90a build spills (stores / loads per thread, bytes): NP 64:
// 80 / 32, NP 80: 488 / 620, NP 96: 1416 / 1960, NP 128: 2376 / 2720.  The kernel is opt-in (SB_DECODER_FUSED).
template <int NP>
__global__ void __launch_bounds__(DS_THREADS, 2) decoder_step_kernel(const __grid_constant__ DsParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int NC = P.NC, flags = P.flags;
  const int grp = blockIdx.x / NC;
  // groups rotate their unit -> CTA map so that phases which keep only part of the machine busy (FFN inner: 64 tiles)
  // land on different SMs for co-resident groups
  const int vc = (blockIdx.x - grp * NC + NC - (grp * NC) / P.G) % NC;
  const int row0 = grp * P.rg;
  const int rg = min(P.rg, P.R - row0);
  const int stages = P.stages;
  constexpr int stage_bytes = DS_W_BYTES + NP * DS_BK * 2;
  unsigned* cnt = P.counters + (size_t)grp * P.n_phases;
  unsigned long long* tl = (P.timeline != nullptr && vc == 0) ? P.timeline + (size_t)grp * P.n_phases * 8 : nullptr;
  uint8_t* ring = smem;
  uint8_t* misc = smem + (size_t)stages * stage_bytes;
  uint64_t* full = (uint64_t*)misc;
  uint64_t* empty = full + DS_MAX_STAGES;
  float* s_red = (float*)(misc + 512);                           // [2][2][8] floats
  elem_t* stage_s = (elem_t*)(misc + 1024) + warp * 3 * DS_HD;   // per-warp [3][64] halves: q | k | v of the new token

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int dim = P.dim, H = P.heads;
  const int step = *P.step_ptr;
  // per-role running state
  int mma_stage = 0;                       // warpgroup 0: ring stage / parity of the next slot
  uint32_t mma_parity = 0;
  int w_stage = 0, x_stage = 0;            // warp 5: ring cursors of the weight / activation requests
  uint32_t w_parity = 0;
  int pre_phase = -1, pre_n = 0;           // warp 5: phase whose first pre_n weight tiles are already requested

  // weight tile (k-block kb, rows w_row..) -> next ring stage (waits for the stage to be free)
  auto issue_w = [&](const CUtensorMap* tm, int kb, int w_row) {
    mbar_wait(&empty[w_stage], w_parity ^ 1);
    if (elect_one()) {
      mbar_expect_tx(&full[w_stage], (uint32_t)stage_bytes);
      tma_load_2d(ring + (size_t)w_stage * stage_bytes, tm, &full[w_stage], kb * DS_BK, w_row);
    }
    __syncwarp();
    if (++w_stage == stages) { w_stage = 0; w_parity ^= 1; }
  };
  // Request the first weight tiles of this CTA's first unit of GEMM phase q ahead of the phase barrier.  Called when every
  // earlier slot already has both of its loads requested, so up to `stages` tiles fit.
  auto prefetch_w = [&](int q) {
    pre_phase = q; pre_n = 0;
    if (q >= P.n_phases || (flags & 4)) return;
    const int ql = (q - 1) / DS_PPL, qk = (q - 1) - ql * DS_PPL;
    const GemmPhase g = gemm_phase(P, ql, (qk == PH_W2) ? G_W2 : (qk >> 1));
    if (vc >= ((g.n_out + DS_TM - 1) / DS_TM) * g.splits) return;
    const UnitRange ur = unit_range(vc, g.splits, g.kb_total);
    pre_n = min(P.pre_max, ur.kb1 - ur.kb0);
    for (int i = 0; i < pre_n; ++i) issue_w(g.tmW, ur.kb0 + i, g.w_row0 + ur.tile * DS_TM);
  };

#pragma unroll 1
  for (int p = 0; p < P.n_phases; ++p) {
    const int layer = p > 0 ? (p - 1) / DS_PPL : 0;
    const int k = p > 0 ? (p - 1) - layer * DS_PPL : PH_RED3;  // phase 0 = embedding + first LayerNorm (a reduce-type phase)
    const DsLayer& L = P.layer[layer];
    if ((0x355 >> k) & 1) {
      // ======================================================================================= GEMM phase
      const GemmPhase g = gemm_phase(P, layer, (k == PH_W2) ? G_W2 : (k >> 1));
      const int units = ((g.n_out + DS_TM - 1) / DS_TM) * g.splits;
      if (warp == 5 && pre_phase != p) prefetch_w(p);  // a GEMM phase that follows a GEMM phase (FFN inner -> FFN out)
      bool dep_ok = false;
#pragma unroll 1
      for (int u = vc; u < units; u += NC) {
        const UnitRange ur = unit_range(u, g.splits, g.kb_total);
        if (ur.kb0 >= ur.kb1) continue;
        if (warp == 5) {
          // ---- TMA producer
#pragma unroll 1
          for (int kb = ur.kb0; kb < ur.kb1; ++kb) {
            if (pre_n > 0) --pre_n;
            else issue_w(g.tmW, kb, g.w_row0 + ur.tile * DS_TM);
            if (!dep_ok) {
              wait_counter(&cnt[p - 1], (unsigned)NC);
              if (!(flags & 2)) asm volatile("fence.proxy.async;" ::: "memory");
              dep_ok = true;
              if (lane == 0) DS_TL(p, 0);
            }
            if (elect_one()) tma_load_2d(ring + (size_t)x_stage * stage_bytes + DS_W_BYTES, g.tmX, &full[x_stage], kb * DS_BK, row0);
            __syncwarp();
            if (++x_stage == stages) x_stage = 0;
          }
          if (lane == 0) DS_TL(p, 3);
        } else if (warp < 4) {
          // ---- MMA: D[feature][row] += W[128 x 64] . X[NP x 64]^T, features 0-63 in acc[0], 64-127 in acc[1]
          float acc[2][NP / 2];
#pragma unroll
          for (int i = 0; i < NP / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
          int prev = 0;
#pragma unroll 1
          for (int kb = ur.kb0; kb < ur.kb1; ++kb) {
            const int s = mma_stage;
            mbar_wait(&full[s], mma_parity);
            if (++mma_stage == stages) { mma_stage = 0; mma_parity ^= 1; }
            if (kb == ur.kb0 && threadIdx.x == 0) DS_TL(p, 6);
            const uint32_t sa = smem_u32(ring + (size_t)s * stage_bytes);
            const uint64_t da = make_smem_desc(sa), db = make_smem_desc(sa + DS_W_BYTES);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < DS_BK / 16; ++kk) {
              Wgmma<NP>::mma(acc[0], da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2));
              Wgmma<NP>::mma(acc[1], da + (uint64_t)(64 * 128 / 16 + kk * 2), db + (uint64_t)(kk * 2));
            }
            wg_commit();
            wg_wait<1>();
            wg_fence_regs(acc[0]);
            wg_fence_regs(acc[1]);
            if (kb > ur.kb0 && threadIdx.x == 0) mbar_arrive(&empty[prev]);
            prev = s;
          }
          wg_wait<0>();
          wg_fence_regs(acc[0]);
          wg_fence_regs(acc[1]);
          if (threadIdx.x == 0) mbar_arrive(&empty[prev]);
          if (threadIdx.x == 0) DS_TL(p, 2);
          // ---- epilogue: register j*4 + 2h + e of acc[mt] = (feature fb + 64 mt + 8h, row j*8 + 2*(lane%4) + e of the group)
          const int fb = ur.tile * DS_TM + warp * 16 + (lane >> 2);
          const int esz = g.relu_f16 ? 2 : 4;
          char* o = reinterpret_cast<char*>(g.out) + ((size_t)(g.relu_f16 ? 0 : ur.split) * P.R + row0) * g.n_out * esz;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int f = fb + 64 * mt + 8 * h;
              if (f >= g.n_out) continue;
              const float bias = g.relu_f16 ? L.bias[G_W1][f] : 0.f;
#pragma unroll
              for (int j = 0; j < NP / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int r = j * 8 + (lane & 3) * 2 + e;
                  if (r >= rg) continue;
                  const float v = acc[mt][j * 4 + 2 * h + e];
                  char* d = o + ((size_t)r * g.n_out + f) * esz;
                  if (g.relu_f16) *reinterpret_cast<elem_t*>(d) = __float2half_rn(fmaxf(v + bias, 0.f));
                  else *reinterpret_cast<float*>(d) = v;
                }
              }
            }
          }
        }
      }
      if (warp < 4) {
        if (threadIdx.x == 0) DS_TL(p, 4);
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (threadIdx.x == 0) {
          DS_TL(p, 5);
          arrive_counter(&cnt[p], flags);
          DS_TL(p, 1);
        }
      }
    } else {
      // ======================================================================================= SIMT phase
      if (p > 0) {
        if (warp == 0) wait_counter(&cnt[p - 1], (unsigned)NC);
        asm volatile("bar.sync 2, 256;" ::: "memory");  // data produced by other CTAs is read with L2 (.cg) loads below
      }
      if (threadIdx.x == 0) DS_TL(p, 0);
      if ((0x22 >> k) & 1) {
        // The TMA ring is idle while a SIMT phase works (every requested slot has been consumed): it serves as scratch.
        const int ring_bytes = stages * stage_bytes;
        if (k == PH_SELF) {
          // ---- self-attention over the KV cache: one warp per (row, head); per-warp scratch = [cap keys][128 B] | p[cap] | slots
          const int wbytes = (ring_bytes / DS_WORKERS) & ~1023;
          const int cap = min((wbytes - 1024) / 128, 128);  // keys per pass (ancestry and probabilities: 512 B each)
          elem_t* kv_s = reinterpret_cast<elem_t*>(ring + (size_t)warp * wbytes);
          float* p_s = reinterpret_cast<float*>(ring + (size_t)warp * wbytes + cap * 128);
          int* slots_s = reinterpret_cast<int*>(p_s + 128);
          const int kg = lane >> 3, dc = lane & 7;
          const int slot_stride = H * P.max_len * DS_HD;
          const int items = rg * H;
          for (int it = vc * DS_WORKERS + warp; it < items; it += NC * DS_WORKERS) {
            const int j = it / H, hd = it - j * H;
            const long long row = row0 + j;
            const int* anc_row = P.anc + row * P.anc_ld;
            const elem_t* kc = L.kc + (long long)hd * P.max_len * DS_HD;
            const elem_t* vcache = L.vc + (long long)hd * P.max_len * DS_HD;
            __syncwarp();
#pragma unroll 1
            for (int t = 0; t < 3; ++t)
              gather_head(P.part_qkv, P.splits[G_QKV], P.R, 3LL * dim, L.bias[G_QKV], row, t * dim + hd * DS_HD, stage_s + t * DS_HD);
            __syncwarp();
            // persist the new K/V (slot = row, position = step)
            const long long o = (((long long)row * H + hd) * P.max_len + step) * DS_HD;
            reinterpret_cast<__half2*>(L.kc + o)[lane] = reinterpret_cast<const __half2*>(stage_s + DS_HD)[lane];
            reinterpret_cast<__half2*>(L.vc + o)[lane] = reinterpret_cast<const __half2*>(stage_s + 2 * DS_HD)[lane];
            AttnState st;
            attn_init(st);
#pragma unroll 1
            for (int k0 = 0; k0 <= step; k0 += cap) {
              const int n = min(cap, step + 1 - k0);
              for (int t = lane; t < n; t += 32) slots_s[t] = (k0 + t < step) ? anc_row[k0 + t] : 0;
              __syncwarp();
              // K rows of this pass: cached positions by asynchronous copy, the new token from its staging buffer
              for (int t = kg; t < n; t += 4) {
                elem_t* dst = kv_s + t * DS_HD + dc * 8;
                if (k0 + t < step) cp_async16(dst, kc + slots_s[t] * slot_stride + (k0 + t) * DS_HD + dc * 8);
                else *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(stage_s + DS_HD + dc * 8);
              }
              cp_async_wait_all();
              __syncwarp();
              attn_scores(st, stage_s, n, kv_s, p_s);
              for (int t = kg; t < n; t += 4) {
                elem_t* dst = kv_s + t * DS_HD + dc * 8;
                if (k0 + t < step) cp_async16(dst, vcache + slots_s[t] * slot_stride + (k0 + t) * DS_HD + dc * 8);
                else *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(stage_s + 2 * DS_HD + dc * 8);
              }
              cp_async_wait_all();
              __syncwarp();
              attn_values(st, n, kv_s, p_s);
              __syncwarp();
            }
            attn_finish(st, P.att_buf + row * dim + hd * DS_HD);
          }
        } else {
          // ---- cross-attention: one CTA per (sentence, head).  The beams of a sentence attend the same keys: the CTA
          // stages them in shared memory once (instead of one read per hypothesis: 160 rows x 16 heads x 63 keys x 256 B
          // = 41 MB per layer, the largest stream of a step) and each warp serves one hypothesis.  Groups hold whole
          // sentences.  Scratch = K[cap] | V[cap] | p[8 warps][cap].
          const int beam = P.beam;
          const int cap = min((ring_bytes - DS_WORKERS * 512) / 256, 128);
          elem_t* k_s = reinterpret_cast<elem_t*>(ring);
          elem_t* v_s = k_s + cap * DS_HD;
          float* p_s = reinterpret_cast<float*>(ring + (size_t)cap * 256) + warp * 128;
          const int items = (rg / beam) * H;
          for (int it = vc; it < items; it += NC) {
            const int sj = it / H, hd = it - sj * H;
            const long long srow = row0 + (long long)sj * beam;
            const int b = (int)(srow / beam);
            const int nkeys = P.enc_lens ? min(P.enc_lens[b], P.s_enc) : P.s_enc;
            const long long kvo = ((long long)b * H + hd) * P.s_enc * DS_HD;
            AttnState st;
            attn_init(st);
            const int qi = warp;  // hypotheses beyond 8 per sentence: see the loop below
#pragma unroll 1
            for (int q0 = 0; q0 < beam; q0 += DS_WORKERS) {
              const bool have_q = q0 + qi < beam;
              if (have_q) {
                __syncwarp();
                gather_head(P.part, P.splits[G_CQ], P.R, dim, L.bias[G_CQ], srow + q0 + qi, hd * DS_HD, stage_s);
                __syncwarp();
                attn_init(st);
              }
#pragma unroll 1
              for (int k0 = 0; k0 < nkeys; k0 += cap) {
                const int n = min(cap, nkeys - k0);
                for (int i = threadIdx.x; i < n * 8; i += DS_THREADS) {
                  cp_async16(k_s + i * 8, L.cross_k + kvo + (long long)k0 * DS_HD + i * 8);
                  cp_async16(v_s + i * 8, L.cross_v + kvo + (long long)k0 * DS_HD + i * 8);
                }
                cp_async_wait_all();
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (have_q) {
                  attn_scores(st, stage_s, n, k_s, p_s);
                  attn_values(st, n, v_s, p_s);
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");  // the staging area is reused (next pass / item / weight prefetch)
              }
              if (have_q) attn_finish(st, P.att_buf + (srow + q0 + qi) * dim + hd * DS_HD);
            }
          }
        }
      } else {
        // ---- x_new = (residual | embedding) + bias + sum_z partial[z]; h = LN(x_new).  One row per CTA iteration, 8 warps
        // per row.  Numerics as sb_splitk_reduce_ln (layernorm.cu): fp32 sum in fixed z order, rounded to fp16, LN over
        // the rounded values.
        const bool embed = (p == 0);
        const int ri = (k == PH_RED1) ? 0 : (k == PH_RED2) ? 1 : 2;
        const int splits = P.splits[2 * ri + 1];
        const float* bias = L.bias[2 * ri + 1];
        const float* lnw = embed ? P.ln0_w : L.ln_w[ri];
        const float* lnb = embed ? P.ln0_b : L.ln_b[ri];
        const bool write_hist = (p == P.n_phases - 1) && P.hist != nullptr;
        const int cpw = dim / DS_WORKERS;
        const int col = warp * cpw + lane * 4;
        const bool act = lane * 4 < cpw;
        int it = 0;
        for (int j = vc; j < rg; j += NC, ++it) {
          const long long row = row0 + j;
          float v[4] = {0.f, 0.f, 0.f, 0.f};
          float s = 0.f;
          if (act) {
            float a[4];
            if (embed) {
              const int tok = P.seqs[row * P.seqs_ld + step];
              const uint2 e = *reinterpret_cast<const uint2*>(P.embed + (long long)tok * dim + col);
              const float4 pp = *reinterpret_cast<const float4*>(P.pos + (long long)step * dim + col);
              const float2 e0 = __half22float2(*reinterpret_cast<const __half2*>(&e.x)), e1 = __half22float2(*reinterpret_cast<const __half2*>(&e.y));
              a[0] = e0.x * P.embed_scale + pp.x; a[1] = e0.y * P.embed_scale + pp.y;
              a[2] = e1.x * P.embed_scale + pp.z; a[3] = e1.y * P.embed_scale + pp.w;
            } else {
              const uint2 xr = __ldcg(reinterpret_cast<const uint2*>(P.x + row * dim + col));
              const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(&xr.x)), x1 = __half22float2(*reinterpret_cast<const __half2*>(&xr.y));
              const float4 b = *reinterpret_cast<const float4*>(bias + col);
              a[0] = x0.x + b.x; a[1] = x0.y + b.y; a[2] = x1.x + b.z; a[3] = x1.y + b.w;
              const float* pp = P.part + row * dim + col;
              const size_t zs = (size_t)P.R * dim;
#pragma unroll 8
              for (int z = 0; z < splits; ++z) {
                const float4 q4 = __ldcg(reinterpret_cast<const float4*>(pp + z * zs));
                a[0] += q4.x; a[1] += q4.y; a[2] += q4.z; a[3] += q4.w;
              }
            }
            uint2 o;
            __half2 h0 = __floats2half2_rn(a[0], a[1]), h1 = __floats2half2_rn(a[2], a[3]);
            o.x = *reinterpret_cast<uint32_t*>(&h0); o.y = *reinterpret_cast<uint32_t*>(&h1);
            *reinterpret_cast<uint2*>(P.x + row * dim + col) = o;
            const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
            v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y;
            s = v[0] + v[1] + v[2] + v[3];
          }
          float* sr = s_red + (it & 1) * 2 * DS_WORKERS;
          if (it == 0 && threadIdx.x == 0) DS_TL(p, 2);
          s = warp_sum(s);
          if (lane == 0) sr[warp] = s;
          asm volatile("bar.sync 2, 256;" ::: "memory");
          float tot = 0.f;
#pragma unroll
          for (int i = 0; i < DS_WORKERS; ++i) tot += sr[i];
          const float mean = tot / dim;
          float sq = 0.f;
          if (act) {
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float d = v[e] - mean; sq += d * d; }
          }
          sq = warp_sum(sq);
          if (lane == 0) sr[DS_WORKERS + warp] = sq;
          asm volatile("bar.sync 2, 256;" ::: "memory");
          float tsq = 0.f;
#pragma unroll
          for (int i = 0; i < DS_WORKERS; ++i) tsq += sr[DS_WORKERS + i];
          const float rstd = rsqrtf(tsq / dim + 1e-5f);
          if (it == 0 && threadIdx.x == 0) DS_TL(p, 3);
          if (act) {
            const float4 w = *reinterpret_cast<const float4*>(lnw + col), b = *reinterpret_cast<const float4*>(lnb + col);
            __half2 h0 = __floats2half2_rn((v[0] - mean) * rstd * w.x + b.x, (v[1] - mean) * rstd * w.y + b.y);
            __half2 h1 = __floats2half2_rn((v[2] - mean) * rstd * w.z + b.z, (v[3] - mean) * rstd * w.w + b.w);
            uint2 o;
            o.x = *reinterpret_cast<uint32_t*>(&h0); o.y = *reinterpret_cast<uint32_t*>(&h1);
            *reinterpret_cast<uint2*>(P.h_buf + row * dim + col) = o;
            if (write_hist) *reinterpret_cast<uint2*>(P.hist + ((long long)step * P.R + row) * dim + col) = o;
          }
        }
      }
      // ---- tail: the producer requests the weights of the GEMM phase that follows (before this phase's barrier), then
      // the CTA arrives
      if (k == PH_SELF) asm volatile("bar.sync 2, 256;" ::: "memory");  // ring scratch (ancestry) is dead before the weight prefetch
      if (warp == 5) prefetch_w(p + 1);
      if (threadIdx.x == 0) DS_TL(p, 4);
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if (threadIdx.x == 0) {
        DS_TL(p, 5);
        arrive_counter(&cnt[p], flags);
        DS_TL(p, 1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_map(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  SB_REQUIRE(fn != nullptr, SB_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {inner * 2};
  cuuint32_t box[2] = {(cuuint32_t)DS_BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_REQUIRE(r == CUDA_SUCCESS, SB_ECUDA, "sb_decoder_plan: cuTensorMapEncodeTiled failed (%d) inner=%llu rows=%llu box_rows=%u",
             (int)r, (unsigned long long)inner, (unsigned long long)rows, box_rows);
  return SB_OK;
}

typedef void (*DsKernel)(DsParams);
DsKernel pick_kernel(int npad) {
  switch (npad) {
    case 16: return decoder_step_kernel<16>;
    case 32: return decoder_step_kernel<32>;
    case 48: return decoder_step_kernel<48>;
    case 64: return decoder_step_kernel<64>;
    case 80: return decoder_step_kernel<80>;
    case 96: return decoder_step_kernel<96>;
    case 112: return decoder_step_kernel<112>;
    default: return decoder_step_kernel<128>;
  }
}

int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e && *e) ? atoi(e) : dflt;
}

}  // namespace
}  // namespace sb


// [batch*s_enc][ld] (k | v concatenated along the features) -> k, v as [batch][heads][s_enc][64]
__global__ void kv_heads_major_kernel(const sb::elem_t* __restrict__ src, long long ld, int s_enc, int heads, sb::elem_t* __restrict__ k_out,
                                      sb::elem_t* __restrict__ v_out, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one 16-byte chunk (8 halves) per thread
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  long long r = i >> 3;
  const int t = (int)(r % s_enc); r /= s_enc;
  const int h = (int)(r % heads); r /= heads;
  const int kv = (int)(r & 1);
  const long long b = r >> 1;
  const uint4 u = *reinterpret_cast<const uint4*>(src + (b * s_enc + t) * ld + (long long)kv * heads * 64 + h * 64 + c8 * 8);
  sb::elem_t* dst = (kv ? v_out : k_out) + (((b * heads + h) * s_enc + t) * 64 + c8 * 8);
  *reinterpret_cast<uint4*>(dst) = u;
}

extern "C" int sb_kv_heads_major(const void* kv, int64_t ld, int32_t batch, int32_t s_enc, int32_t heads, void* k_out, void* v_out,
                                 sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(kv && k_out && v_out && batch > 0 && s_enc > 0 && heads > 0 && ld >= 2LL * heads * 64 && ld % 8 == 0, SB_EINVAL,
             "sb_kv_heads_major: bad args");
  const long long total = 2LL * batch * heads * s_enc * 8;
  kv_heads_major_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const elem_t*)kv, ld, s_enc, heads, (elem_t*)k_out,
                                                                                         (elem_t*)v_out, total);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_decoder_plan_query(int32_t layers, int32_t dim, int32_t ffn_dim, int32_t rows, int32_t beam, int32_t groups,
                                     sb_decoder_plan_info_t* info) {
  using namespace sb;
  SB_REQUIRE(info != nullptr && layers >= 1 && rows >= 1 && beam >= 1 && rows % beam == 0, SB_EINVAL, "sb_decoder_plan_query: bad args");
  SB_REQUIRE(layers <= DS_MAX_LAYERS, SB_ENOSUP, "sb_decoder_plan_query: at most %d layers", DS_MAX_LAYERS);
  SB_REQUIRE(dim % 64 == 0 && dim >= 64 && dim <= 1024 && ffn_dim % 64 == 0 && ffn_dim >= 64, SB_ENOSUP,
             "sb_decoder_plan_query: dim %d / ffn_dim %d unsupported (multiples of 64, dim <= 1024)", dim, ffn_dim);
  int dev = 0, sms = 0, smem_optin = 0, smem_sm = 0;
  SB_CUDA_OK(cudaGetDevice(&dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
  memset(info, 0, sizeof(*info));
  int G = groups;
  if (G <= 0) G = env_int("SB_DS_GROUPS", rows >= 96 ? 2 : 1);
  if (G > 2) G = 2;
  if (G > rows) G = 1;
  int rg = (rows + G - 1) / G;
  if (rg > DS_MAX_NPAD) { G = 2; rg = (rows + 1) / 2; }
  if (beam > 1) rg = (rg + beam - 1) / beam * beam;  // groups hold whole sentences (cross-attention shares K/V across the beams)
  SB_REQUIRE(rg <= DS_MAX_NPAD, SB_ENOSUP, "sb_decoder_plan_query: %d rows exceed 2 groups x %d", rows, DS_MAX_NPAD);
  const int npad = (rg + 15) / 16 * 16;
  const int stage_bytes = DS_W_BYTES + npad * DS_BK * 2;
  // every resident CTA also pays 1 KB of system shared memory
  const int budget = (G == 1 ? smem_optin : (smem_sm - 2 * 1024) / 2 - 512) - DS_MISC_BYTES - 1024;
  int stages = budget / stage_bytes;
  if (stages > DS_MAX_STAGES) stages = DS_MAX_STAGES;
  if (env_int("SB_DS_STAGES", 0) >= 2 && env_int("SB_DS_STAGES", 0) < stages) stages = env_int("SB_DS_STAGES", 0);
  SB_REQUIRE(stages >= 2, SB_ENOSUP, "sb_decoder_plan_query: not enough shared memory for %d rows per group", rg);
  info->groups = G;
  info->rows_per_group = rg;
  info->npad = npad;
  info->ctas_per_group = sms;
  info->stages = stages;
  info->smem_bytes = stages * stage_bytes + DS_MISC_BYTES + 1024;
  info->n_phases = 1 + DS_PPL * layers;
  // split-K policy: fill the machine, but keep >= 2 k-blocks per unit (each split costs a 128 x rows fp32 partial tile)
  const int kb_d = dim / DS_BK, kb_f = ffn_dim / DS_BK;
  auto pick = [&](int n_out, int kb, int min_kb, int cap) {
    const int tiles = (n_out + DS_TM - 1) / DS_TM;
    int s = sms / tiles;
    if (s > kb / min_kb) s = kb / min_kb;
    if (s > cap) s = cap;
    return s < 1 ? 1 : s;
  };
  info->splits[0] = pick(3 * dim, kb_d, 2, 8);
  info->splits[1] = info->splits[2] = info->splits[3] = pick(dim, kb_d, 2, 8);
  info->splits[4] = 1;
  info->splits[5] = pick(dim, kb_f, 4, 16);
  const char* e = getenv("SB_DS_SPLITS");  // "qkv,out,cq,co,ffn2"
  if (e && *e) {
    int v[5] = {0, 0, 0, 0, 0};
    if (sscanf(e, "%d,%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3], &v[4]) == 5) {
      const int idx[5] = {0, 1, 2, 3, 5};
      for (int i = 0; i < 5; ++i) {
        const int kb = idx[i] == 5 ? kb_f : kb_d;
        if (v[i] >= 1) info->splits[idx[i]] = v[i] > kb ? kb : v[i];
      }
    }
  }
  int smax = info->splits[1];
  for (int i : {2, 3, 5}) smax = info->splits[i] > smax ? info->splits[i] : smax;
  info->part_qkv_floats = (int64_t)info->splits[0] * rows * 3 * dim;
  info->part_floats = (int64_t)smax * rows * dim;
  info->counters_len = (int64_t)G * info->n_phases;
  return SB_OK;
}

extern "C" int sb_decoder_plan_init(const sb_decoder_plan_desc_t* d, sb_decoder_launch_t* launch) {
  using namespace sb;
  SB_REQUIRE(d != nullptr && launch != nullptr && d->layer != nullptr, SB_EINVAL, "sb_decoder_plan_init: null argument");
  SB_REQUIRE(d->heads * DS_HD == d->dim, SB_ENOSUP, "sb_decoder_plan_init: head_dim must be 64 (dim %d, heads %d)", d->dim, d->heads);
  sb_decoder_plan_info_t info;
  int rc = sb_decoder_plan_query(d->layers, d->dim, d->ffn_dim, d->rows, d->beam, d->groups, &info);
  if (rc) return rc;
  SB_REQUIRE(d->part_qkv_floats >= info.part_qkv_floats && d->part_floats >= info.part_floats && d->counters_len >= info.counters_len,
             SB_EINVAL, "sb_decoder_plan_init: workspace too small (see sb_decoder_plan_query)");
  SB_REQUIRE(d->x && d->h && d->att && d->ffn_act && d->part_qkv && d->part && d->counters && d->seqs && d->anc && d->step_ptr &&
                 d->embed && d->pos && d->ln0_w && d->ln0_b && d->w_dim_stack && d->w_ffn_stack,
             SB_EINVAL, "sb_decoder_plan_init: null buffer");
  SB_REQUIRE(d->beam >= 1 && d->s_enc >= 1 && d->max_len >= 1, SB_EINVAL, "sb_decoder_plan_init: bad beam / s_enc / max_len");
  SB_REQUIRE((long long)d->rows * d->heads * d->max_len * DS_HD < (1ll << 31), SB_ENOSUP, "sb_decoder_plan_init: K/V cache of one layer exceeds 2^31 elements");
  static_assert(sizeof(DsParams) <= sizeof(launch->params), "sb_decoder_launch_t::params too small");
  static_assert(sizeof(DsParams) <= 32764, "kernel parameter limit");
  DsParams* P = (DsParams*)calloc(1, sizeof(DsParams));
  SB_REQUIRE(P != nullptr, SB_EINVAL, "sb_decoder_plan_init: out of host memory");
  auto fail = [&](int code) { free(P); return code; };
  P->layers = d->layers; P->dim = d->dim; P->ffn = d->ffn_dim; P->heads = d->heads;
  P->R = d->rows; P->G = info.groups; P->rg = info.rows_per_group; P->npad = info.npad; P->NC = info.ctas_per_group;
  P->stages = info.stages;
  for (int i = 0; i < 6; ++i) P->splits[i] = info.splits[i];
  P->beam = d->beam; P->s_enc = d->s_enc; P->max_len = d->max_len; P->seqs_ld = d->seqs_ld; P->anc_ld = d->anc_ld;
  P->n_phases = info.n_phases;
  P->flags = env_int("SB_DS_FLAGS", 0);
  P->pre_max = env_int("SB_DS_PREFETCH", info.stages);
  if (P->pre_max > info.stages) P->pre_max = info.stages;
  if (P->pre_max < 0) P->pre_max = 0;
  P->embed_scale = d->embed_scale;
  P->seqs = d->seqs; P->anc = d->anc; P->step_ptr = d->step_ptr; P->enc_lens = d->enc_lens;
  P->embed = (const elem_t*)d->embed; P->pos = d->pos; P->ln0_w = d->ln0_w; P->ln0_b = d->ln0_b;
  P->x = (elem_t*)d->x; P->h_buf = (elem_t*)d->h; P->att_buf = (elem_t*)d->att; P->t_buf = (elem_t*)d->ffn_act;
  P->part_qkv = d->part_qkv; P->part = d->part; P->hist = (elem_t*)d->hist;
  P->counters = d->counters; P->timeline = (unsigned long long*)d->timeline;
  DsParams& maps = *P;
  if ((rc = encode_map(&maps.h, d->h, (uint64_t)d->dim, (uint64_t)d->rows, (uint32_t)info.npad))) return fail(rc);
  if ((rc = encode_map(&maps.att, d->att, (uint64_t)d->dim, (uint64_t)d->rows, (uint32_t)info.npad))) return fail(rc);
  if ((rc = encode_map(&maps.t, d->ffn_act, (uint64_t)d->ffn_dim, (uint64_t)d->rows, (uint32_t)info.npad))) return fail(rc);
  if ((rc = encode_map(&maps.w_dim, d->w_dim_stack, (uint64_t)d->dim, (uint64_t)d->layers * (6ull * d->dim + d->ffn_dim), DS_TM))) return fail(rc);
  if ((rc = encode_map(&maps.w_ffn, d->w_ffn_stack, (uint64_t)d->ffn_dim, (uint64_t)d->layers * d->dim, DS_TM))) return fail(rc);
  for (int l = 0; l < d->layers; ++l) {
    const sb_decoder_layer_t& s = d->layer[l];
    DsLayer& L = P->layer[l];
    const float* b[6] = {s.qkv_b, s.out_b, s.cq_b, s.co_b, s.ffn1_b, s.ffn2_b};
    for (int i = 0; i < 6; ++i) {
      if (b[i] == nullptr) { set_error("sb_decoder_plan_init: layer %d: null bias %d", l, i); return fail(SB_EINVAL); }
      L.bias[i] = b[i];
    }
    L.ln_w[0] = s.ca_ln_w; L.ln_b[0] = s.ca_ln_b; L.ln_w[1] = s.ffn_ln_w; L.ln_b[1] = s.ffn_ln_b;
    L.ln_w[2] = s.next_ln_w; L.ln_b[2] = s.next_ln_b;
    for (int i = 0; i < 3; ++i)
      if (L.ln_w[i] == nullptr || L.ln_b[i] == nullptr) { set_error("sb_decoder_plan_init: layer %d: null LayerNorm %d", l, i); return fail(SB_EINVAL); }
    if (!s.k_cache || !s.v_cache || !s.cross_k || !s.cross_v) { set_error("sb_decoder_plan_init: layer %d: null K/V", l); return fail(SB_EINVAL); }
    L.kc = (elem_t*)s.k_cache; L.vc = (elem_t*)s.v_cache;
    L.cross_k = (const elem_t*)s.cross_k; L.cross_v = (const elem_t*)s.cross_v;
  }
  memset(launch, 0, sizeof(*launch));
  memcpy(launch->params, P, sizeof(DsParams));
  free(P);
  DsKernel kern = pick_kernel(info.npad);
  {
    int dev = 0, smem_optin = 0;
    SB_CUDA_OK(cudaGetDevice(&dev));
    SB_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    SB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    SB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  }
  // Co-residency of all groups x NC CTAs is required (phase barriers spin): check registers and shared memory per SM.
  {
    cudaFuncAttributes fa;
    SB_CUDA_OK(cudaFuncGetAttributes(&fa, kern));
    int dev = 0, smem_sm = 0, regs_sm = 0;
    SB_CUDA_OK(cudaGetDevice(&dev));
    SB_CUDA_OK(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    SB_CUDA_OK(cudaDeviceGetAttribute(&regs_sm, cudaDevAttrMaxRegistersPerMultiprocessor, dev));
    const int regs_cta = ((fa.numRegs + 7) / 8 * 8) * DS_THREADS;
    SB_REQUIRE(info.groups * regs_cta <= regs_sm && info.groups * (info.smem_bytes + 1024 + (int)fa.sharedSizeBytes) <= smem_sm,
               SB_ENOSUP, "sb_decoder_plan_init: %d CTAs per SM do not fit (regs %d x %d threads, smem %d B)",
               info.groups, fa.numRegs, DS_THREADS, info.smem_bytes);
  }
  launch->npad = info.npad;
  launch->counters = d->counters;
  launch->counters_len = info.counters_len;
  launch->grid = info.groups * info.ctas_per_group;
  launch->block = DS_THREADS;
  launch->smem_bytes = info.smem_bytes;
  // two-group plans use a plain launch (the resource check above + an otherwise idle stream order guarantee residency;
  // every spin in the kernel is bounded)
  launch->cooperative = env_int("SB_DS_COOPERATIVE", info.groups == 1 ? 1 : 0);
  return SB_OK;
}

extern "C" int sb_decoder_step(const sb_decoder_launch_t* l, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(l != nullptr && l->counters != nullptr && l->grid > 0, SB_EINVAL, "sb_decoder_step: bad launch descriptor");
  cudaStream_t st = (cudaStream_t)stream;
  SB_CUDA_OK(cudaMemsetAsync(l->counters, 0, (size_t)l->counters_len * sizeof(unsigned int), st));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)l->grid);
  cfg.blockDim = dim3((unsigned)l->block);
  cfg.dynamicSmemBytes = (size_t)l->smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = l->cooperative ? 1 : 0;
  static thread_local DsParams prm;  // 64-byte aligned copy of the opaque blob (CUtensorMap alignment), one per launching host thread
  memcpy(&prm, l->params, sizeof(prm));
  SB_CUDA_OK(cudaLaunchKernelEx(&cfg, pick_kernel(l->npad), prm));
  count_launch();
  return SB_OK;
}
