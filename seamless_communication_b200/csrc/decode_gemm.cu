// The weight-stationary ("transposed") wgmma GEMM of a beam-search step: <= 256 rows (one step: 160 rows).
//
// The general kernel (gemm_tcgen05.cu) makes the rows its MMA M operand in 128-row tiles and gives a CTA 64 output
// features: at 160 rows it is bound by L2 -> SM traffic, not by HBM, since every CTA re-reads its 128-row activation
// tile for its few weight rows, and the second row tile is 80 % padding.  Here a 128-row WEIGHT tile is the wgmma A
// operand (two consumer warpgroups, 64 weight rows each) and ALL rows are the B operand (N = rows rounded up to 32, 64,
// 128, 160 or 256; 160 is a beam-search step of 32 sentences x beam 5; fp32 accumulators in registers): a CTA reads its
// weight tile once and the activations once per k-block.  One TMA producer warp feeds a ring of [128 x 64 weights |
// N x 64 activations] stages; the activation box is N rows, zero-filled past the last row, and the MMA columns beyond
// the rows are never stored.  Two kernels share the producer, the ring and the consumers' k-loop:
//
// decode_gemm_kernel (sb_gemm_decode): the six weight products of a decoder layer.  Replaces Linear_forward
// (fairseq2.cpp:251) in StandardTransformerDecoderLayer_forward (fairseq2.cpp:979-1094): self-attention q|k|v and
// output, cross-attention q and output, FFN inner and output.  One (tile, K-slice) unit per CTA.
//   split-K mode : slice z writes raw fp32 partial products to partials[(z * slice_rows + row) * n + feature]
//                  (same contract as sb_gemm_splitk; reduced by sb_splitk_reduce_ln or the attention kernels)
//   direct mode  : out[row * out_ld + feature] = act(acc + bias) in fp16, act in {none, relu}
// Bytes per call at a beam-search step of 160 rows (seamlessM4T_large, at the K slices of ops.decode_splits):
//   product              n x k        tiles x splits   weights (HBM)  activations (L2 -> SM)  fp32 partials written
//   self-attn q|k|v   3072 x 1024        24 x 2   =  48     6.3 MB          7.9 MB                3.9 MB
//   attn out / cross q 1024 x 1024        8 x 8   =  64     2.1 MB          2.6 MB                5.2 MB
//     / cross out
//   FFN inner         8192 x 1024        64 x 1   =  64    16.8 MB         21.0 MB                -  (fp16 out 2.6 MB)
//   FFN out           1024 x 8192         8 x 8   =  64    16.8 MB         21.0 MB                5.2 MB
// A slice sums its k-blocks in order with the same m64 x k16 tensor-core steps as the row-major kernel, so at the same
// contiguous K slices the partials are bit-identical to sb_gemm_splitk's (tests/test_decode_gemm.py): the search does
// not depend on which path runs.  More slices would fill more SMs but change the fp32 sums, and measured no faster at
// 160 rows on an H100: q|k|v 8.5 us at 4 slices against 8.8 at 2; FFN out 12.3 us at 16 against 11.9 at 8.
// Activations: tiles x rows x k x 2 B (each (tile, slice) unit reads its K slice of all rows once), so L2 -> SM traffic is
// weights + activations = 2.25x the weight bytes for every product.  FFN inner keeps its fused bias + ReLU at 64 CTAs:
// 64-feature tiles would give 128 CTAs but read the activations twice (42 MB, 3.5x the weights), and splitting K over
// a 2-CTA cluster that adds the halves through distributed shared memory kept the bytes but measured slower on an H100
// (13.5 us per call against 11.8 us for the same kernel at one slice per tile).
// Residency: one CTA per SM.  At N = 160 the 80 fp32 accumulators per consumer thread take the kernel to 106 registers
// (no spills); two CTAs of 9 warps per SM would have to fit in 96 per thread, which ptxas refuses for the N = 160 MMA.
// So the ring takes the SM's shared memory, up to the K slice: a CTA streams at ~77 GB/s with 3 stages (108 KB) in
// flight and ~92 GB/s with 6 (measured on an H100 SXM, 700 W), and the next kernel's weights are pulled into L2
// instead of being loaded by a co-resident CTA (DgArgs::prefetch).  The epilogue stages the tile in the drained ring.
//
// vocab_proj_kernel (sb_gemm with tile_stats): the tied vocabulary projection logits[r][v] = h[r] . E[v] (fp32) with
// per-(row, 128-column tile) log-softmax statistics, against the whole 256102 x 1024 embedding.  One CTA per SM walks
// the 2001 vocabulary tiles and the producer keeps the ring running across tiles, so the next tile's weights stream
// while the consumers run the epilogue in a staging buffer of their own.  At 160 rows a step moves 0.52 GB of weights
// once from HBM and 0.66 GB of h L2 -> SM, and writes 164 MB of logits.  Registers: a 9-warp CTA gets at most 168 per
// thread; N = 160 uses 167 with no spills, N = 256 (161-256 rows) spills 68 bytes in the epilogue.
// Epilogue, per 64-feature half of the tile: the warpgroup that holds it writes (acc + bias) * alpha * gamma into an
// fp32 staging buffer laid out as the output ([row][32 features] groups, 128B-swizzled), one thread issues the TMA
// stores, and every thread owns one row and folds the half into the row's running (max, sum exp) exactly as
// gemm_tc_kernel's epilogue does: 32-column chunks in ascending order, the same running max / __expf merge.  With the K
// order also unchanged (16 k-blocks of 64, k16 steps in order) the logits and the statistics match the general kernel's
// bit for bit.
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace sb {
namespace {

constexpr int DG_BK = 64;
constexpr int DG_TM = 128;  // weight rows (output features, vocabulary entries) per tile
constexpr int DG_W_BYTES = DG_TM * DG_BK * 2;
constexpr int DG_THREADS = 288;  // warps 0-7 two consumer warpgroups (MMA + epilogue), warp 8 TMA producer
constexpr int DG_MAX_STAGES = 8;
constexpr int DG_SMEM_MISC = 1024 + 2 * DG_MAX_STAGES * 8;  // alignment slack + barriers
// the products' CTAs reserve 384 bytes they do not use: their footprint decides which other streams' kernels can share
// an SM under lanes, and the lanes' throughput has only been measured at this footprint
constexpr int DG_PRODUCTS_SLACK = 384;
constexpr int DG_SP = DG_TM + 4;                             // row pitch (floats) of the products' staging tile

struct DgArgs {
  int rows, n_out, kb_total, stages;
  int splits, relu;  // products
  int tiles;         // projection
  const float* bias;
  float* partials;
  long long slice_rows;
  elem_t* out;
  long long out_ld;
  const char* prefetch;  // the next kernel's weights: pulled into L2 by the producer warp once its loads are issued
  long long prefetch_bytes;
  float post_scale;  // projection: logits = (acc + bias) * post_scale
  float2* tile_stats;
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // warps 0-7

// Shared memory: `stages` ring stages, `extra` bytes (the projection's staging buffer), the full / empty barriers.
template <int NT>
struct Ring {
  static constexpr int STAGE_BYTES = DG_W_BYTES + NT * DG_BK * 2;
  static constexpr int GROUP_BYTES = NT * 128;           // projection: [NT rows][32 fp32], one TMA store box
  static constexpr int STAGING_BYTES = 2 * GROUP_BYTES;  // projection: one 64-feature half of a tile
  static_assert(NT % 16 == 0 && NT <= 256, "wgmma N");

  uint8_t* smem;
  uint64_t *full, *empty;
  int stages, s = 0;
  uint32_t ph = 0;

  __device__ Ring(uint8_t* raw, int n, int extra)
      : smem((uint8_t*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023)),
        full((uint64_t*)(smem + (size_t)n * STAGE_BYTES + extra)),
        empty(full + DG_MAX_STAGES),
        stages(n) {}

  // thread 0, before the CTA's first __syncthreads
  __device__ __forceinline__ void init(const CUtensorMap* tmW, const CUtensorMap* tmX, const CUtensorMap* tmO) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmW)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmX)) : "memory");
    if (tmO != nullptr) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmO)) : "memory");
    for (int i = 0; i < stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  __device__ __forceinline__ void advance() {
    if (++s == stages) { s = 0; ph ^= 1; }
  }

  // Producer warp: k-blocks [kb0, kb1) of weight tile `tile` and of the activations.  Weights first: they do not depend
  // on the upstream kernel, so under PDL they stream while it still runs; `waited` carries the one pdl_wait across tiles.
  __device__ __forceinline__ void produce(const CUtensorMap& tmW, const CUtensorMap& tmX, int tile, int kb0, int kb1,
                                          bool& waited) {
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&empty[s], ph ^ 1);
      uint8_t* st = smem + (size_t)s * STAGE_BYTES;
      if (elect_one()) {
        mbar_expect_tx(&full[s], STAGE_BYTES);
        tma_load_2d(st, &tmW, &full[s], kb * DG_BK, tile * DG_TM);
        if (!waited) pdl_wait();
        tma_load_2d(st + DG_W_BYTES, &tmX, &full[s], kb * DG_BK, 0);
      }
      waited = true;
      __syncwarp();
      advance();
    }
  }

  // Consumer warpgroups: acc = D[feature][row] = W[64 features of warpgroup wg] . X[NT rows]^T over k-blocks [kb0, kb1).
  // A stage is released once the next stage's MMAs are issued; the last one is returned unreleased.
  __device__ __forceinline__ int consume(float (&acc)[NT / 2], int kb0, int kb1) {
    const int wg = threadIdx.x >> 7;
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    int prev = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * STAGE_BYTES);
      const uint64_t da = make_smem_desc(sa + wg * 64 * 128), db = make_smem_desc(sa + DG_W_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < DG_BK / 16; ++k) Wgmma<NT>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
      wg_commit();
      wg_wait<1>();
      wg_fence_regs(acc);
      if (kb > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      prev = s;
      advance();
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    return prev;
  }
};

template <int NT>
__global__ void __launch_bounds__(DG_THREADS, 1)
decode_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const DgArgs g) {
  extern __shared__ uint8_t smem_raw[];
  Ring<NT> ring(smem_raw, g.stages, 0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int u = blockIdx.x;
  const int tile = u / g.splits, split = u - tile * g.splits;
  const int kb0 = (g.kb_total * split) / g.splits, kb1 = (g.kb_total * (split + 1)) / g.splits;
  if (threadIdx.x == 0) ring.init(&tmW, &tmX, nullptr);
  __syncthreads();

  if (warp == 8) {
    bool waited = false;
    ring.produce(tmW, tmX, tile, kb0, kb1, waited);
    if (g.prefetch_bytes > 0) {
      constexpr long long CH = 16384;
      const long long share = ((g.prefetch_bytes + gridDim.x - 1) / gridDim.x + 4095) / 4096 * 4096;
      const long long lo = (long long)blockIdx.x * share, hi = min(lo + share, g.prefetch_bytes);
      if (elect_one())
        for (long long o = lo; o < hi; o += CH)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(g.prefetch + o), "r"((uint32_t)min(CH, hi - o)) : "memory");
      __syncwarp();
    }
    return;
  }
  float acc[NT / 2];
  ring.consume(acc, kb0, kb1);
  // both warpgroups are past their last MMA (the other one may still read the last stage): from here the ring is scratch
  consumer_bar();
  // ---- epilogue: register j*4 + 2h + e of the accumulator fragment = (feature fl + 8h, row j*8 + 2*(lane%4) + e).  It
  // goes through shared memory as [row][128 features] (pitch DG_SP floats: the fragment writes hit 32 distinct banks)
  // and leaves as whole rows in 16-byte stores, instead of 4-row x 32-byte scatters
  const int wg = warp >> 2;
  float* stage = reinterpret_cast<float*>(ring.smem);
  const int fl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < NT / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) stage[(j * 8 + (lane & 3) * 2 + e) * DG_SP + fl + 8 * h] = acc[j * 4 + 2 * h + e];
  consumer_bar();
  pdl_sync();
  const int f_tile = tile * DG_TM;
  const int tid = threadIdx.x;
  if (g.partials != nullptr) {
    // 32 chunks of 4 features per row: one warp writes one 512-byte row segment
    const bool vec = (g.n_out & 3) == 0;
    for (int i = tid; i < g.rows * 32; i += 256) {
      const int r = i >> 5, c = (i & 31) * 4, f = f_tile + c;
      if (f >= g.n_out) continue;
      const float4 v = *reinterpret_cast<const float4*>(stage + r * DG_SP + c);
      float* dst = g.partials + ((long long)split * g.slice_rows + r) * g.n_out + f;
      if (vec && f + 4 <= g.n_out) {
        *reinterpret_cast<float4*>(dst) = v;
      } else {
        const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (f + q < g.n_out) dst[q] = x[q];
      }
    }
  } else {
    // 16 chunks of 8 features per row, bias + activation, fp16
    const bool vec = (g.out_ld & 7) == 0 && ((uintptr_t)g.out & 15) == 0;
    for (int i = tid; i < g.rows * 16; i += 256) {
      const int r = i >> 4, c = (i & 15) * 8, f = f_tile + c;
      if (f >= g.n_out) continue;
      const float4 lo = *reinterpret_cast<const float4*>(stage + r * DG_SP + c);
      const float4 hi = *reinterpret_cast<const float4*>(stage + r * DG_SP + c + 4);
      float x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      const int nq = min(8, g.n_out - f);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        x[q] += (g.bias != nullptr && q < nq) ? g.bias[f + q] : 0.f;
        if (g.relu) x[q] = fmaxf(x[q], 0.f);
      }
      elem_t* dst = g.out + (long long)r * g.out_ld + f;
      if (vec && nq == 8) {
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) hv[q] = __floats2half2_rn(x[2 * q], x[2 * q + 1]);
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hv);
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (q < nq) dst[q] = __float2half_rn(x[q]);
      }
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(DG_THREADS, 1)
vocab_proj_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ CUtensorMap tmO, const DgArgs g) {
  using R = Ring<NT>;
  extern __shared__ uint8_t smem_raw[];
  R ring(smem_raw, g.stages, R::STAGING_BYTES);
  uint8_t* staging = ring.smem + (size_t)g.stages * R::STAGE_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) ring.init(&tmW, &tmX, &tmO);
  __syncthreads();

  if (warp == 8) {
    bool waited = false;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) ring.produce(tmW, tmX, tile, 0, g.kb_total, waited);
    return;
  }
  const int wg = warp >> 2;
  const int row = threadIdx.x;  // epilogue: this thread's row of h
  float acc[NT / 2];
  bool synced = false;
  for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
    const int last = ring.consume(acc, 0, g.kb_total);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&ring.empty[last]);
    if (!synced) {
      pdl_sync();  // logits / statistics writes must not overtake the upstream kernel; dependents may launch now
      synced = true;
    }

    // ---- epilogue: half q = features [64 q, 64 q + 64) of the tile, held by warpgroup q
    const int f0 = tile * DG_TM;
    float st_m = -INFINITY, st_s = 0.f;  // running log-sum-exp statistics of this thread's row over the tile
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int fq = f0 + q * 64;
      // the previous half's TMA stores have read the staging buffer and every thread has finished its statistics
      if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      consumer_bar();
      if (wg == q) {
        // register j*4 + 2h + e = (feature (warp & 3) * 16 + lane / 4 + 8h, row j*8 + 2*(lane % 4) + e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int fl = (warp & 3) * 16 + (lane >> 2) + 8 * h;  // feature inside the half
          const int f = fq + fl;
          const float b = (g.bias != nullptr && f < g.n_out) ? g.bias[f] : 0.f;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            // row r = 8j + r0: the swizzle (r & 7 = r0) does not depend on j, so j only adds an immediate 1 KB offset
            const int r0 = (lane & 3) * 2 + e;
            float* p = reinterpret_cast<float*>(staging + (fl >> 5) * R::GROUP_BYTES + r0 * 128 + ((((fl & 31) >> 2) ^ r0) << 4) +
                                                (fl & 3) * 4);
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) p[j * 256] = (acc[j * 4 + 2 * h + e] + b) * g.post_scale;
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      }
      consumer_bar();
      if (threadIdx.x == 0) {
        for (int c = 0; c < 2; ++c)
          if (fq + 32 * c < g.n_out) tma_store_2d(&tmO, staging + c * R::GROUP_BYTES, fq + 32 * c, 0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      if (g.tile_stats != nullptr && row < g.rows) {
#pragma unroll 1
        for (int c = 0; c < 2; ++c) {
          const int oc = fq + 32 * c;
          if (oc >= g.n_out) break;
          float v[32];
          const uint8_t* ap = staging + c * R::GROUP_BYTES + row * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 a = *reinterpret_cast<const float4*>(ap + ((j ^ (row & 7)) << 4));
            v[4 * j] = a.x; v[4 * j + 1] = a.y; v[4 * j + 2] = a.z; v[4 * j + 3] = a.w;
          }
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < 32; ++j) if (oc + j < g.n_out) cm = fmaxf(cm, v[j]);
          if (cm > -INFINITY) {
            const float nm = fmaxf(st_m, cm);
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) if (oc + j < g.n_out) sum += __expf(v[j] - nm);
            st_s = st_s * __expf(st_m - nm) + sum;
            st_m = nm;
          }
        }
        if (q == 1) g.tile_stats[(long long)tile * g.rows + row] = make_float2(st_m, st_s);
      }
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Shapes both kernels take: one tap, dense rows from row 0, whole k-blocks, no GLU / residual / second output /
// sequence masking, 1-256 rows, 16-byte aligned operands.
bool wt_supported(const sb_gemm_t* g) {
  return g != nullptr && g->taps == 1 && g->m >= 1 && g->m <= 256 && g->c_in % DG_BK == 0 && g->a_row0 == 0 && !g->glu &&
         (g->a_ld % 8) == 0 && ((uintptr_t)g->a % 16) == 0 && ((uintptr_t)g->w % 16) == 0 && g->res1 == nullptr &&
         g->res2 == nullptr && g->out2 == nullptr && g->seq_rows == 0;
}

bool dg_supported(const sb_gemm_t* g, int splits) { return wt_supported(g) && splits >= 1 && splits <= g->c_in / DG_BK; }

// Ring depth, shared memory, tensor maps and launch of either kernel at wgmma N = NT.  The ring is as deep as the
// opt-in shared memory allows; the products cap it at their K slice and raise it to hold their epilogue's staging
// tile, which reuses the drained ring.
template <int NT>
int wt_launch(const sb_gemm_t* g, DgArgs a, bool proj, cudaStream_t st) {
  using R = Ring<NT>;
  int dev = 0, smem_optin = 0;
  SB_CUDA_OK(cudaGetDevice(&dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int extra = proj ? R::STAGING_BYTES : DG_PRODUCTS_SLACK;
  const int tiles = (g->n + DG_TM - 1) / DG_TM;
  int stages = (smem_optin - DG_SMEM_MISC - extra) / R::STAGE_BYTES;
  if (stages > DG_MAX_STAGES) stages = DG_MAX_STAGES;
  int grid;
  if (proj) {
    SB_REQUIRE(stages >= 2, SB_ENOSUP, "vocabulary projection: not enough shared memory for %d rows", g->m);
    grid = tiles < sm_count() ? tiles : sm_count();
  } else {
    const int kb_max = (a.kb_total + a.splits - 1) / a.splits;
    if (stages > kb_max) stages = kb_max;
    const int epi_bytes = NT * DG_SP * 4;
    if (stages * R::STAGE_BYTES < epi_bytes) stages = (epi_bytes + R::STAGE_BYTES - 1) / R::STAGE_BYTES;
    if (stages < 2) stages = 2;
    grid = tiles * a.splits;
  }
  a.stages = stages;
  a.tiles = tiles;
  const size_t smem = (size_t)stages * R::STAGE_BYTES + extra + DG_SMEM_MISC;
  CUtensorMap tmW, tmX, tmO;
  int rc = make_tmap(&tmW, g->w, (uint64_t)g->c_in, (uint64_t)g->n, (uint64_t)g->c_in, DG_TM);
  if (rc == SB_OK) rc = make_tmap(&tmX, g->a, (uint64_t)g->c_in, (uint64_t)g->m, (uint64_t)g->a_ld, NT);
  if (rc == SB_OK && proj) rc = make_tmap(&tmO, g->out, (uint64_t)g->n, (uint64_t)g->m, (uint64_t)g->out_ld, NT, 4);
  if (rc) return rc;
  static size_t configured[2] = {0, 0};  // per NT, for each kernel
  if (smem > configured[proj]) {
    const void* k = proj ? (const void*)vocab_proj_kernel<NT> : (const void*)decode_gemm_kernel<NT>;
    SB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[proj] = smem;
  }
  SB_CUDA_OK(proj ? launch_k(vocab_proj_kernel<NT>, dim3(grid), dim3(DG_THREADS), smem, st, tmW, tmX, tmO, a)
                  : launch_k(decode_gemm_kernel<NT>, dim3(grid), dim3(DG_THREADS), smem, st, tmW, tmX, a));
  count_launch();
  return SB_OK;
}

int wt_run(const sb_gemm_t* g, const DgArgs& a, bool proj, cudaStream_t st) {
  if (g->m <= 32) return wt_launch<32>(g, a, proj, st);
  if (g->m <= 64) return wt_launch<64>(g, a, proj, st);
  if (g->m <= 128) return wt_launch<128>(g, a, proj, st);
  if (g->m <= 160) return wt_launch<160>(g, a, proj, st);
  return wt_launch<256>(g, a, proj, st);
}

}  // namespace

bool vocab_proj(const sb_gemm_t* g, cudaStream_t st, int* rc) {
  if (!(wt_supported(g) && g->tile_stats != nullptr && g->act == SB_ACT_NONE && g->out_row0 == 0 && g->out_f32 &&
        g->prefetch == nullptr && ((uintptr_t)g->out % 16) == 0 && (g->out_ld % 4) == 0))
    return false;
  DgArgs a = {};
  a.rows = g->m;
  a.n_out = g->n;
  a.kb_total = g->c_in / DG_BK;
  a.bias = g->bias;
  a.post_scale = g->alpha * g->gamma;
  a.tile_stats = (float2*)g->tile_stats;
  *rc = wt_run(g, a, true, st);
  return true;
}

}  // namespace sb

extern "C" int sb_gemm_decode_supported(const sb_gemm_t* g, int32_t splits) { return sb::dg_supported(g, splits) ? 1 : 0; }

extern "C" int sb_gemm_decode(const sb_gemm_t* g, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(dg_supported(g, splits), SB_ENOSUP, "sb_gemm_decode: shape not supported (rows <= 256, taps 1, c_in %% 64 == 0, no GLU / residual)");
  SB_REQUIRE(partials != nullptr || (splits == 1 && g->out != nullptr && !g->out_f32 && (g->act == SB_ACT_NONE || g->act == SB_ACT_RELU)),
             SB_EINVAL, "sb_gemm_decode: direct mode needs splits == 1, an fp16 output and act in {none, relu}");
  SB_REQUIRE(partials == nullptr || slice_rows >= g->m, SB_EINVAL, "sb_gemm_decode: slice_rows (%lld) < m (%d)", (long long)slice_rows, g->m);
  DgArgs a = {};
  a.rows = g->m;
  a.n_out = g->n;
  a.kb_total = g->c_in / DG_BK;
  a.splits = splits;
  a.relu = g->act == SB_ACT_RELU;
  a.bias = g->bias;
  a.partials = partials;
  a.slice_rows = slice_rows;
  a.out = (elem_t*)g->out;
  a.out_ld = g->out_ld;
  a.prefetch = (const char*)g->prefetch;
  a.prefetch_bytes = g->prefetch ? g->prefetch_bytes / 4096 * 4096 : 0;
  return wt_run(g, a, false, (cudaStream_t)stream);
}
