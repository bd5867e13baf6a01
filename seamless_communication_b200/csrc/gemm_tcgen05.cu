// sb_gemm: fused Linear / Conv1d-as-GEMM for sm_90a.
//
//   TMA (cp.async.bulk.tensor, 128B swizzle) -> 3/4-stage smem ring -> wgmma (m64nBNk16, fp16 in, fp32 accumulate in
//   registers of two consumer warpgroups, 64 tile rows each) -> fp32 tile staged in the drained ring -> epilogue (bias,
//   activation / GLU, residuals, sequence mask, fp16|fp32 store, optional leaky-relu'd second output).
//
// Warp roles: warps 0-7 consumers (warpgroup = 64 tile rows; warps 0-3 then run the epilogue, one tile row per
// thread), warp 8 TMA producer.  One 128 x BN output tile per CTA; up to BN = 128 two CTAs co-reside per SM so one
// CTA's epilogue overlaps the other's main loop.  The epilogue stages the output tile in shared memory (128B-swizzled,
// conflict free) and writes it with TMA bulk stores (full 128 B rows; tile tails are clipped by the tensor map).
//
// Conv taps are realised purely through the TMA row coordinate: tap j of output row m reads A row
// a_row0 + m + j*dil, the weight K index is j*c_in + c.  Rows outside [0, a_rows) and channels >= c_in are
// zero-filled by TMA, so c_in need not be a multiple of 64.
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace sb {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 fp16 = 128 B = one swizzle atom row
constexpr int A_TILE_BYTES = BM * BK * 2;

struct GemmArgs {
  int m, n, c_in, taps, dil, a_row0;
  const float* bias;
  int act;
  float act_slope;
  int glu;
  float alpha, gamma;
  const elem_t* res1;
  long long res1_ld;
  const elem_t* res2;
  long long res2_ld;
  void* out;
  long long out_ld;
  int out_f32;
  elem_t* out2;
  long long out2_ld;
  float out2_slope;
  long long out_row0;
  int seq_rows, seq_halo, seq_len;
  const int* seq_lens;
  int tma_store;  // epilogue through smem + cp.async.bulk.tensor stores
  int m_fast;  // skinny-M problems: blockIdx.x walks the M tiles so CTAs sharing a weight tile are co-scheduled (L2 reuse)
  int kb_per_split;  // split-K: k-blocks per blockIdx.z slice (0 = no split)
  long long slice_rows;  // split-K: slice z writes rows [z*slice_rows, z*slice_rows + m) of out
  float2* tile_stats;    // optional [n tiles][m]: (max, sum exp(x - max)) of every output row over this CTA's BN columns
  const char* prefetch;  // weights of the kernel that follows: pulled into L2 by the idle epilogue warp during the main loop
  long long prefetch_bytes;
  unsigned long long* argmin;  // sb_nearest_centroid: per row atomicMin of (orderable -2 v bits << 32 | column); no stores
};

template <int BN>
struct TileCfg {
  // BN <= 128: two CTAs per SM (<= 113 KB of shared memory each) so that one CTA's epilogue overlaps the other's main
  // loop.  BN = 256: every A tile feeds twice the columns (85 instead of 64 FLOP per byte moved L2 -> SM); its 128 x 256
  // fp32 accumulator needs 128 registers per consumer thread and 128 KB of staging, so it runs one CTA per SM.
  static constexpr int STAGES = BN >= 128 ? 3 : 4;
  static constexpr int MIN_CTAS = BN >= 256 ? 1 : 2;
  static constexpr int B_TILE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + BN * 4;
  static constexpr int THREADS = 32 * 9;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
  // After the main loop the drained ring holds the fp32 accumulator tile: 16 KB chunks of [128 rows][32 columns], 16-byte
  // units XOR (row & 7).  The epilogue stages its outputs in place (out groups of chunk c land in chunks <= c of the same
  // row, already read by the thread that owns the row); out2 groups follow the accumulator chunks.
  // fp32 worst case: 32 columns per 16 KB group; the 256-wide tile stages fp16 outputs only (no fp32 / second output: the
  // host never selects it for those)
  static constexpr int OUT_GROUPS_MAX = BN >= 256 ? BN * 2 / 128 : BN * 4 / 128;
  static constexpr int OUT2_OFFSET = OUT_GROUPS_MAX * 16384;
  static_assert(BM * BN * 4 <= STAGES * STAGE_BYTES, "accumulator staging does not fit");
  static_assert(BN >= 256 || OUT2_OFFSET + (BN / 64 > 0 ? BN / 64 : 1) * 16384 <= STAGES * STAGE_BYTES, "staging does not fit");
};

__device__ unsigned long long* g_timeline = nullptr;
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define TL(i) do { if (g_timeline != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) g_timeline[i] = gtime(); } while (0)

template <int BN>
__global__ void __launch_bounds__(TileCfg<BN>::THREADS, TileCfg<BN>::MIN_CTAS)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmO2, const GemmArgs g) {
  using Cfg = TileCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* bias_s = (float*)(smem + STAGES * Cfg::STAGE_BYTES + 256);

  if (threadIdx.x == 0) {
    TL(0);
    // hide the descriptor fetch of the first TMA behind the barrier setup
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    if (g.tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (g.m_fast ? blockIdx.y : blockIdx.x) * BN;
  const int m0 = (g.m_fast ? blockIdx.x : blockIdx.y) * BM;
  const int cblocks = (g.c_in + BK - 1) / BK;
  const int kb_total = g.taps * cblocks;
  const int kb_begin = g.kb_per_split > 0 ? blockIdx.z * g.kb_per_split : 0;
  const int kb_stop = g.kb_per_split > 0 ? min(kb_total, kb_begin + g.kb_per_split) : kb_total;
  const int kblocks = kb_stop - kb_begin;  // k-blocks of this CTA

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp < 4) {
    for (int i = threadIdx.x; i < BN; i += 128) {
      int n = n0 + i;
      bias_s[i] = (g.bias != nullptr && n < g.n) ? g.bias[n] : 0.f;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) TL(1);

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    int s = 0;
    uint32_t ph = 0;
    for (int kr = 0; kr < kblocks; ++kr) {
      mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
      const int kb = kb_begin + kr;
      const int tap = kb / cblocks, c0 = (kb - tap * cblocks) * BK;
      if (elect_one()) {
        if (kr == 0) TL(2);
        mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
        // weights first: they do not depend on the upstream kernel, so under PDL they stream while it still runs
        tma_load_2d(sa + A_TILE_BYTES, &tmW, &full_bar[s], tap * g.c_in + c0, n0);
        if (kr == 0) pdl_wait();
        tma_load_2d(sa, &tmA, &full_bar[s], c0, m0 + g.a_row0 + tap * g.dil);
      }
      __syncwarp();
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    if (g.prefetch_bytes > 0) {
      // latency-bound chains (decoder step): the next GEMM's weights do not depend on this kernel's result, so each CTA
      // asks L2 for its share once its own loads are issued; the next kernel's first TMA loads then hit L2 instead of
      // paying an HBM round trip (one elected lane issues, in 16 KB pieces of this CTA's contiguous share)
      constexpr long long CH = 16384;
      const long long cta = blockIdx.x + (long long)gridDim.x * (blockIdx.y + (long long)gridDim.y * blockIdx.z);
      const long long ncta = (long long)gridDim.x * gridDim.y * gridDim.z;
      const long long share = ((g.prefetch_bytes + ncta - 1) / ncta + 4095) / 4096 * 4096;
      const long long lo = cta * share, hi = min(lo + share, g.prefetch_bytes);
      if (elect_one()) {
        for (long long o = lo; o < hi; o += CH)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(g.prefetch + o), "r"((uint32_t)min(CH, hi - o)) : "memory");
      }
      __syncwarp();
    }
    return;
  }
  // -------------------------------------------------------------------- consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
  {
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0, prev = 0;
    uint32_t ph = 0;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(&full_bar[s], ph);
      const uint32_t sa = smem_u32(smem + s * Cfg::STAGE_BYTES);
      const uint64_t da = make_smem_desc(sa + wg * (BM / 2) * 128), db = make_smem_desc(sa + A_TILE_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
      wg_commit();
      // the previous k-block's MMAs have read their stage once at most this block's group is in flight.  (Channels past
      // c_in are zero-filled by TMA, so a partial last channel block contributes exact zeros.)
      wg_wait<1>();
      wg_fence_regs(acc);
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (threadIdx.x == 0) TL(3);
    // every MMA of both warpgroups has read the ring: it now stages the fp32 tile (layout: see TileCfg)
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h, col = j * 8 + (lane & 3) * 2;
        *reinterpret_cast<float2*>(smem + (col >> 5) * 16384 + r * 128 + ((((col & 31) >> 2) ^ (r & 7)) << 4) + (col & 3) * 4) =
            make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
  if (warp >= 4) return;
  {
    // ------------------------------------------------------------------ epilogue (warps 0..3, one tile row per thread)
    pdl_sync();  // residual reads / output writes below must not overtake the upstream kernel; dependents may launch now
    if (threadIdx.x == 0) TL(4);
    const int row = warp * 32 + lane;
    const long long m = (long long)m0 + row;
    const bool row_ok = m < g.m;
    const long long q = m + g.out_row0 + (g.kb_per_split > 0 ? (long long)blockIdx.z * g.slice_rows : 0);
    const bool valid = row_ok && seq_row_valid(q, g.seq_rows, g.seq_halo, g.seq_len, g.seq_lens);
    const int n_out_total = g.glu ? g.n / 2 : g.n;
    // NOTE: every access to v[] below uses compile-time indices (fully unrolled loops with predicates); a single
    // runtime-indexed access would push the whole array to local memory.
    const bool has_res = valid && (g.res1 != nullptr || g.res2 != nullptr);
    const float post_scale = has_res ? g.gamma : g.alpha * g.gamma;
    float st_m = -INFINITY, st_s = 0.f;  // running log-sum-exp statistics of this thread's row (tile_stats)
    unsigned long long best = ~0ull;      // argmin mode: this row's best (distance, column) over the tile
#pragma unroll 1
    for (int c0 = 0; c0 < BN; c0 += 32) {
      if (n0 + c0 >= g.n) break;  // warp-uniform
      float v[32];
      const uint8_t* ap = smem + (c0 >> 5) * 16384 + row * 128;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(ap + ((j ^ (row & 7)) << 4));
        v[4 * j] = a.x + bias_s[c0 + 4 * j];
        v[4 * j + 1] = a.y + bias_s[c0 + 4 * j + 1];
        v[4 * j + 2] = a.z + bias_s[c0 + 4 * j + 2];
        v[4 * j + 3] = a.w + bias_s[c0 + 4 * j + 3];
      }
      if (!row_ok) continue;
      int nv = 32;         // number of output values in this chunk
      int oc = n0 + c0;    // first output column
      if (g.glu) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = __fdividef(v[2 * j], 1.f + __expf(-v[2 * j + 1]));
        nv = 16;
        oc = (n0 + c0) >> 1;
      } else if (g.act == SB_ACT_RELU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
      } else if (g.act == SB_ACT_SILU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __fdividef(v[j], 1.f + __expf(-v[j]));
      } else if (g.act == SB_ACT_LRELU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * g.act_slope;
      } else if (g.act == SB_ACT_TANH) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = tanhf(v[j]);
      } else if (g.act == SB_ACT_GELU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
      }
      if (g.argmin != nullptr) {
        // v = x.c - |c|^2 / 2, so -2 v = |c|^2 - 2 x.c exactly (a power-of-two scale); the packed key orders by distance,
        // then by column, and the running minimum over this row's chunks keeps the lowest column of equal distances
        if (valid) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            if (oc + j < g.n) {
              const unsigned int u = __float_as_uint(-2.f * v[j]);
              const unsigned int key = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
              const unsigned long long pk = ((unsigned long long)key << 32) | (unsigned int)(oc + j);
              best = pk < best ? pk : best;
            }
          }
        }
        continue;
      }
      const bool full = (oc + nv <= n_out_total);
      if (has_res) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] *= g.alpha;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const elem_t* rp = t == 0 ? g.res1 : g.res2;
          const long long rl = t == 0 ? g.res1_ld : g.res2_ld;
          if (rp == nullptr) continue;
          const elem_t* p = rp + q * rl + oc;
          if (full && ((rl | oc) & 7) == 0) {
#pragma unroll
            for (int j8 = 0; j8 < 4; ++j8) {
              if (8 * j8 < nv) {
                const uint4 u = *reinterpret_cast<const uint4*>(p + 8 * j8);
                const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 f = __half22float2(h[e]);
                  v[8 * j8 + 2 * e] += f.x;
                  v[8 * j8 + 2 * e + 1] += f.y;
                }
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (j < nv && oc + j < n_out_total) v[j] += __half2float(p[j]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = valid ? v[j] * post_scale : 0.f;
      if (g.tile_stats != nullptr) {
        // per (row, column tile) softmax statistics of what is being stored: the consumer (sb_logits_topk_tiles) gets the
        // row's log-sum-exp and the tiles that can hold its top-K without reading the logits back
        float cm = -INFINITY;
#pragma unroll
        for (int j = 0; j < 32; ++j) if (j < nv && oc + j < n_out_total) cm = fmaxf(cm, v[j]);
        if (cm > -INFINITY) {
          const float nm = fmaxf(st_m, cm);
          float acc = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) if (j < nv && oc + j < n_out_total) acc += __expf(v[j] - nm);
          st_s = st_s * __expf(st_m - nm) + acc;
          st_m = nm;
        }
      }
      // stores
      if (g.tma_store) {
        // stage into shared memory: 16 KB groups of [128 rows][128 B], 16-byte chunk index XOR (row & 7) (SWIZZLE_128B)
        const int rsw = row & 7;
        const int oc_local = g.glu ? (c0 >> 1) : c0;  // first output column of this chunk inside the tile
        if (g.out_f32) {
          uint8_t* gb = smem + (oc_local >> 5) * 16384 + row * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(gb + ((j ^ rsw) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        } else {
          uint8_t* gb = smem + (oc_local >> 6) * 16384 + row * 128;
          const int cb = (oc_local & 63) >> 3;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (8 * j < nv) {
              uint4 u;
              __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
              for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[8 * j + 2 * e], v[8 * j + 2 * e + 1]);
              *reinterpret_cast<uint4*>(gb + (((cb + j) ^ rsw) << 4)) = u;
            }
          }
        }
        if (g.out2 != nullptr) {
          uint8_t* gb = smem + Cfg::OUT2_OFFSET + (oc_local >> 6) * 16384 + row * 128;
          const int cb = (oc_local & 63) >> 3;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (8 * j < nv) {
              uint4 u;
              __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float a = v[8 * j + 2 * e], b = v[8 * j + 2 * e + 1];
                h[e] = __floats2half2_rn(a > 0.f ? a : a * g.out2_slope, b > 0.f ? b : b * g.out2_slope);
              }
              *reinterpret_cast<uint4*>(gb + (((cb + j) ^ rsw) << 4)) = u;
            }
          }
        }
        continue;
      }
      // direct (per-thread row) stores: small tiles / unaligned outputs
      if (g.out_f32) {
        float* p = reinterpret_cast<float*>(g.out) + q * g.out_ld + oc;
        if (full && ((g.out_ld | oc) & 3) == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (4 * j < nv) *reinterpret_cast<float4*>(p + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (j < nv && oc + j < n_out_total) p[j] = v[j];
        }
      } else {
        elem_t* p = reinterpret_cast<elem_t*>(g.out) + q * g.out_ld + oc;
        if (full && ((g.out_ld | oc) & 7) == 0) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (8 * j < nv) {
              uint4 u;
              __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
              for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[8 * j + 2 * e], v[8 * j + 2 * e + 1]);
              *reinterpret_cast<uint4*>(p + 8 * j) = u;
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (j < nv && oc + j < n_out_total) p[j] = __float2half_rn(v[j]);
        }
      }
      if (g.out2 != nullptr) {
        elem_t* p = g.out2 + q * g.out2_ld + oc;
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nv && oc + j < n_out_total) p[j] = __float2half_rn(v[j] > 0.f ? v[j] : v[j] * g.out2_slope);
      }
    }
    if (g.tile_stats != nullptr && row_ok) g.tile_stats[(long long)(n0 / BN) * g.m + m] = make_float2(st_m, st_s);
    if (g.argmin != nullptr && best != ~0ull) atomicMin(g.argmin + m, best);
    if (g.tma_store) {
      // make the staged tile visible to the async proxy, then one thread issues the bulk tensor stores
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 2, 128;" ::: "memory");
      if (threadIdx.x == 0) {
        const int n_tile_out = g.glu ? BN / 2 : BN;
        const int oc0 = g.glu ? (n0 >> 1) : n0;
        const int q0 = (int)(m0 + g.out_row0 + (g.kb_per_split > 0 ? (long long)blockIdx.z * g.slice_rows : 0));
        const int gcols = g.out_f32 ? 32 : 64;
        for (int c = 0; c < n_tile_out; c += gcols)
          if (oc0 + c < n_out_total) tma_store_2d(&tmO, smem + (c / gcols) * 16384, oc0 + c, q0);
        if (g.out2 != nullptr)
          for (int c = 0; c < n_tile_out; c += 64)
            if (oc0 + c < n_out_total) tma_store_2d(&tmO2, smem + Cfg::OUT2_OFFSET + (c / 64) * 16384, oc0 + c, q0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      }
    }
  }
  if (threadIdx.x == 0) TL(5);
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2D tensor (inner = channels, outer = rows), box box_cols x box_rows (box_cols * esize = 128 B), 128B swizzle, OOB -> 0.
// esize 1 (e4m3 weight bytes): box 64 x box_rows, unswizzled 64-byte rows.
int make_tmap(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint64_t ld_elems, uint32_t box_rows,
              int esize) {
  EncodeTiledFn fn = get_encode_fn();
  SB_REQUIRE(fn != nullptr, SB_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld_elems * (uint64_t)esize};
  cuuint32_t box[2] = {(cuuint32_t)(esize == 1 ? 64 : 128 / esize), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  esize == 1 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_REQUIRE(r == CUDA_SUCCESS, SB_ECUDA, "cuTensorMapEncodeTiled failed (%d): inner=%llu rows=%llu ld=%llu esize=%d", (int)r,
             (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)ld_elems, esize);
  return SB_OK;
}

// SMs of the current device (tile-size choice); cached per device
int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

static int validate(const sb_gemm_t* g) {
  SB_REQUIRE(g != nullptr && g->a != nullptr && g->w != nullptr && g->out != nullptr, SB_EINVAL, "sb_gemm: null operand");
  SB_REQUIRE(g->m > 0 && g->n > 0 && g->c_in > 0 && g->taps > 0, SB_EINVAL, "sb_gemm: bad shape m=%d n=%d c_in=%d taps=%d",
             g->m, g->n, g->c_in, g->taps);
  SB_REQUIRE((g->a_ld % 8) == 0 && (g->c_in % 8) == 0, SB_ENOSUP, "sb_gemm: a_ld (%lld) and c_in (%d) must be multiples of 8",
             (long long)g->a_ld, g->c_in);
  SB_REQUIRE(((uintptr_t)g->a % 16) == 0 && ((uintptr_t)g->w % 16) == 0, SB_EINVAL, "sb_gemm: operands must be 16B aligned");
  // the direct-store epilogue's 16-byte residual loads and output stores check only ld and the column for alignment
  SB_REQUIRE(((uintptr_t)g->out % 16) == 0 && ((uintptr_t)g->out2 % 16) == 0 && ((uintptr_t)g->res1 % 16) == 0 &&
                 ((uintptr_t)g->res2 % 16) == 0,
             SB_EINVAL, "sb_gemm: out, out2, res1 and res2 must be 16B aligned");
  SB_REQUIRE(g->m <= 65535 * BM, SB_EINVAL, "sb_gemm: m (%d) exceeds %d rows (65535 row tiles)", g->m, 65535 * BM);
  SB_REQUIRE(!g->glu || (g->n % 2) == 0, SB_EINVAL, "sb_gemm: glu needs even n");
  return SB_OK;
}

static void fill_args(const sb_gemm_t* g, GemmArgs* a) {
  a->m = g->m; a->n = g->n; a->c_in = g->c_in; a->taps = g->taps; a->dil = g->dil; a->a_row0 = g->a_row0;
  a->bias = g->bias; a->act = g->act; a->act_slope = g->act_slope; a->glu = g->glu;
  a->alpha = g->alpha; a->gamma = g->gamma;
  a->res1 = (const elem_t*)g->res1; a->res1_ld = g->res1_ld; a->res2 = (const elem_t*)g->res2; a->res2_ld = g->res2_ld;
  a->out = g->out; a->out_ld = g->out_ld; a->out_f32 = g->out_f32;
  a->out2 = (elem_t*)g->out2; a->out2_ld = g->out2_ld; a->out2_slope = g->out2_slope;
  a->out_row0 = g->out_row0;
  a->seq_rows = g->seq_rows; a->seq_halo = g->seq_halo; a->seq_len = g->seq_len; a->seq_lens = g->seq_lens;
  a->tile_stats = (float2*)g->tile_stats;
  a->prefetch = (const char*)g->prefetch; a->prefetch_bytes = g->prefetch ? g->prefetch_bytes / 4096 * 4096 : 0;
  a->argmin = nullptr;
  a->tma_store = 0;
  a->kb_per_split = 0;
  a->slice_rows = 0;
  a->m_fast = 0;
}

template <int BN>
static int launch(const sb_gemm_t* g, cudaStream_t st, int splits = 1, long long slice_rows = 0,
                  unsigned long long* argmin = nullptr) {
  using Cfg = TileCfg<BN>;
  static bool configured = false;
  if (!configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  CUtensorMap tmA, tmW, tmO, tmO2;
  int rc = make_tmap(&tmA, g->a, (uint64_t)g->c_in, (uint64_t)g->a_rows, (uint64_t)g->a_ld, BM);
  if (rc) return rc;
  rc = make_tmap(&tmW, g->w, (uint64_t)g->taps * g->c_in, (uint64_t)g->n, (uint64_t)g->taps * g->c_in, BN);
  if (rc) return rc;
  GemmArgs args;
  fill_args(g, &args);
  // staged TMA-store epilogue needs 128 B output groups (64 fp16 / 32 fp32 columns) and 16 B aligned rows.  The bulk
  // store writes a row's last 16-byte unit whole, so a row that ends inside one (n_out * esize not a multiple of 16)
  // would also overwrite the caller's columns after n_out: such outputs take the direct store.
  const int esize = g->out_f32 ? 4 : 2;
  const int n_tile_out = g->glu ? BN / 2 : BN;
  const int n_out_total = g->glu ? g->n / 2 : g->n;
  bool tma_ok = n_tile_out * esize >= 128 && ((uintptr_t)g->out % 16) == 0 && ((g->out_ld * esize) % 16) == 0 &&
                (n_out_total * esize) % 16 == 0 && g->out_row0 >= 0 && (g->out_row0 + g->m) < (1ll << 31) &&
                !(g->glu && g->out_f32);
  if (g->out2 != nullptr)
    tma_ok = tma_ok && ((uintptr_t)g->out2 % 16) == 0 && ((g->out2_ld * 2) % 16) == 0 && (n_out_total * 2) % 16 == 0 &&
             n_tile_out >= 64;
  static int force_direct = -1;
  if (force_direct < 0) { const char* e = getenv("SB_GEMM_DIRECT_STORE"); force_direct = e ? atoi(e) : 0; }
  if (force_direct) tma_ok = false;
  args.argmin = argmin;
  if (argmin != nullptr) tma_ok = false;  // nothing is stored
  int kb_per = 0;
  if (splits > 1) {
    const int kb_total = g->taps * ((g->c_in + BK - 1) / BK);
    // consumers (sb_splitk_reduce_ln, the decode attention kernels) sum exactly the caller's `splits` slices: an uneven split
    // would leave slices unwritten
    SB_REQUIRE(kb_total % splits == 0, SB_EINVAL, "sb_gemm_splitk: %d k-blocks are not divisible by %d splits", kb_total, splits);
    kb_per = kb_total / splits;
    args.kb_per_split = kb_per;
    args.slice_rows = slice_rows > 0 ? slice_rows : g->m;
    // one tensor map covers all slices, so an M-tail tile of slice z would spill into slice z+1 unless the slice
    // stride is a multiple of the tile height
    if (args.slice_rows % BM != 0) tma_ok = false;
  }
  if (tma_ok) {
    rc = make_tmap(&tmO, g->out, (uint64_t)n_out_total, (uint64_t)(g->out_row0 + (splits > 1 ? args.slice_rows * splits : (long long)g->m)),
                   (uint64_t)g->out_ld, BM, esize);
    if (rc) return rc;
    if (g->out2 != nullptr) {
      rc = make_tmap(&tmO2, g->out2, (uint64_t)n_out_total, (uint64_t)(g->out_row0 + g->m), (uint64_t)g->out2_ld, BM, 2);
      if (rc) return rc;
    } else {
      tmO2 = tmO;
    }
    args.tma_store = 1;
  } else {
    tmO = tmA;
    tmO2 = tmA;
  }
  dim3 grid((g->n + BN - 1) / BN, (g->m + BM - 1) / BM, splits > 1 ? splits : 1);
  if (g->m <= 2 * BM && grid.y > 1) {
    args.m_fast = 1;
    grid = dim3(grid.y, grid.x, grid.z);
  }
  SB_CUDA_OK(launch_k(gemm_tc_kernel<BN>, grid, dim3(Cfg::THREADS), Cfg::SMEM_BYTES, st, tmA, tmW, tmO, tmO2, args));
  count_launch();
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------- CUDA-core cross-check
__global__ void gemm_ref_kernel(const elem_t* __restrict__ A, long long a_rows, long long a_ld, const elem_t* __restrict__ W,
                                const GemmArgs g) {
  const int n_out_total = g.glu ? g.n / 2 : g.n;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)g.m * n_out_total) return;
  const long long m = idx / n_out_total;
  const int oc = (int)(idx - m * n_out_total);
  const long long ktot = (long long)g.taps * g.c_in;
  auto dot = [&](int n) {
    float acc = 0.f;
    for (int t = 0; t < g.taps; ++t) {
      long long r = m + g.a_row0 + (long long)t * g.dil;
      if (r < 0 || r >= a_rows) continue;
      const elem_t* ap = A + r * a_ld;
      const elem_t* wp = W + (long long)n * ktot + (long long)t * g.c_in;
      for (int c = 0; c < g.c_in; ++c) acc += __half2float(ap[c]) * __half2float(wp[c]);
    }
    return acc + (g.bias ? g.bias[n] : 0.f);
  };
  float v;
  if (g.glu) {
    float a = dot(2 * oc), b = dot(2 * oc + 1);
    v = a / (1.f + __expf(-b));
  } else {
    v = apply_act(dot(oc), g.act, g.act_slope);
  }
  const long long q = m + g.out_row0;
  const bool valid = seq_row_valid(q, g.seq_rows, g.seq_halo, g.seq_len, g.seq_lens);
  if (g.res1 != nullptr || g.res2 != nullptr) {
    v *= g.alpha;
    if (g.res1) v += __half2float(g.res1[q * g.res1_ld + oc]);
    if (g.res2) v += __half2float(g.res2[q * g.res2_ld + oc]);
    v *= g.gamma;
  } else {
    v *= g.alpha * g.gamma;
  }
  if (!valid) v = 0.f;
  if (g.out_f32) reinterpret_cast<float*>(g.out)[q * g.out_ld + oc] = v;
  else reinterpret_cast<elem_t*>(g.out)[q * g.out_ld + oc] = __float2half_rn(v);
  if (g.out2) g.out2[q * g.out2_ld + oc] = __float2half_rn(v > 0.f ? v : v * g.out2_slope);
}

}  // namespace sb

extern "C" int sb_gemm(const sb_gemm_t* g_in, sb_stream_t stream) {
  int rc = sb::validate(g_in);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // Narrow-channel undilated convs (HiFi-GAN stages with C = 16/32): the taps of an output row are `taps` consecutive
  // input rows, i.e. one contiguous run of taps*C elements when rows are dense.  Describing A as overlapping rows of
  // that length (row pitch still C) turns `taps` nearly empty 64-deep k-blocks into ceil(taps*C/64) full ones.  TMA
  // zero-fills such a window as a whole, so the collapse applies only when every window lies inside [0, a_rows): a
  // window that starts before row 0 or runs past a_rows keeps the per-tap path, which zero-fills just its outside taps.
  sb_gemm_t gc;
  const sb_gemm_t* g = g_in;
  if (g_in->taps > 1 && g_in->dil == 1 && g_in->c_in < sb::BK && g_in->a_ld == g_in->c_in && g_in->a_row0 >= 0 &&
      (long long)g_in->a_row0 + g_in->m + g_in->taps - 1 <= g_in->a_rows) {
    gc = *g_in;
    gc.c_in = g_in->taps * g_in->c_in;
    gc.taps = 1;
    gc.a_rows = g_in->a_rows - (g_in->taps - 1);
    g = &gc;
  }
  const long long mt = (g->m + sb::BM - 1) / sb::BM;
  const int sms = sb::sm_count();
  auto tiles = [&](int bn) { return mt * ((g->n + bn - 1) / bn); };
  if (g->tile_stats != nullptr) {
    // the statistics are taken of the fp32 values the epilogue stores; an fp16 output would round after them
    SB_REQUIRE(g->out_f32, SB_EINVAL, "sb_gemm: tile_stats needs out_f32");
    SB_REQUIRE(!g->glu && g->n >= 128, SB_ENOSUP, "sb_gemm: tile_stats needs n >= 128 and no GLU");
    // up to 256 rows (a beam-search step): the weight-stationary kernel of decode_gemm.cu, which reads each weight row once.
    // SB_PROJ_T=0 selects the general kernel (read per call: tools compare both inside one process)
    const char* ep = getenv("SB_PROJ_T");
    int rc = SB_OK;
    if ((ep == nullptr || atoi(ep) != 0) && sb::vocab_proj(g, st, &rc)) return rc;
    return sb::launch<128>(g, st);  // the statistics are per 128-column tile (SB_STATS_TILE)
  }
  // 256-wide tiles for the large products (encoder / T2U / vocoder GEMMs): fp16 single-output epilogues, whole tiles only
  const char* e256 = getenv("SB_GEMM_BN256");  // read per call: tools toggle it inside one process
  const int bn256 = (e256 == nullptr || atoi(e256) != 0) ? 1 : 0;
  if (bn256 && (g->n % 256) == 0 && !g->out_f32 && g->out2 == nullptr && tiles(256) >= 2 * sms) return sb::launch<256>(g, st);
  // largest N tile that still gives every SM a CTA; fall back to smaller tiles for skinny problems
  if (g->n >= 128 && tiles(128) >= sms) return sb::launch<128>(g, st);
  if (g->n >= 64 && tiles(64) >= sms) return sb::launch<64>(g, st);
  if (g->n > 64) return sb::launch<64>(g, st);
  return sb::launch<32>(g, st);
}

// split-K: raw fp32 partial products, slice z at rows [z*slice_rows, z*slice_rows + m) of `partials` (ld = n)
extern "C" int sb_gemm_splitk(const sb_gemm_t* g_in, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream) {
  int rc = sb::validate(g_in);
  if (rc) return rc;
  SB_REQUIRE(splits >= 1 && partials != nullptr && !g_in->glu, SB_EINVAL, "sb_gemm_splitk: bad args");
  sb_gemm_t g = *g_in;
  g.bias = nullptr; g.act = SB_ACT_NONE; g.alpha = 1.f; g.gamma = 1.f; g.res1 = nullptr; g.res2 = nullptr;
  g.out = partials; g.out_ld = g.n; g.out_f32 = 1; g.out2 = nullptr; g.out_row0 = 0; g.seq_rows = 0;
  SB_REQUIRE(slice_rows >= g.m, SB_EINVAL, "sb_gemm_splitk: slice_rows (%lld) < m (%d)", (long long)slice_rows, g.m);
  // 64-wide tiles: twice the CTAs and half the (fp32) epilogue per CTA - these problems are latency bound
  return sb::launch<64>(&g, (cudaStream_t)stream, splits, slice_rows);
}

static __global__ void argmin_fill_kernel(unsigned long long* best, int rows) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) best[r] = ~0ull;
}

static __global__ void argmin_finish_kernel(const unsigned long long* best, int rows, int32_t* units) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) units[r] = best[r] == ~0ull ? -1 : (int32_t)(best[r] & 0xffffffffull);
}

extern "C" int sb_nearest_centroid(const void* x, int64_t x_ld, int32_t rows, int32_t dim, const void* centroids,
                                   const float* neg_half_norm, int32_t K, int32_t seq_rows, const int32_t* seq_lens,
                                   uint64_t* best, int32_t* units, sb_stream_t stream) {
  SB_REQUIRE(x && centroids && neg_half_norm && best && units && rows > 0 && K > 0 && dim > 0, SB_EINVAL,
             "sb_nearest_centroid: bad args");
  SB_REQUIRE(seq_rows == 0 || seq_lens != nullptr, SB_EINVAL, "sb_nearest_centroid: seq_rows needs seq_lens");
  sb_gemm_t g = {};
  g.a = x; g.a_rows = rows; g.a_ld = x_ld; g.c_in = dim; g.taps = 1; g.dil = 1; g.a_row0 = 0;
  g.w = centroids; g.n = K; g.m = rows; g.bias = neg_half_norm; g.act = SB_ACT_NONE; g.alpha = 1.f; g.gamma = 1.f;
  g.out = best; g.out_ld = K;
  g.seq_rows = seq_rows; g.seq_halo = 0; g.seq_len = 0; g.seq_lens = seq_lens;
  int rc = sb::validate(&g);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((rows + 255) / 256);
  argmin_fill_kernel<<<blocks, 256, 0, st>>>((unsigned long long*)best, rows);
  SB_LAUNCH_OK();
  rc = sb::launch<128>(&g, st, 1, 0, (unsigned long long*)best);
  if (rc) return rc;
  argmin_finish_kernel<<<blocks, 256, 0, st>>>((const unsigned long long*)best, rows, units);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_gemm_debug_timeline(unsigned long long* buf) {
  SB_CUDA_OK(cudaMemcpyToSymbol(sb::g_timeline, &buf, sizeof(buf)));
  return SB_OK;
}

extern "C" int sb_gemm_ref(const sb_gemm_t* g, sb_stream_t stream) {
  int rc = sb::validate(g);
  if (rc) return rc;
  sb::GemmArgs args;
  sb::fill_args(g, &args);
  const int n_out = g->glu ? g->n / 2 : g->n;
  long long total = (long long)g->m * n_out;
  int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  sb::gemm_ref_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>((const sb::elem_t*)g->a, g->a_rows, g->a_ld,
                                                                            (const sb::elem_t*)g->w, args);
  SB_LAUNCH_OK();
  return SB_OK;
}
