// Tied vocabulary projection of a beam-search step: logits[r][v] = h[r] . E[v] (fp32) and per-(row, 128-column tile)
// log-softmax statistics, for <= 256 rows against the whole 256102 x 1024 embedding.
//
// The general kernel (gemm_tcgen05.cu) makes the rows its MMA M operand in 128-row tiles: at 160 rows every weight tile
// is read by two CTAs and the second row tile is 80 % padding.  Here the weight rows are the wgmma M operand (128 per
// tile, 64 per consumer warpgroup) and all rows of h the N operand (N = rows rounded up to 32, 64, 128, 160 or 256; 160
// is a beam-search step of 32 sentences x beam 5), so each weight byte crosses L2 -> SM once.  One CTA per SM walks
// vocabulary tiles; one TMA producer warp keeps the smem ring running across tiles, so the next tile's weights stream
// while the consumers run the epilogue.  Registers: a 9-warp CTA gets at most 168 per thread; N = 160 uses 167 with no
// spills, N = 256 (161-256 rows) spills 68 bytes in the epilogue.
//
// Epilogue, per 64-feature half of the tile: the warpgroup that holds it writes (acc + bias) * alpha * gamma into an
// fp32 staging buffer laid out as the output ([row][32 features] groups, 128B-swizzled), one thread issues the TMA
// stores, and every thread owns one row and folds the half into the row's running (max, sum exp) exactly as
// gemm_tc_kernel's epilogue does: 32-column chunks in ascending order, the same running max / __expf merge.  With the K
// order also unchanged (16 k-blocks of 64, k16 steps in order) the logits and the statistics match the general kernel's.
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace sb {
namespace {

constexpr int VP_BK = 64;
constexpr int VP_FT = 128;       // vocabulary rows per tile
constexpr int VP_THREADS = 288;  // warps 0-7: two consumer warpgroups (MMA + epilogue), warp 8: TMA producer
constexpr int VP_STAGE_CAP = 8;
constexpr int VP_W_BYTES = VP_FT * VP_BK * 2;

struct VpArgs {
  int m, n, kb_total, tiles, stages;
  const float* bias;
  float post_scale;
  float2* tile_stats;
};

// NT: wgmma N (rows of h, padded).  Shared memory: `stages` ring stages, the staging buffer, the barriers.
template <int NT>
struct VpCfg {
  static constexpr int STAGE_BYTES = VP_W_BYTES + NT * VP_BK * 2;
  static constexpr int GROUP_BYTES = NT * 128;           // [NT rows][32 fp32]: one TMA store box
  static constexpr int STAGING_BYTES = 2 * GROUP_BYTES;  // one 64-feature half of a tile
  static_assert(NT % 16 == 0 && NT <= 256, "wgmma N");
};

template <int NT>
__global__ void __launch_bounds__(VP_THREADS, 1)
vocab_proj_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmH,
                  const __grid_constant__ CUtensorMap tmO, const VpArgs g) {
  using Cfg = VpCfg<NT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* staging = smem + (size_t)g.stages * Cfg::STAGE_BYTES;
  uint64_t* full = (uint64_t*)(staging + Cfg::STAGING_BYTES);
  uint64_t* empty = full + VP_STAGE_CAP;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmH)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    for (int s = 0; s < g.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ---- TMA producer: weights first (they do not depend on the upstream kernel: under PDL they stream while it still runs)
    int s = 0;
    uint32_t ph = 0;
    bool waited = false;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
      for (int kb = 0; kb < g.kb_total; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + (size_t)s * Cfg::STAGE_BYTES;
        if (elect_one()) {
          mbar_expect_tx(&full[s], Cfg::STAGE_BYTES);
          tma_load_2d(st, &tmW, &full[s], kb * VP_BK, tile * VP_FT);
          if (!waited) pdl_wait();
          tma_load_2d(st + VP_W_BYTES, &tmH, &full[s], kb * VP_BK, 0);
        }
        waited = true;
        __syncwarp();
        if (++s == g.stages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ---- consumers: D[feature][row] += W[64 features of warpgroup wg][64] . H[NT rows][64]^T
  const int wg = warp >> 2;
  const int row = threadIdx.x;  // epilogue: this thread's row of h
  float acc[NT / 2];
  int s = 0, prev = 0;
  uint32_t ph = 0;
  bool synced = false;
  for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < g.kb_total; ++kb) {
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * Cfg::STAGE_BYTES);
      const uint64_t da = make_smem_desc(sa + wg * 64 * 128), db = make_smem_desc(sa + VP_W_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < VP_BK / 16; ++k) Wgmma<NT>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
      wg_commit();
      wg_wait<1>();
      wg_fence_regs(acc);
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == g.stages) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
    if (!synced) {
      pdl_sync();  // logits / statistics writes must not overtake the upstream kernel; dependents may launch now
      synced = true;
    }

    // ---- epilogue: half q = features [64 q, 64 q + 64) of the tile, held by warpgroup q
    const int f0 = tile * VP_FT;
    float st_m = -INFINITY, st_s = 0.f;  // running log-sum-exp statistics of this thread's row over the tile
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int fq = f0 + q * 64;
      // the previous half's TMA stores have read the staging buffer and every thread has finished its statistics
      if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (wg == q) {
        // register j*4 + 2h + e = (feature (warp & 3) * 16 + lane / 4 + 8h, row j*8 + 2*(lane % 4) + e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int fl = (warp & 3) * 16 + (lane >> 2) + 8 * h;  // feature inside the half
          const int f = fq + fl;
          const float b = (g.bias != nullptr && f < g.n) ? g.bias[f] : 0.f;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            // row r = 8j + r0: the swizzle (r & 7 = r0) does not depend on j, so j only adds an immediate 1 KB offset
            const int r0 = (lane & 3) * 2 + e;
            float* p = reinterpret_cast<float*>(staging + (fl >> 5) * Cfg::GROUP_BYTES + r0 * 128 + ((((fl & 31) >> 2) ^ r0) << 4) +
                                                (fl & 3) * 4);
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) p[j * 256] = (acc[j * 4 + 2 * h + e] + b) * g.post_scale;
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (threadIdx.x == 0) {
        for (int c = 0; c < 2; ++c)
          if (fq + 32 * c < g.n) tma_store_2d(&tmO, staging + c * Cfg::GROUP_BYTES, fq + 32 * c, 0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      if (g.tile_stats != nullptr && row < g.m) {
#pragma unroll 1
        for (int c = 0; c < 2; ++c) {
          const int oc = fq + 32 * c;
          if (oc >= g.n) break;
          float v[32];
          const uint8_t* ap = staging + c * Cfg::GROUP_BYTES + row * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 a = *reinterpret_cast<const float4*>(ap + ((j ^ (row & 7)) << 4));
            v[4 * j] = a.x; v[4 * j + 1] = a.y; v[4 * j + 2] = a.z; v[4 * j + 3] = a.w;
          }
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < 32; ++j) if (oc + j < g.n) cm = fmaxf(cm, v[j]);
          if (cm > -INFINITY) {
            const float nm = fmaxf(st_m, cm);
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) if (oc + j < g.n) sum += __expf(v[j] - nm);
            st_s = st_s * __expf(st_m - nm) + sum;
            st_m = nm;
          }
        }
        if (q == 1) g.tile_stats[(long long)tile * g.m + row] = make_float2(st_m, st_s);
      }
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int NT>
int vp_launch(const sb_gemm_t* g, cudaStream_t st) {
  using Cfg = VpCfg<NT>;
  int dev = 0, smem_optin = 0;
  SB_CUDA_OK(cudaGetDevice(&dev));
  SB_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  VpArgs a;
  a.m = g->m;
  a.n = g->n;
  a.kb_total = g->c_in / VP_BK;
  a.tiles = (g->n + VP_FT - 1) / VP_FT;
  const int fixed = 1024 /*align slack*/ + Cfg::STAGING_BYTES + 2 * VP_STAGE_CAP * 8;
  a.stages = (smem_optin - fixed) / Cfg::STAGE_BYTES;
  if (a.stages > VP_STAGE_CAP) a.stages = VP_STAGE_CAP;
  SB_REQUIRE(a.stages >= 2, SB_ENOSUP, "vocabulary projection: not enough shared memory for %d rows", g->m);
  a.bias = g->bias;
  a.post_scale = g->alpha * g->gamma;
  a.tile_stats = (float2*)g->tile_stats;
  const size_t smem = (size_t)a.stages * Cfg::STAGE_BYTES + fixed;
  static size_t configured = 0;
  if (smem > configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(vocab_proj_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  CUtensorMap tmW, tmH, tmO;
  int rc = make_tmap(&tmW, g->w, (uint64_t)g->c_in, (uint64_t)g->n, (uint64_t)g->c_in, VP_FT);
  if (rc) return rc;
  rc = make_tmap(&tmH, g->a, (uint64_t)g->c_in, (uint64_t)g->m, (uint64_t)g->a_ld, NT);
  if (rc) return rc;
  rc = make_tmap(&tmO, g->out, (uint64_t)g->n, (uint64_t)g->m, (uint64_t)g->out_ld, NT, 4);
  if (rc) return rc;
  const int grid = a.tiles < sm_count() ? a.tiles : sm_count();
  SB_CUDA_OK(launch_k(vocab_proj_kernel<NT>, dim3(grid), dim3(VP_THREADS), smem, st, tmW, tmH, tmO, a));
  count_launch();
  return SB_OK;
}

}  // namespace

bool vocab_proj_supported(const sb_gemm_t* g) {
  return g->tile_stats != nullptr && g->m <= 256 && g->taps == 1 && g->a_row0 == 0 && g->c_in % VP_BK == 0 && !g->glu &&
         g->act == SB_ACT_NONE && g->res1 == nullptr && g->res2 == nullptr && g->out2 == nullptr && g->seq_rows == 0 &&
         g->out_row0 == 0 && g->out_f32 && g->prefetch == nullptr && ((uintptr_t)g->out % 16) == 0 && (g->out_ld % 4) == 0;
}

int vocab_proj(const sb_gemm_t* g, cudaStream_t st) {
  const int npad = (g->m + 15) / 16 * 16;
  if (npad <= 32) return vp_launch<32>(g, st);
  if (npad <= 64) return vp_launch<64>(g, st);
  if (npad <= 128) return vp_launch<128>(g, st);
  if (npad <= 160) return vp_launch<160>(g, st);
  return vp_launch<256>(g, st);
}

}  // namespace sb
