// Skinny GEMM for the incremental decoder step: out (rows <= 160) x N = A (rows x K) . W^T (N x K), sm_90a.
//
// At 160 rows (32 sentences x beam 5, SURVEY 8a a8) a decoder-layer GEMM streams 2-16 MB of weights for 0.3-2.7 GFLOP:
// every CTA sees a few dozen KB and the kernel is a single latency chain.  The TMA / tensor-core GEMM pays a fixed latency per launch for
// that chain (tensor-map fetch, mbarrier setup, TMA round trip, MMA group wait, accumulator staging, staged TMA store).  This kernel does the same product with the shortest chain that still uses tensor cores:
// cp.async straight into padded shared memory (all loads of a CTA in flight at once), ldmatrix + mma.sync.m16n8k16
// (fp16 in, fp32 accumulate), results stored from registers.  One warp owns one 16-row m-tile and all 64 columns of the
// CTA's n-tile, so A fragments are read once and the 64-column W tile is shared through smem.
//
// Two output modes, selected by the caller:
//   split-K : CTA (n-tile, z) covers K range z and stores raw fp32 partial products to rows [z*slice_rows, ..+rows) of
//             `partials` (row stride N) - same contract as sb_gemm_splitk, consumed by sb_splitk_reduce_ln / attention;
//   direct  : one CTA per n-tile over the whole K, epilogue bias + activation -> fp16 (the FFN inner projection).
#include "common.cuh"

namespace sb {
namespace {

constexpr int SK_BN = 64;        // output columns per CTA
constexpr int SK_KCH = 64;       // K elements per pipeline stage
constexpr int SK_LD = SK_KCH + 8;  // padded smem row (halves): 144 B rows -> conflict-free ldmatrix
constexpr int SK_MAXROWS = 160;  // 10 m16 tiles, one per warp
constexpr int SK_WARPS = SK_MAXROWS / 16;
constexpr int SK_THREADS = SK_WARPS * 32;
constexpr int SK_STAGES = 3;
constexpr int SK_STAGE_HALVES = (SK_MAXROWS + SK_BN) * SK_LD;
constexpr int SK_SMEM_BYTES = SK_STAGES * SK_STAGE_HALVES * 2;  // 96 768 B: two CTAs per SM

struct SkinnyArgs {
  const elem_t* a;
  long long a_ld;
  const elem_t* w;  // (N, K) row-major
  int rows, n, k;
  int k_per_split;       // K range of one blockIdx.y slice (multiple of SK_KCH)
  float* partials;       // split-K mode (else nullptr)
  long long slice_rows;
  const float* bias;     // direct mode
  int act;
  elem_t* out;
  long long out_ld;
  const char* prefetch;  // weights of the kernel that follows, pulled into L2 (see gemm_tcgen05.cu)
  long long prefetch_bytes;
};

__device__ __forceinline__ void sk_cp16(void* smem_dst, const void* gsrc, bool pred) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int bytes = pred ? 16 : 0;  // src-size 0: the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sk_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void sk_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void sk_ldsm_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void sk_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(SK_THREADS, 2) skinny_gemm_kernel(const SkinnyArgs p) {
  extern __shared__ __align__(16) uint8_t sk_smem[];
  elem_t* smem = reinterpret_cast<elem_t*>(sk_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * SK_BN;
  const int k_begin = blockIdx.y * p.k_per_split;
  const int chunks = p.k_per_split / SK_KCH;

  // stage loader: A rows [0, 160) (rows >= p.rows zero-filled) then the W rows of this n-tile, 8 x 16 B per row
  auto load_stage = [&](int chunk, int stage) {
    elem_t* sa = smem + stage * SK_STAGE_HALVES;
    const int k0 = k_begin + chunk * SK_KCH;
    for (int i = threadIdx.x; i < (SK_MAXROWS + SK_BN) * (SK_KCH / 8); i += SK_THREADS) {
      const int r = i >> 3, v = i & 7;
      if (r < SK_MAXROWS) {
        const bool ok = r < p.rows;
        sk_cp16(sa + r * SK_LD + v * 8, p.a + (long long)(ok ? r : 0) * p.a_ld + k0 + v * 8, ok);
      } else {
        sk_cp16(sa + r * SK_LD + v * 8, p.w + (long long)(n0 + r - SK_MAXROWS) * p.k + k0 + v * 8, true);
      }
    }
  };
  // a stage mixes weights with activations of the upstream kernel, so the wait precedes the first copy
  pdl_sync();
#pragma unroll
  for (int s = 0; s < SK_STAGES - 1; ++s) {
    if (s < chunks) load_stage(s, s);
    sk_commit();
  }
  if (warp == 0 && p.prefetch_bytes > 0) {
    const long long ncta = (long long)gridDim.x * gridDim.y, cta = blockIdx.x + (long long)gridDim.x * blockIdx.y;
    const long long share = ((p.prefetch_bytes + ncta - 1) / ncta + 4095) / 4096 * 4096;
    const long long lo = cta * share, hi = min(lo + share, p.prefetch_bytes);
    if (lane == 0)
      for (long long o = lo; o < hi; o += 16384)
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.prefetch + o), "r"((uint32_t)min(16384ll, hi - o)) : "memory");
    __syncwarp();
  }

  float acc[SK_BN / 8][4];
#pragma unroll
  for (int nt = 0; nt < SK_BN / 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
  const bool warp_active = warp * 16 < p.rows;  // m-tiles past the last row hold zeros: skip their math
  // ldmatrix source addresses (see resblock.cu): A rows of this warp's m-tile; W rows as the col-major B operand
  const int a_off = (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * SK_LD + (lane >> 4) * 8;
  const int b_off = (SK_MAXROWS + ((lane >> 4) & 1) * 8 + (lane & 7)) * SK_LD + ((lane >> 3) & 1) * 8;

  for (int c = 0; c < chunks; ++c) {
    sk_wait<SK_STAGES - 2>();  // chunk c has landed (for this thread's copies) ...
    __syncthreads();           // ... and for everyone's; the stage consumed in iteration c-1 is free
    if (c + SK_STAGES - 1 < chunks) load_stage(c + SK_STAGES - 1, (c + SK_STAGES - 1) % SK_STAGES);
    sk_commit();
    if (warp_active) {
      const elem_t* st = smem + (c % SK_STAGES) * SK_STAGE_HALVES;
#pragma unroll
      for (int ks = 0; ks < SK_KCH / 16; ++ks) {
        uint32_t a[4];
        sk_ldsm_x4(a, st + a_off + ks * 16);
#pragma unroll
        for (int np = 0; np < SK_BN / 16; ++np) {  // two n8 tiles per ldmatrix.x4: {n0-7 k0-7, n0-7 k8-15, n8-15 k0-7, n8-15 k8-15}
          uint32_t b[4];
          sk_ldsm_x4(b, st + b_off + np * 16 * SK_LD + ks * 16);
          sk_mma(acc[2 * np], a, b[0], b[1]);
          sk_mma(acc[2 * np + 1], a, b[2], b[3]);
        }
      }
    }
  }
  sk_wait<0>();
  if (!warp_active) return;
  // epilogue from registers: row = lane/4 (+8), columns 2*(lane%4) + {0,1} of each n8 tile
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int r = warp * 16 + (lane >> 2) + half * 8;
    if (r >= p.rows) continue;
    if (p.partials != nullptr) {
      float* o = p.partials + ((long long)blockIdx.y * p.slice_rows + r) * p.n + n0 + (lane & 3) * 2;
#pragma unroll
      for (int nt = 0; nt < SK_BN / 8; ++nt) *reinterpret_cast<float2*>(o + nt * 8) = make_float2(acc[nt][2 * half], acc[nt][2 * half + 1]);
    } else {
      elem_t* o = p.out + (long long)r * p.out_ld + n0 + (lane & 3) * 2;
#pragma unroll
      for (int nt = 0; nt < SK_BN / 8; ++nt) {
        const int c = n0 + nt * 8 + (lane & 3) * 2;
        float v0 = acc[nt][2 * half], v1 = acc[nt][2 * half + 1];
        if (p.bias != nullptr) { v0 += __ldg(p.bias + c); v1 += __ldg(p.bias + c + 1); }
        if (p.act == SB_ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        *reinterpret_cast<__half2*>(o + nt * 8) = __floats2half2_rn(v0, v1);
      }
    }
  }
}

}  // namespace
}  // namespace sb

extern "C" int sb_gemm_skinny_supported(const sb_gemm_t* g, int32_t splits) {
  if (g == nullptr || splits < 1) return 0;
  if (g->taps != 1 || g->glu || g->m < 1 || g->m > sb::SK_MAXROWS) return 0;
  if (g->n % sb::SK_BN != 0 || g->c_in % (splits * sb::SK_KCH) != 0) return 0;
  if (g->a_ld % 8 != 0 || ((uintptr_t)g->a % 16) != 0 || ((uintptr_t)g->w % 16) != 0 || g->a_row0 != 0) return 0;
  return 1;
}

extern "C" int sb_gemm_skinny(const sb_gemm_t* g, int32_t splits, float* partials, int64_t slice_rows, sb_stream_t stream) {
  SB_REQUIRE(g != nullptr && g->a != nullptr && g->w != nullptr, SB_EINVAL, "sb_gemm_skinny: null argument");
  SB_REQUIRE(sb_gemm_skinny_supported(g, splits), SB_EINVAL,
             "sb_gemm_skinny: unsupported problem (rows %d <= %d, n %d %% 64, k %d %% (64 * %d splits), taps %d)", g->m,
             sb::SK_MAXROWS, g->n, g->c_in, splits, g->taps);
  sb::SkinnyArgs a;
  a.a = (const sb::elem_t*)g->a; a.a_ld = g->a_ld; a.w = (const sb::elem_t*)g->w;
  a.rows = g->m; a.n = g->n; a.k = g->c_in; a.k_per_split = g->c_in / splits;
  a.prefetch = (const char*)g->prefetch; a.prefetch_bytes = g->prefetch ? g->prefetch_bytes / 4096 * 4096 : 0;
  if (partials != nullptr) {
    SB_REQUIRE(slice_rows >= g->m, SB_EINVAL, "sb_gemm_skinny: slice_rows (%lld) < rows (%d)", (long long)slice_rows, g->m);
    a.partials = partials; a.slice_rows = slice_rows; a.bias = nullptr; a.act = SB_ACT_NONE; a.out = nullptr; a.out_ld = 0;
  } else {
    SB_REQUIRE(splits == 1 && g->out != nullptr && !g->out_f32 && g->res1 == nullptr && g->res2 == nullptr &&
                   g->out2 == nullptr && g->seq_rows == 0 && g->out_row0 == 0 && g->alpha == 1.f && g->gamma == 1.f &&
                   (g->act == SB_ACT_NONE || g->act == SB_ACT_RELU) && g->out_ld % 2 == 0,
               SB_EINVAL, "sb_gemm_skinny: direct mode supports bias + none/relu -> fp16 only");
    a.partials = nullptr; a.slice_rows = 0; a.bias = g->bias; a.act = g->act; a.out = (sb::elem_t*)g->out; a.out_ld = g->out_ld;
  }
  static bool configured = false;
  if (!configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(sb::skinny_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sb::SK_SMEM_BYTES));
    configured = true;
  }
  dim3 grid(g->n / sb::SK_BN, splits);
  SB_CUDA_OK(sb::launch_k(sb::skinny_gemm_kernel, grid, dim3(sb::SK_THREADS), (size_t)sb::SK_SMEM_BYTES, (cudaStream_t)stream, a));
  sb::count_launch();
  return SB_OK;
}
