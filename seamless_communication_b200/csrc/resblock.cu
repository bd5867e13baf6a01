// Fused HiFi-GAN ResBlock for the narrow stages of the generator (C = 16 / 32 channels), sm_90a.
//
// Reference semantics (models/vocoder/hifigan.py:114-121, one ResBlock with dilations (d0, d1, d2)):
//     for c1, c2 in zip(convs1, convs2):  xt = c2(lrelu(c1(lrelu(x)))) ;  x = xt + x
// and the generator's multi-receptive-field sum xs = sum_j resblock_j(x), x = xs / num_kernels (hifigan.py:186-191).
//
// Why a dedicated kernel: at C = 16 / 32 a conv run as one GEMM launch moves a 160 MB activation in and two out for a
// few hundred MFLOP per MB, and a 128 x C output tile holds an SM far longer than its tensor work takes.
// Here one CTA keeps a time tile of the residual stream in shared memory and runs all six
// convs of the ResBlock on it; HBM sees the tile once in and once out.  Tap j of a dilated conv is the same smem tile
// shifted by (j - k/2) * d rows, which ldmatrix addresses directly, so the convs run on mma.sync.m16n8k16 (fp16 in,
// fp32 accumulate) without any im2col; the wgmma GEMM keeps the wide stages (C >= 64) where GEMM tiles are full.
//
// Rounding points equal the unfused path: every inter-conv activation is rounded to fp16 once (smem), biases and
// residual adds happen in fp32 before that rounding.  The final (x + res2) * gamma is formed from the fp16 x tile.
#include "common.cuh"

namespace sb {
namespace {

constexpr int RB_ROWS = 640;    // time rows per tile: valid outputs plus both halos
constexpr int RB_GUARD = 32;    // guard rows either side of a buffer: the largest tap offset is 5 * 5 = 25 rows
constexpr int RB_WARPS = 10;    // 64 rows = 4 m16 tiles per warp
constexpr int RB_THREADS = RB_WARPS * 32;
constexpr int RB_MT = 4;
constexpr int RB_KMAX = 11;

struct ResblockArgs {
  const elem_t* x;     // (B, Tp, C) sequence layout, data rows at [PH, PH + T)
  const elem_t* res2;  // optional running sum of the previous ResBlocks (same layout)
  elem_t* out;         // (x_final + res2) * gamma
  elem_t* out2;        // optional lrelu(out, out2_slope)
  const elem_t* w1[3];
  const elem_t* w2[3];
  const float* b1[3];
  const float* b2[3];
  int dil[3];
  int k, T, Tp, PH;
  float slope, gamma, out2_slope;
};

template <int C>
struct RbCfg {
  static constexpr int LD = C + 8;  // padded smem row (halves): 48 / 80 B rows make ldmatrix and fragment stores conflict-free
  static constexpr int NT = C / 8;
  static constexpr int KC = C / 16;
  static constexpr int BUF = (RB_ROWS + 2 * RB_GUARD) * LD;  // halves per activation buffer
  static constexpr int W_LD_MAX = RB_KMAX * C + 8;
  static constexpr int SMEM_BYTES = (3 * BUF + C * W_LD_MAX) * 2;
};

__device__ __forceinline__ void rb_ldsm_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void rb_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float rb_lrelu(float v, float s) { return v > 0.f ? v : v * s; }

// weights of one conv, (C, k*C) row-major in global -> rows padded to k*C + 8 halves in smem (conflict-free B fragments)
template <int C>
__device__ __forceinline__ void rb_load_weights(elem_t* ws, const elem_t* __restrict__ w, int k) {
  const int row_vecs = k * C / 8, w_ld = k * C + 8;
  for (int i = threadIdx.x; i < C * row_vecs; i += RB_THREADS) {
    const int r = i / row_vecs, v = i - r * row_vecs;
    *reinterpret_cast<uint4*>(ws + r * w_ld + v * 8) = *reinterpret_cast<const uint4*>(w + (long long)r * k * C + v * 8);
  }
}

// One 'same'-padded conv over the whole tile: out[r][co] = sum_{tap, ci} w[co][tap][ci] * in[r + (tap - k/2) * d][ci].
// SECOND = false: ts = mask(lrelu(conv + b))                       (convs1 followed by the activation of convs2)
// SECOND = true : xs = mask(conv + b + xs) ; as = lrelu(xs)         (convs2, residual add, activation of the next convs1)
template <int C, bool SECOND>
__device__ __forceinline__ void rb_conv(const elem_t* __restrict__ in, elem_t* __restrict__ xs, elem_t* __restrict__ as,
                                        elem_t* __restrict__ ts, const elem_t* __restrict__ ws, const float* __restrict__ bias,
                                        int k, int d, int t_first, int T, float slope) {
  using Cfg = RbCfg<C>;
  constexpr int LD = Cfg::LD, NT = Cfg::NT, KC = Cfg::KC;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hk = (k - 1) >> 1, w_ld = k * C + 8;
  float acc[RB_MT][NT][4];
#pragma unroll
  for (int mt = 0; mt < RB_MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
  // ldmatrix.x4 source rows: lanes 0-7 rows 0-7 / k 0-7, lanes 8-15 rows 8-15 / k 0-7, lanes 16-31 the same for k 8-15
  const elem_t* abase = in + (RB_GUARD + warp * (16 * RB_MT) + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
  const elem_t* wbase = ws + (lane >> 2) * w_ld + (lane & 3) * 2;
  for (int tap = 0; tap < k; ++tap) {
    const int shift = (tap - hk) * d;
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      uint32_t bf[NT][2];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const elem_t* wp = wbase + nt * 8 * w_ld + tap * C + kc * 16;
        bf[nt][0] = *reinterpret_cast<const uint32_t*>(wp);
        bf[nt][1] = *reinterpret_cast<const uint32_t*>(wp + 8);
      }
#pragma unroll
      for (int mt = 0; mt < RB_MT; ++mt) {
        uint32_t a[4];
        rb_ldsm_x4(a, abase + (mt * 16 + shift) * LD + kc * 16);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) rb_mma(acc[mt][nt], a, bf[nt][0], bf[nt][1]);
      }
    }
  }
  // epilogue: accumulator (row = lane/4 (+8), cols = 2*(lane%4) + {0,1}) -> fp16 pairs in smem
#pragma unroll
  for (int mt = 0; mt < RB_MT; ++mt) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int r = warp * (16 * RB_MT) + mt * 16 + (lane >> 2) + half * 8;
      const int t = t_first + r;
      const bool valid = t >= 0 && t < T;  // rows outside the sequence are the conv's zero padding
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int c = nt * 8 + (lane & 3) * 2;
        const int off = (RB_GUARD + r) * LD + c;
        float v0 = acc[mt][nt][2 * half] + __ldg(bias + c), v1 = acc[mt][nt][2 * half + 1] + __ldg(bias + c + 1);
        if (SECOND) {
          const float2 xr = __half22float2(*reinterpret_cast<const __half2*>(xs + off));
          v0 = valid ? v0 + xr.x : 0.f;
          v1 = valid ? v1 + xr.y : 0.f;
          *reinterpret_cast<__half2*>(xs + off) = __floats2half2_rn(v0, v1);
          *reinterpret_cast<__half2*>(as + off) = __floats2half2_rn(rb_lrelu(v0, slope), rb_lrelu(v1, slope));
        } else {
          v0 = valid ? rb_lrelu(v0, slope) : 0.f;
          v1 = valid ? rb_lrelu(v1, slope) : 0.f;
          *reinterpret_cast<__half2*>(ts + off) = __floats2half2_rn(v0, v1);
        }
      }
    }
  }
}

template <int C>
__global__ void __launch_bounds__(RB_THREADS, C == 16 ? 2 : 1) resblock_kernel(const ResblockArgs p) {
  using Cfg = RbCfg<C>;
  constexpr int LD = Cfg::LD, VEC = C / 8;
  extern __shared__ __align__(16) uint8_t rb_smem[];
  elem_t* xs = reinterpret_cast<elem_t*>(rb_smem);  // residual stream x
  elem_t* as = xs + Cfg::BUF;                        // lrelu(x)
  elem_t* ts = as + Cfg::BUF;                        // lrelu(convs1(lrelu(x)))
  elem_t* ws = ts + Cfg::BUF;                        // weights of the conv in flight
  const int hk = (p.k - 1) >> 1;
  const int H = hk * (p.dil[0] + p.dil[1] + p.dil[2] + 3);  // receptive-field half width of the whole ResBlock
  const int TT = RB_ROWS - 2 * H;                            // valid outputs per tile
  const int b = blockIdx.y;
  const int t_first = blockIdx.x * TT - H;                   // time index of tile row 0
  const long long seq0 = ((long long)b * p.Tp + p.PH) * C;   // element offset of (b, t = 0)
  pdl_sync();
  // guard rows (never part of a valid output's receptive field, zeroed so that no NaN pattern is ever multiplied)
  for (int i = threadIdx.x; i < RB_GUARD * LD / 8 * 2; i += RB_THREADS) {
    const int side = i / (RB_GUARD * LD / 8), j = i - side * (RB_GUARD * LD / 8);
    const int off = (side ? (RB_GUARD + RB_ROWS) * LD : 0) + j * 8;
    const uint4 z = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(as + off) = z;
    *reinterpret_cast<uint4*>(ts + off) = z;
  }
  // tile load: x and lrelu(x); rows outside [0, T) are zero
  for (int i = threadIdx.x; i < RB_ROWS * VEC; i += RB_THREADS) {
    const int r = i / VEC, v = i - r * VEC;
    const int t = t_first + r;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (t >= 0 && t < p.T) u = *reinterpret_cast<const uint4*>(p.x + seq0 + (long long)t * C + v * 8);
    uint4 a;
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    __half2* ha = reinterpret_cast<__half2*>(&a);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h[e]);
      ha[e] = __floats2half2_rn(rb_lrelu(f.x, p.slope), rb_lrelu(f.y, p.slope));
    }
    const int off = (RB_GUARD + r) * LD + v * 8;
    *reinterpret_cast<uint4*>(xs + off) = u;
    *reinterpret_cast<uint4*>(as + off) = a;
  }
#pragma unroll 1
  for (int pair = 0; pair < 3; ++pair) {
    rb_load_weights<C>(ws, p.w1[pair], p.k);
    __syncthreads();  // weights + the previous stage's activations are in place
    rb_conv<C, false>(as, xs, as, ts, ws, p.b1[pair], p.k, p.dil[pair], t_first, p.T, p.slope);
    __syncthreads();  // ts complete, ws free
    rb_load_weights<C>(ws, p.w2[pair], p.k);
    __syncthreads();
    rb_conv<C, true>(ts, xs, as, ts, ws, p.b2[pair], p.k, 1, t_first, p.T, p.slope);
    __syncthreads();  // xs / as complete, ws free
  }
  // write the valid rows: out = (x + res2) * gamma, out2 = lrelu(out)
  for (int i = threadIdx.x; i < TT * VEC; i += RB_THREADS) {
    const int rr = i / VEC, v = i - rr * VEC;
    const int r = H + rr, t = t_first + r;
    if (t >= p.T) continue;
    const long long g = seq0 + (long long)t * C + v * 8;
    const uint4 u = *reinterpret_cast<const uint4*>(xs + (RB_GUARD + r) * LD + v * 8);
    uint4 rz = make_uint4(0, 0, 0, 0);
    if (p.res2 != nullptr) rz = *reinterpret_cast<const uint4*>(p.res2 + g);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    const __half2* hr = reinterpret_cast<const __half2*>(&rz);
    uint4 o, o2;
    __half2* ho = reinterpret_cast<__half2*>(&o);
    __half2* ho2 = reinterpret_cast<__half2*>(&o2);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h[e]), fr = __half22float2(hr[e]);
      const float a0 = (f.x + fr.x) * p.gamma, a1 = (f.y + fr.y) * p.gamma;
      ho[e] = __floats2half2_rn(a0, a1);
      ho2[e] = __floats2half2_rn(rb_lrelu(a0, p.out2_slope), rb_lrelu(a1, p.out2_slope));
    }
    *reinterpret_cast<uint4*>(p.out + g) = o;
    if (p.out2 != nullptr) *reinterpret_cast<uint4*>(p.out2 + g) = o2;
  }
  // halo rows of this sequence stay zero (the next conv reads them as padding): first / last tile rewrite them
  const bool first = blockIdx.x == 0, last = blockIdx.x == gridDim.x - 1;
  if (first || last) {
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int i = threadIdx.x; i < p.PH * VEC; i += RB_THREADS) {
      if (first) {
        const long long g = seq0 - (long long)p.PH * C + (long long)i * 8;
        *reinterpret_cast<uint4*>(p.out + g) = z;
        if (p.out2 != nullptr) *reinterpret_cast<uint4*>(p.out2 + g) = z;
      }
      if (last) {
        const long long g = seq0 + (long long)p.T * C + (long long)i * 8;
        *reinterpret_cast<uint4*>(p.out + g) = z;
        if (p.out2 != nullptr) *reinterpret_cast<uint4*>(p.out2 + g) = z;
      }
    }
  }
}

template <int C>
int launch_resblock(const ResblockArgs& a, int batch, cudaStream_t st) {
  using Cfg = RbCfg<C>;
  static bool configured = false;
  if (!configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(resblock_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int hk = (a.k - 1) / 2;
  const int H = hk * (a.dil[0] + a.dil[1] + a.dil[2] + 3);
  const int TT = RB_ROWS - 2 * H;
  dim3 grid((a.T + TT - 1) / TT, batch);
  SB_CUDA_OK(launch_k(resblock_kernel<C>, grid, dim3(RB_THREADS), (size_t)Cfg::SMEM_BYTES, st, a));
  count_launch();
  return SB_OK;
}

}  // namespace
}  // namespace sb

extern "C" int sb_hifigan_resblock(const sb_resblock_t* r, sb_stream_t stream) {
  SB_REQUIRE(r != nullptr && r->x != nullptr && r->out != nullptr, SB_EINVAL, "sb_hifigan_resblock: null argument");
  SB_REQUIRE(r->channels == 16 || r->channels == 32, SB_EINVAL, "sb_hifigan_resblock: channels must be 16 or 32 (got %d)",
             r->channels);
  SB_REQUIRE(r->kernel_size >= 1 && r->kernel_size <= sb::RB_KMAX && (r->kernel_size & 1), SB_EINVAL,
             "sb_hifigan_resblock: kernel size must be odd and <= %d (got %d)", sb::RB_KMAX, r->kernel_size);
  SB_REQUIRE(r->batch > 0 && r->T > 0 && r->halo >= 0 && r->rows_per_seq >= r->T + 2 * r->halo, SB_EINVAL,
             "sb_hifigan_resblock: bad geometry (batch %d, T %d, halo %d, rows %d)", r->batch, r->T, r->halo, r->rows_per_seq);
  sb::ResblockArgs a;
  const int hk = (r->kernel_size - 1) / 2;
  for (int i = 0; i < 3; ++i) {
    SB_REQUIRE(r->w1[i] && r->w2[i] && r->b1[i] && r->b2[i], SB_EINVAL, "sb_hifigan_resblock: null weights of pair %d", i);
    SB_REQUIRE(r->dilation[i] >= 1 && hk * r->dilation[i] <= sb::RB_GUARD, SB_EINVAL,
               "sb_hifigan_resblock: tap offset %d exceeds the %d guard rows", hk * r->dilation[i], sb::RB_GUARD);
    a.w1[i] = (const sb::elem_t*)r->w1[i]; a.w2[i] = (const sb::elem_t*)r->w2[i];
    a.b1[i] = r->b1[i]; a.b2[i] = r->b2[i];
    a.dil[i] = r->dilation[i];
  }
  a.x = (const sb::elem_t*)r->x; a.res2 = (const sb::elem_t*)r->res2;
  a.out = (sb::elem_t*)r->out; a.out2 = (sb::elem_t*)r->out2;
  a.k = r->kernel_size; a.T = r->T; a.Tp = r->rows_per_seq; a.PH = r->halo;
  a.slope = r->slope; a.gamma = r->gamma; a.out2_slope = r->out2_slope;
  cudaStream_t st = (cudaStream_t)stream;
  return r->channels == 16 ? sb::launch_resblock<16>(a, r->batch, st) : sb::launch_resblock<32>(a, r->batch, st);
}
