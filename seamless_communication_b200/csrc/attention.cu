// sb_attention: flash-style multi-head attention, head_dim 64, fp16 in/out, fp32 softmax & accumulation.
//
// One CTA = 64 query rows of one (batch, head); 4 warps x 16 rows; key/value blocks of 64 staged in shared memory.
// Tensor-core math uses mma.sync.m16n8k16 (attention is ~4 % of the encoder FLOPs; the GEMMs around it are wgmma).
// Shaw relative-position bias (models/conformer_shaw/builder.py:127-146): instead of the reference's (S,S,64) gather
// + einsum, each warp computes QR = q . rel_k^T once (16 x 73, a tiny GEMM) and the score tile adds
// QR[i, clamp(j-i,-L,R)+L] by a shared-memory lookup.
// Transformer-XL relative attention of w2v-BERT v1 (RelativePositionSDPA; mirrored ggml/examples/unity/fairseq2.cpp:605-696):
// scores[i][j] = ((q_i + u).k_j + (q_i + v).R[S-1+j-i]) / 8, R = r_proj(pos table) of shape (2S-1, H*64).  The (S, 2S-1)
// positional scores are never materialised: for each 64 x 64 (query, key) tile the 127 R rows it touches are staged in shared
// memory (a 128-row window), each warp multiplies its 16 rows of q + v against the 80 rows its queries reach (16 x 80, five
// m16n8k16 column pairs) and the score tile adds them by diagonal lookup: row il, key jl reads column jl - il + 15.
#include "common.cuh"

#include <type_traits>

namespace sb {

constexpr int HD = 64;          // head dim
constexpr int AQ = 64, AK = 64; // query / key block
constexpr int LDS = HD + 8;     // padded smem row (halves): conflict-free ldmatrix
constexpr int REL_MAX = 80;     // rel table rows padded to a multiple of 16
constexpr int XL_ROWS = 128;    // R window per (query tile, key tile): rows S-1+k0-q0-63 .. +127 (the last one unused)
constexpr int XL_MAX_S = 4096;  // fairseq2's relative position table covers distances up to n_ctx - 1 = 4095

__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

struct AttnArgs {
  const elem_t *q, *k, *v;
  elem_t* out;
  long long q_ld, k_ld, v_ld, out_ld;
  int batch, heads, sq, sk, q_rows, q_halo, kv_rows, kv_halo;
  const int* kv_lens;
  int causal;
  const elem_t* rel_k;
  int rel_left, rel_right;
};
// Transformer-XL mode: R fp16 [2*sq-1][r_ld] (head h at columns h*64..), u / v fp32 [heads][64] (NULL = 0)
struct XlAttnArgs : AttnArgs {
  const elem_t* r;
  long long r_ld;
  const float *bias_u, *bias_v;
};

// XL = false: plain or Shaw attention (sb_attention); XL = true: Transformer-XL relative attention (sb_attention_relpos)
template <bool XL>
__global__ void __launch_bounds__(128) attention_kernel(const std::conditional_t<XL, XlAttnArgs, AttnArgs> p) {
  extern __shared__ __align__(16) uint8_t smem_attn[];
  elem_t* sQ = reinterpret_cast<elem_t*>(smem_attn);  // [AQ][LDS]   (XL: q + u)
  elem_t* sK = sQ + AQ * LDS;                         // [AK][LDS]
  elem_t* sV = sK + AK * LDS;                         // [AK][LDS]
  elem_t* sR = sV + AK * LDS;                         // [REL_MAX][LDS]   (Shaw) / [XL_ROWS][LDS] (XL: R window)
  float* sQR = reinterpret_cast<float*>(sR + (XL ? XL_ROWS : REL_MAX) * LDS);  // [4 warps][16][REL_MAX+1]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  const int q0 = blockIdx.x * AQ;
  const int h = blockIdx.y, b = blockIdx.z;
  const int kv_len = p.kv_lens ? min(p.kv_lens[b], p.sk) : p.sk;
  const bool shaw = !XL && p.rel_k != nullptr;
  const int nrel = p.rel_left + p.rel_right + 1;

  // ---- stage Q tile (and the rel table) ----
  if constexpr (XL) {
    // sQ = q + u, sQv = q + v: summed in fp32, rounded once to fp16 (with u == NULL, sQ is q bit for bit)
    elem_t* sQv = reinterpret_cast<elem_t*>(sQR + 4 * 16 * (REL_MAX + 1));  // [AQ][LDS]
    for (int i = threadIdx.x; i < AQ * (HD / 8); i += blockDim.x) {
      int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
      uint4 qu = make_uint4(0, 0, 0, 0), qv = make_uint4(0, 0, 0, 0);
      if (q0 + r < p.sq) {
        const uint4 raw = *reinterpret_cast<const uint4*>(p.q + ((long long)b * p.q_rows + p.q_halo + q0 + r) * p.q_ld + h * HD + c);
        const __half2* hq = reinterpret_cast<const __half2*>(&raw);
        __half2* hu = reinterpret_cast<__half2*>(&qu);
        __half2* hv = reinterpret_cast<__half2*>(&qv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(hq[e]);
          const int o = h * HD + c + 2 * e;
          hu[e] = p.bias_u ? __floats2half2_rn(f.x + p.bias_u[o], f.y + p.bias_u[o + 1]) : hq[e];
          hv[e] = p.bias_v ? __floats2half2_rn(f.x + p.bias_v[o], f.y + p.bias_v[o + 1]) : hq[e];
        }
      }
      *reinterpret_cast<uint4*>(sQ + r * LDS + c) = qu;
      *reinterpret_cast<uint4*>(sQv + r * LDS + c) = qv;
    }
  } else {
    for (int i = threadIdx.x; i < AQ * (HD / 8); i += blockDim.x) {
      int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (q0 + r < p.sq) u = *reinterpret_cast<const uint4*>(p.q + ((long long)b * p.q_rows + p.q_halo + q0 + r) * p.q_ld + h * HD + c);
      *reinterpret_cast<uint4*>(sQ + r * LDS + c) = u;
    }
  }
  if (shaw) {
    for (int i = threadIdx.x; i < REL_MAX * (HD / 8); i += blockDim.x) {
      int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (r < nrel) u = *reinterpret_cast<const uint4*>(p.rel_k + r * HD + c);
      *reinterpret_cast<uint4*>(sR + r * LDS + c) = u;
    }
  }
  __syncthreads();

  // Q fragments: 16 rows x 64 dims per warp = 4 k-steps
  uint32_t qa[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const elem_t* ptr = sQ + (warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LDS + ks * 16 + 8 * (lane >> 4);
    ldsm_x4(qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], ptr);
  }
  uint32_t qva[XL ? 4 : 1][4];  // XL: (q + v) fragments
  if constexpr (XL) {
    const elem_t* sQv = reinterpret_cast<const elem_t*>(sQR + 4 * 16 * (REL_MAX + 1));
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const elem_t* ptr = sQv + (warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LDS + ks * 16 + 8 * (lane >> 4);
      ldsm_x4(qva[ks][0], qva[ks][1], qva[ks][2], qva[ks][3], ptr);
    }
  }
  float* qr = sQR + warp * 16 * (REL_MAX + 1);
  if (shaw) {
    // QR[16][nrel] = Q_warp . rel^T
#pragma unroll
    for (int nt2 = 0; nt2 < REL_MAX / 16; ++nt2) {
      float c0[4] = {0, 0, 0, 0}, c1[4] = {0, 0, 0, 0};
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sR + (nt2 * 16 + (lane & 7) + 8 * (lane >> 4)) * LDS + ks * 16 + 8 * ((lane >> 3) & 1);
        ldsm_x4(b0, b1, b2, b3, ptr);
        mma16816(c0, qa[ks], b0, b1);
        mma16816(c1, qa[ks], b2, b3);
      }
      const int col = nt2 * 16 + 2 * tq;
      qr[g * (REL_MAX + 1) + col] = c0[0];
      qr[g * (REL_MAX + 1) + col + 1] = c0[1];
      qr[(g + 8) * (REL_MAX + 1) + col] = c0[2];
      qr[(g + 8) * (REL_MAX + 1) + col + 1] = c0[3];
      qr[g * (REL_MAX + 1) + col + 8] = c1[0];
      qr[g * (REL_MAX + 1) + col + 9] = c1[1];
      qr[(g + 8) * (REL_MAX + 1) + col + 8] = c1[2];
      qr[(g + 8) * (REL_MAX + 1) + col + 9] = c1[3];
    }
    __syncwarp();
  }

  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const int irow[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};
  const int causal_off = p.sk - p.sq;
  int k_end = kv_len;
  if (p.causal) k_end = min(k_end, q0 + AQ + causal_off);  // keys beyond the last query row of this CTA are masked

  for (int k0 = 0; k0 < k_end; k0 += AK) {
    __syncthreads();
    for (int i = threadIdx.x; i < AK * (HD / 8); i += blockDim.x) {
      int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
      uint4 uk = make_uint4(0, 0, 0, 0), uv = make_uint4(0, 0, 0, 0);
      if (k0 + r < kv_len) {
        long long row = (long long)b * p.kv_rows + p.kv_halo + k0 + r;
        uk = *reinterpret_cast<const uint4*>(p.k + row * p.k_ld + h * HD + c);
        uv = *reinterpret_cast<const uint4*>(p.v + row * p.v_ld + h * HD + c);
      }
      *reinterpret_cast<uint4*>(sK + r * LDS + c) = uk;
      *reinterpret_cast<uint4*>(sV + r * LDS + c) = uv;
    }
    if constexpr (XL) {
      // R rows S-1+j-i for j in [k0, k0+64), i in [q0, q0+64): window base S-1+k0-q0-63; rows outside [0, 2S-1) read as 0
      const int rbase = p.sq - 1 + k0 - q0 - (AQ - 1);
      for (int i = threadIdx.x; i < XL_ROWS * (HD / 8); i += blockDim.x) {
        int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
        const int row = rbase + r;
        uint4 u = make_uint4(0, 0, 0, 0);
        if (row >= 0 && row < 2 * p.sq - 1) u = *reinterpret_cast<const uint4*>(p.r + (long long)row * p.r_ld + h * HD + c);
        *reinterpret_cast<uint4*>(sR + r * LDS + c) = u;
      }
    }
    __syncthreads();
    if constexpr (XL) {
      // QR[il][n] = (q + v)_{q0+16w+il} . R[rbase + 48 - 16w + n], n < 80: column jl - il + 15 holds key k0 + jl
      const elem_t* sRw = sR + (AQ - 16 - 16 * warp) * LDS;
#pragma unroll
      for (int nt2 = 0; nt2 < REL_MAX / 16; ++nt2) {
        float c0[4] = {0, 0, 0, 0}, c1[4] = {0, 0, 0, 0};
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          uint32_t b0, b1, b2, b3;
          const elem_t* ptr = sRw + (nt2 * 16 + (lane & 7) + 8 * (lane >> 4)) * LDS + ks * 16 + 8 * ((lane >> 3) & 1);
          ldsm_x4(b0, b1, b2, b3, ptr);
          mma16816(c0, qva[ks], b0, b1);
          mma16816(c1, qva[ks], b2, b3);
        }
        const int col = nt2 * 16 + 2 * tq;
        qr[g * (REL_MAX + 1) + col] = c0[0];
        qr[g * (REL_MAX + 1) + col + 1] = c0[1];
        qr[(g + 8) * (REL_MAX + 1) + col] = c0[2];
        qr[(g + 8) * (REL_MAX + 1) + col + 1] = c0[3];
        qr[g * (REL_MAX + 1) + col + 8] = c1[0];
        qr[g * (REL_MAX + 1) + col + 9] = c1[1];
        qr[(g + 8) * (REL_MAX + 1) + col + 8] = c1[2];
        qr[(g + 8) * (REL_MAX + 1) + col + 9] = c1[3];
      }
      __syncwarp();
    }

    // S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int nt2 = 0; nt2 < 4; ++nt2) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sK + (nt2 * 16 + (lane & 7) + 8 * (lane >> 4)) * LDS + ks * 16 + 8 * ((lane >> 3) & 1);
        ldsm_x4(b0, b1, b2, b3, ptr);
        mma16816(s[2 * nt2], qa[ks], b0, b1);
        mma16816(s[2 * nt2 + 1], qa[ks], b2, b3);
      }
    }
    // bias, scale, masks, running max
    float mnew[2] = {mrow[0], mrow[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rr = e >> 1;
        const int i = irow[rr];
        const int j = k0 + nt * 8 + 2 * tq + (e & 1);
        float val = s[nt][e];
        if constexpr (XL) {
          val += qr[(g + 8 * rr) * (REL_MAX + 1) + nt * 8 + 2 * tq + (e & 1) - (g + 8 * rr) + 15];
        } else if (shaw) {
          int d = j - i;
          d = d < -p.rel_left ? -p.rel_left : (d > p.rel_right ? p.rel_right : d);
          val += qr[(g + 8 * rr) * (REL_MAX + 1) + d + p.rel_left];
        }
        val *= 0.125f;
        if (j >= kv_len || (p.causal && j > i + causal_off)) val = -INFINITY;
        s[nt][e] = val;
        mnew[rr] = fmaxf(mnew[rr], val);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 1));
      mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 2));
    }
    float corr[2], msafe[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      msafe[rr] = (mnew[rr] == -INFINITY) ? 0.f : mnew[rr];
      corr[rr] = (mrow[rr] == -INFINITY) ? 0.f : __expf(mrow[rr] - msafe[rr]);
      mrow[rr] = mnew[rr];
      lrow[rr] *= corr[rr];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      o[nt][0] *= corr[0]; o[nt][1] *= corr[0]; o[nt][2] *= corr[1]; o[nt][3] *= corr[1];
    }
    // P = exp(S - m), row sums, P V
    uint32_t pa[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      float p0 = __expf(s[nt][0] - msafe[0]), p1 = __expf(s[nt][1] - msafe[0]);
      float p2 = __expf(s[nt][2] - msafe[1]), p3 = __expf(s[nt][3] - msafe[1]);
      lrow[0] += p0 + p1;
      lrow[1] += p2 + p3;
      const int ks = nt >> 1;
      if ((nt & 1) == 0) { pa[ks][0] = pack_h2(p0, p1); pa[ks][1] = pack_h2(p2, p3); }
      else               { pa[ks][2] = pack_h2(p0, p1); pa[ks][3] = pack_h2(p2, p3); }
    }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {      // 16 keys per k-step
#pragma unroll
      for (int nt2 = 0; nt2 < 4; ++nt2) { // 16 output dims per ldmatrix
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sV + (ks * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LDS + nt2 * 16 + 8 * (lane >> 4);
        ldsm_x4_t(b0, b1, b2, b3, ptr);
        mma16816(o[2 * nt2], pa[ks], b0, b1);
        mma16816(o[2 * nt2 + 1], pa[ks], b2, b3);
      }
    }
  }
  // finalize
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    lrow[rr] += __shfl_xor_sync(0xffffffffu, lrow[rr], 1);
    lrow[rr] += __shfl_xor_sync(0xffffffffu, lrow[rr], 2);
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int i = irow[rr];
    if (i >= p.sq) continue;
    const float inv = lrow[rr] > 0.f ? 1.f / lrow[rr] : 0.f;
    elem_t* op = p.out + ((long long)b * p.q_rows + p.q_halo + i) * p.out_ld + h * HD;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      __half2 hv = __floats2half2_rn(o[nt][2 * rr] * inv, o[nt][2 * rr + 1] * inv);
      *reinterpret_cast<__half2*>(op + nt * 8 + 2 * tq) = hv;
    }
  }
}


// ---- v2: 128 query rows per CTA (4 warps x 32 rows: every K / V fragment read from shared memory feeds two m-tiles, which
// halves the ldmatrix traffic per MMA - at 16 rows per warp shared-memory bandwidth and mma.sync throughput cost the same),
// K/V blocks double-buffered with cp.async (the next block streams in while this one is multiplied), and the Shaw bias
// looked up per element only in key blocks that touch the clamping window [i - L, i + R]: everywhere else the bias of a row is
// one of two constants (QR[i][0] left of the window, QR[i][L + R] right of it).
constexpr int AQ2 = 128;

__device__ __forceinline__ void at_cp16(void* smem_dst, const void* gsrc, bool pred) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int bytes = pred ? 16 : 0;  // src-size 0: zero-fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(128, 2) attention2_kernel(const AttnArgs p) {
  extern __shared__ __align__(16) uint8_t smem_attn[];
  elem_t* sQ = reinterpret_cast<elem_t*>(smem_attn);  // [AQ2][LDS]
  elem_t* sKV = sQ + AQ2 * LDS;                       // [2 stages][K: AK x LDS | V: AK x LDS]
  elem_t* sR = sKV + 4 * AK * LDS;                    // [REL_MAX][LDS]   (Shaw only)
  float* sQR = reinterpret_cast<float*>(sR + REL_MAX * LDS);  // [4 warps][32][REL_MAX+1]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  const int q0 = blockIdx.x * AQ2;
  const int h = blockIdx.y, b = blockIdx.z;
  const int kv_len = p.kv_lens ? min(p.kv_lens[b], p.sk) : p.sk;
  const bool shaw = p.rel_k != nullptr;
  const int nrel = p.rel_left + p.rel_right + 1;
  const int causal_off = p.sk - p.sq;
  int k_end = kv_len;
  if (p.causal) k_end = min(k_end, q0 + AQ2 + causal_off);
  const int ntiles = (k_end + AK - 1) / AK;

  auto load_tile = [&](int t, int stage) {
    elem_t* dK = sKV + stage * 2 * AK * LDS;
    elem_t* dV = dK + AK * LDS;
    const int k0 = t * AK;
    for (int i = threadIdx.x; i < AK * (HD / 8); i += 128) {
      const int r = i >> 3, c = (i & 7) * 8;
      const bool ok = k0 + r < kv_len;
      const long long row = (long long)b * p.kv_rows + p.kv_halo + (ok ? k0 + r : 0);
      at_cp16(dK + r * LDS + c, p.k + row * p.k_ld + h * HD + c, ok);
      at_cp16(dV + r * LDS + c, p.v + row * p.v_ld + h * HD + c, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (ntiles > 0) load_tile(0, 0);

  // ---- stage the Q tile (and the rel table) ----
  for (int i = threadIdx.x; i < AQ2 * (HD / 8); i += 128) {
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (q0 + r < p.sq) u = *reinterpret_cast<const uint4*>(p.q + ((long long)b * p.q_rows + p.q_halo + q0 + r) * p.q_ld + h * HD + c);
    *reinterpret_cast<uint4*>(sQ + r * LDS + c) = u;
  }
  if (shaw) {
    for (int i = threadIdx.x; i < REL_MAX * (HD / 8); i += 128) {
      const int r = i >> 3, c = (i & 7) * 8;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (r < nrel) u = *reinterpret_cast<const uint4*>(p.rel_k + r * HD + c);
      *reinterpret_cast<uint4*>(sR + r * LDS + c) = u;
    }
  }
  __syncthreads();

  // Q fragments: 2 m-tiles x 4 k-steps per warp
  uint32_t qa[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const elem_t* ptr = sQ + (warp * 32 + mt * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LDS + ks * 16 + 8 * (lane >> 4);
      ldsm_x4(qa[mt][ks][0], qa[mt][ks][1], qa[mt][ks][2], qa[mt][ks][3], ptr);
    }
  float* qr = sQR + warp * 32 * (REL_MAX + 1);
  if (shaw) {
#pragma unroll
    for (int nt2 = 0; nt2 < REL_MAX / 16; ++nt2) {
      float c[2][2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) c[mt][0][e] = c[mt][1][e] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sR + (nt2 * 16 + (lane & 7) + 8 * (lane >> 4)) * LDS + ks * 16 + 8 * ((lane >> 3) & 1);
        ldsm_x4(b0, b1, b2, b3, ptr);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(c[mt][0], qa[mt][ks], b0, b1);
          mma16816(c[mt][1], qa[mt][ks], b2, b3);
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int col = nt2 * 16 + hf * 8 + 2 * tq;
          float* r0 = qr + (mt * 16 + g) * (REL_MAX + 1) + col;
          float* r1 = qr + (mt * 16 + g + 8) * (REL_MAX + 1) + col;
          r0[0] = c[mt][hf][0]; r0[1] = c[mt][hf][1];
          r1[0] = c[mt][hf][2]; r1[1] = c[mt][hf][3];
        }
    }
    __syncwarp();
  }

  float o[2][8][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int i = 0; i < 8; ++i) o[mt][i][0] = o[mt][i][1] = o[mt][i][2] = o[mt][i][3] = 0.f;
  float mrow[2][2], lrow[2][2];
  int irow[2][2];
  float bias_l[2][2], bias_r[2][2];  // the two constant biases of each row (outside the clamping window)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mrow[mt][rr] = -INFINITY;
      lrow[mt][rr] = 0.f;
      irow[mt][rr] = q0 + warp * 32 + mt * 16 + g + 8 * rr;
      bias_l[mt][rr] = shaw ? qr[(mt * 16 + g + 8 * rr) * (REL_MAX + 1)] : 0.f;
      bias_r[mt][rr] = shaw ? qr[(mt * 16 + g + 8 * rr) * (REL_MAX + 1) + nrel - 1] : 0.f;
    }
  const int i_lo = q0 + warp * 32, i_hi = i_lo + 31;  // query rows of this warp

  for (int t = 0; t < ntiles; ++t) {
    if (t + 1 < ntiles) {
      load_tile(t + 1, (t + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const elem_t* sK = sKV + (t & 1) * 2 * AK * LDS;
    const elem_t* sV = sK + AK * LDS;
    const int k0 = t * AK;

    // S = Q K^T  (32 x 64 per warp)
    float s[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 8; ++i) s[mt][i][0] = s[mt][i][1] = s[mt][i][2] = s[mt][i][3] = 0.f;
#pragma unroll
    for (int nt2 = 0; nt2 < 4; ++nt2) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sK + (nt2 * 16 + (lane & 7) + 8 * (lane >> 4)) * LDS + ks * 16 + 8 * ((lane >> 3) & 1);
        ldsm_x4(b0, b1, b2, b3, ptr);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(s[mt][2 * nt2], qa[mt][ks], b0, b1);
          mma16816(s[mt][2 * nt2 + 1], qa[mt][ks], b2, b3);
        }
      }
    }
    // bias mode of this (warp, key block): 0 none, 1 all keys left of every row's window, 2 all right of it, 3 mixed
    int bmode = 0;
    if (shaw) {
      if (k0 + AK - 1 - i_lo <= -p.rel_left) bmode = 1;
      else if (k0 - i_hi >= p.rel_right) bmode = 2;
      else bmode = 3;
    }
    const bool need_mask = (k0 + AK > kv_len) || p.causal;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      float mnew[2] = {mrow[mt][0], mrow[mt][1]};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int rr = e >> 1;
          const int i = irow[mt][rr];
          const int j = k0 + nt * 8 + 2 * tq + (e & 1);
          float val = s[mt][nt][e];
          if (bmode == 1) val += bias_l[mt][rr];
          else if (bmode == 2) val += bias_r[mt][rr];
          else if (bmode == 3) {
            int d = j - i;
            d = d < -p.rel_left ? -p.rel_left : (d > p.rel_right ? p.rel_right : d);
            val += qr[(mt * 16 + g + 8 * rr) * (REL_MAX + 1) + d + p.rel_left];
          }
          val *= 0.125f;
          if (need_mask && (j >= kv_len || (p.causal && j > i + causal_off))) val = -INFINITY;
          s[mt][nt][e] = val;
          mnew[rr] = fmaxf(mnew[rr], val);
        }
      }
      float corr[2], msafe[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 1));
        mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 2));
        msafe[rr] = (mnew[rr] == -INFINITY) ? 0.f : mnew[rr];
        corr[rr] = (mrow[mt][rr] == -INFINITY) ? 0.f : __expf(mrow[mt][rr] - msafe[rr]);
        mrow[mt][rr] = mnew[rr];
        lrow[mt][rr] *= corr[rr];
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        o[mt][nt][0] *= corr[0]; o[mt][nt][1] *= corr[0]; o[mt][nt][2] *= corr[1]; o[mt][nt][3] *= corr[1];
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = __expf(s[mt][nt][0] - msafe[0]), p1 = __expf(s[mt][nt][1] - msafe[0]);
        const float p2 = __expf(s[mt][nt][2] - msafe[1]), p3 = __expf(s[mt][nt][3] - msafe[1]);
        lrow[mt][0] += p0 + p1;
        lrow[mt][1] += p2 + p3;
        // keep P in the s registers as packed halves: s[mt][nt][0..1] <- (p0,p1), (p2,p3)
        s[mt][nt][0] = __uint_as_float(pack_h2(p0, p1));
        s[mt][nt][1] = __uint_as_float(pack_h2(p2, p3));
      }
    }
    // O += P V
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {      // 16 keys per k-step
      uint32_t pa[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        pa[mt][0] = __float_as_uint(s[mt][2 * ks][0]);
        pa[mt][1] = __float_as_uint(s[mt][2 * ks][1]);
        pa[mt][2] = __float_as_uint(s[mt][2 * ks + 1][0]);
        pa[mt][3] = __float_as_uint(s[mt][2 * ks + 1][1]);
      }
#pragma unroll
      for (int nt2 = 0; nt2 < 4; ++nt2) { // 16 output dims per ldmatrix
        uint32_t b0, b1, b2, b3;
        const elem_t* ptr = sV + (ks * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LDS + nt2 * 16 + 8 * (lane >> 4);
        ldsm_x4_t(b0, b1, b2, b3, ptr);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(o[mt][2 * nt2], pa[mt], b0, b1);
          mma16816(o[mt][2 * nt2 + 1], pa[mt], b2, b3);
        }
      }
    }
    __syncthreads();  // this stage is overwritten by the load issued in the next iteration
  }
  // finalize
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float l = lrow[mt][rr];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int i = irow[mt][rr];
      if (i >= p.sq) continue;
      const float inv = l > 0.f ? 1.f / l : 0.f;
      elem_t* op = p.out + ((long long)b * p.q_rows + p.q_halo + i) * p.out_ld + h * HD;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        __half2 hv = __floats2half2_rn(o[mt][nt][2 * rr] * inv, o[mt][nt][2 * rr + 1] * inv);
        *reinterpret_cast<__half2*>(op + nt * 8 + 2 * tq) = hv;
      }
    }
}

}  // namespace sb

extern "C" int sb_attention(const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld,
                            void* out, int64_t out_ld, int32_t batch, int32_t heads, int32_t sq, int32_t sk,
                            int32_t q_rows, int32_t q_halo, int32_t kv_rows, int32_t kv_halo, const int32_t* kv_lens,
                            int32_t causal, const void* rel_k, int32_t rel_left, int32_t rel_right, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(q && k && v && out && batch > 0 && heads > 0 && sq > 0 && sk > 0, SB_EINVAL, "sb_attention: bad args");
  SB_REQUIRE((q_ld % 8) == 0 && (k_ld % 8) == 0 && (v_ld % 8) == 0 && (out_ld % 2) == 0, SB_ENOSUP,
             "sb_attention: row strides must be multiples of 8 elements");
  SB_REQUIRE(rel_k == nullptr || rel_left + rel_right + 1 <= REL_MAX, SB_ENOSUP, "sb_attention: rel table too large");
  AttnArgs a;
  a.q = (const elem_t*)q; a.k = (const elem_t*)k; a.v = (const elem_t*)v; a.out = (elem_t*)out;
  a.q_ld = q_ld; a.k_ld = k_ld; a.v_ld = v_ld; a.out_ld = out_ld;
  a.batch = batch; a.heads = heads; a.sq = sq; a.sk = sk; a.q_rows = q_rows; a.q_halo = q_halo;
  a.kv_rows = kv_rows; a.kv_halo = kv_halo; a.kv_lens = kv_lens; a.causal = causal;
  a.rel_k = (const elem_t*)rel_k; a.rel_left = rel_left; a.rel_right = rel_right;
  // opt-in (not timed on H100; tools/attn_bench.py compares the two): the 128-row kernel needs 244 registers per thread in
  // the sm_90a build and 108 KB of shared memory, so fewer warps share an SM, and with one warp doing QK^T -> softmax -> PV
  // in turn the tensor pipe idles during the softmax unless other warps fill in
  static int v2 = -1;
  if (v2 < 0) { const char* e = getenv("SB_ATTENTION_V2"); v2 = (e != nullptr && atoi(e) != 0) ? 1 : 0; }
  if (v2) {
    size_t smem = (size_t)(AQ2 + 4 * AK) * LDS * sizeof(elem_t);
    if (rel_k) smem += (size_t)REL_MAX * LDS * sizeof(elem_t) + 4 * 32 * (REL_MAX + 1) * sizeof(float);
    static bool configured2 = false;
    if (!configured2) {
      SB_CUDA_OK(cudaFuncSetAttribute(attention2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
      configured2 = true;
    }
    dim3 grid((sq + AQ2 - 1) / AQ2, heads, batch);
    attention2_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>(a);
    SB_LAUNCH_OK();
    return SB_OK;
  }
  size_t smem = (size_t)(AQ + 2 * AK) * LDS * sizeof(elem_t);
  if (rel_k) smem += (size_t)REL_MAX * LDS * sizeof(elem_t) + 4 * 16 * (REL_MAX + 1) * sizeof(float);
  static bool configured = false;
  if (!configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  dim3 grid((sq + AQ - 1) / AQ, heads, batch);
  attention_kernel<false><<<grid, 128, smem, (cudaStream_t)stream>>>(a);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_attention_relpos(const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld,
                                   void* out, int64_t out_ld, int32_t batch, int32_t heads, int32_t s, int32_t q_rows,
                                   int32_t q_halo, int32_t kv_rows, int32_t kv_halo, const int32_t* kv_lens, const void* r,
                                   int64_t r_ld, const float* bias_u, const float* bias_v, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(q && k && v && out && r && batch > 0 && heads > 0 && s > 0, SB_EINVAL, "sb_attention_relpos: bad args");
  SB_REQUIRE(s <= XL_MAX_S, SB_ENOSUP, "sb_attention_relpos: sequence length %d exceeds %d", s, XL_MAX_S);
  SB_REQUIRE((q_ld % 8) == 0 && (k_ld % 8) == 0 && (v_ld % 8) == 0 && (r_ld % 8) == 0 && (out_ld % 2) == 0, SB_ENOSUP,
             "sb_attention_relpos: row strides must be multiples of 8 elements");
  XlAttnArgs a = {};
  a.q = (const elem_t*)q; a.k = (const elem_t*)k; a.v = (const elem_t*)v; a.out = (elem_t*)out;
  a.q_ld = q_ld; a.k_ld = k_ld; a.v_ld = v_ld; a.out_ld = out_ld;
  a.batch = batch; a.heads = heads; a.sq = s; a.sk = s; a.q_rows = q_rows; a.q_halo = q_halo;
  a.kv_rows = kv_rows; a.kv_halo = kv_halo; a.kv_lens = kv_lens;
  a.r = (const elem_t*)r; a.r_ld = r_ld; a.bias_u = bias_u; a.bias_v = bias_v;
  // Q, K, V, the 128-row R window, the per-warp 16 x 81 fp32 QR tiles and the (q + v) tile: 77 KB
  const size_t smem = (size_t)(AQ + 2 * AK + XL_ROWS + AQ) * LDS * sizeof(elem_t) + 4 * 16 * (REL_MAX + 1) * sizeof(float);
  static bool configured = false;
  if (!configured) {
    SB_CUDA_OK(cudaFuncSetAttribute(attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  dim3 grid((s + AQ - 1) / AQ, heads, batch);
  attention_kernel<true><<<grid, 128, smem, (cudaStream_t)stream>>>(a);
  SB_LAUNCH_OK();
  return SB_OK;
}
