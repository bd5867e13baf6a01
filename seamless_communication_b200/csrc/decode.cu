// Text-decoder step kernels: embedding frontend, single-token self/cross attention over the KV cache, fused
// log-softmax statistics + top-K, and the device-resident beam-search bookkeeping.
//
// The reference runs beam search on the host (fairseq2 BeamSearchSeq2SeqGenerator; C++ mirror
// ggml/examples/unity/fairseq2.cpp:1371-1608) with one host round trip per step and an index_select copy of the
// whole KV cache per step (reorder_kv_cache, fairseq2.cpp:170-198).  Here the search state lives in device memory,
// no step synchronises with the host, and beam reordering is an ancestor-index table: row r at position t reads
// cache slot anc[r][t]; K/V are written once and never moved.
#include <stdlib.h>

#include "common.cuh"

namespace sb {

constexpr int HD = 64;

// ------------------------------------------------------------------------------------------- embedding frontend
__global__ void embed_kernel(const int* __restrict__ ids, long long ids_ld, const int* __restrict__ step_ptr, int L,
                             const elem_t* __restrict__ embed, const float* __restrict__ pos, float scale,
                             elem_t* __restrict__ x, int dim) {
  // grid: (rows, L); x row = r*L + t.  With step_ptr the single column `*step_ptr` is embedded at position *step_ptr.
  pdl_sync();
  const int r = blockIdx.x, t = blockIdx.y;
  const int id_col0 = step_ptr ? *step_ptr : 0, pos0 = id_col0;
  const int tok = ids[(long long)r * ids_ld + id_col0 + t];
  const elem_t* e = embed + (long long)tok * dim;
  const float* pp = pos + (long long)(pos0 + t) * dim;
  elem_t* xp = x + ((long long)r * L + t) * dim;
  for (int c = threadIdx.x * 2; c < dim; c += blockDim.x * 2) {
    float2 ev = __half22float2(*reinterpret_cast<const __half2*>(e + c));
    *reinterpret_cast<__half2*>(xp + c) = __floats2half2_rn(ev.x * scale + pp[c], ev.y * scale + pp[c + 1]);
  }
}

// ------------------------------------------------------------------------------------------- single-token attention
// One warp per (row, head).  Lane l = (key group kg = l/8, dim chunk dc = l%8): every iteration the warp covers 4
// keys with one 16-byte load per lane (128 B contiguous per key), so loads are independent and coalesced; scores
// are reduced over the 8 lanes of a group with 3 shuffles, outputs over the 4 groups with 2.
template <typename KeyPtr, typename ValPtr>
__device__ __forceinline__ void attend_one(const elem_t* __restrict__ qp, int nkeys, KeyPtr kptr, ValPtr vptr, float* sc,
                                           elem_t* __restrict__ outp) {
  const int lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
  float q[8];
  {
    uint4 u = *reinterpret_cast<const uint4*>(qp + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { float2 f = __half22float2(hh[e]); q[2 * e] = f.x; q[2 * e + 1] = f.y; }
  }
  float mx = -INFINITY;
  // 32 keys per iteration: 8 independent 16-byte loads in flight per lane
  for (int t0 = 0; t0 < nkeys; t0 += 32) {
    uint4 u[8];
    bool ok[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + 4 * i + kg;
      ok[i] = t < nkeys;
      u[i] = ok[i] ? *reinterpret_cast<const uint4*>(kptr(t) + dc * 8) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __half2* hh = reinterpret_cast<const __half2*>(&u[i]);
      float acc = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) { float2 f = __half22float2(hh[e]); acc += q[2 * e] * f.x + q[2 * e + 1] * f.y; }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
      acc *= 0.125f;
      if (ok[i]) {
        if (dc == 0) sc[t0 + 4 * i + kg] = acc;
        mx = fmaxf(mx, acc);
      }
    }
  }
  mx = warp_max(mx);
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < nkeys; t += 32) {
    const float p = __expf(sc[t] - mx);
    sc[t] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;
  for (int t0 = 0; t0 < nkeys; t0 += 32) {
    uint4 u[8];
    float pw[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + 4 * i + kg;
      const bool ok = t < nkeys;
      pw[i] = ok ? sc[t] : 0.f;
      u[i] = ok ? *reinterpret_cast<const uint4*>(vptr(t) + dc * 8) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __half2* hh = reinterpret_cast<const __half2*>(&u[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) { float2 f = __half22float2(hh[e]); o[2 * e] += pw[i] * f.x; o[2 * e + 1] += pw[i] * f.y; }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 8);
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 16);
  }
  if (kg == 0) {
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    uint4 u;
    __half2* hh = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) hh[e] = __floats2half2_rn(o[2 * e] * inv, o[2 * e + 1] * inv);
    *reinterpret_cast<uint4*>(outp + dc * 8) = u;
  }
}

// q / k / v of the new token either come as fp16 (`qkv`) or as split-K partial products of the projection
// (`part`: [splits][slice_rows][3*dim] fp32, plus the projection bias): summing the slices here removes the separate
// reduction pass between the skinny qkv GEMM and the attention.
__device__ __forceinline__ void gather_head_vec(const float* __restrict__ part, int splits, long long slice_rows, long long ld,
                                                const float* __restrict__ bias, long long row, int col0, elem_t* dst) {
  // All slices are requested before the first one is used (a plain loop serialises one L2 round trip per slice: with 4-8
  // slices that was most of the attention kernels' time).
  const int lane = threadIdx.x & 31;
  float2 acc = *reinterpret_cast<const float2*>(bias + col0 + 2 * lane);
  const float* pp = part + row * ld + col0 + 2 * lane;
  const long long zs = slice_rows * ld;
  int z = 0;
  for (; z + 8 <= splits; z += 8) {
    float2 p[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) p[u] = *reinterpret_cast<const float2*>(pp + (z + u) * zs);
#pragma unroll
    for (int u = 0; u < 8; ++u) { acc.x += p[u].x; acc.y += p[u].y; }
  }
  if (z + 4 <= splits) {
    float2 p[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) p[u] = *reinterpret_cast<const float2*>(pp + (z + u) * zs);
#pragma unroll
    for (int u = 0; u < 4; ++u) { acc.x += p[u].x; acc.y += p[u].y; }
    z += 4;
  }
  for (; z < splits; ++z) {
    const float2 p = *reinterpret_cast<const float2*>(pp + z * zs);
    acc.x += p.x; acc.y += p.y;
  }
  reinterpret_cast<__half2*>(dst)[lane] = __floats2half2_rn(acc.x, acc.y);
}

__global__ void __launch_bounds__(128) decode_self_attn_kernel(const elem_t* __restrict__ qkv, const float* __restrict__ part,
                                                               int splits, long long slice_rows, const float* __restrict__ bias,
                                                               elem_t* __restrict__ kcache, elem_t* __restrict__ vcache,
                                                               const int* __restrict__ anc, int anc_ld,
                                                               const int* __restrict__ step_ptr, int max_len,
                                                               elem_t* __restrict__ out, int rows, int heads) {
  extern __shared__ float sc_all[];  // [4][max_len] scores + [4][max_len] ancestor slots
  __shared__ __align__(16) elem_t s_new[4][3][HD];
  pdl_sync();
  const int step = *step_ptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x;
  const int h = blockIdx.y * 4 + warp;
  if (h >= heads) return;
  const int dim = heads * HD;
  float* sc = sc_all + warp * max_len;
  int* slots = reinterpret_cast<int*>(sc_all + 4 * max_len) + warp * max_len;
  const elem_t *qp, *knew, *vnew;
  if (part != nullptr) {
#pragma unroll
    for (int t = 0; t < 3; ++t) gather_head_vec(part, splits, slice_rows, 3LL * dim, bias, r, t * dim + h * HD, s_new[warp][t]);
    __syncwarp();
    qp = s_new[warp][0]; knew = s_new[warp][1]; vnew = s_new[warp][2];
  } else {
    qp = qkv + (long long)r * 3 * dim + h * HD;
    knew = qp + dim;
    vnew = qp + 2 * dim;
  }
  // persist the new K/V (slot r, position step)
  {
    elem_t* kd = kcache + ((long long)step * rows + r) * dim + h * HD;
    elem_t* vd = vcache + ((long long)step * rows + r) * dim + h * HD;
    reinterpret_cast<__half2*>(kd)[lane] = reinterpret_cast<const __half2*>(knew)[lane];
    reinterpret_cast<__half2*>(vd)[lane] = reinterpret_cast<const __half2*>(vnew)[lane];
  }
  for (int t = lane; t < step; t += 32) slots[t] = anc[(long long)r * anc_ld + t];
  __syncwarp();
  const long long hoff = (long long)h * HD;
  auto kptr = [&](int t) -> const elem_t* {
    return (t == step) ? knew : kcache + ((long long)t * rows + slots[t]) * dim + hoff;
  };
  auto vptr = [&](int t) -> const elem_t* {
    return (t == step) ? vnew : vcache + ((long long)t * rows + slots[t]) * dim + hoff;
  };
  attend_one(qp, step + 1, kptr, vptr, sc, out + (long long)r * dim + hoff);
}

// Same computation with the dependent round trips removed (a kernel of this size pays a full L2 / HBM latency per
// DEPENDENT global access, and the version above chains 13 of them: step, three slice gathers, ancestry, four key rounds, four value rounds):
//   round 1: step index, every split-K slice of q | k | v, the whole ancestry row - all independent, requested together;
//   then 32 keys per round with the key AND the value rows of the round in flight together (online softmax).
__global__ void __launch_bounds__(128) decode_self_attn2_kernel(const float* __restrict__ part, int splits, long long slice_rows,
                                                                const float* __restrict__ bias, elem_t* __restrict__ kcache,
                                                                elem_t* __restrict__ vcache, const int* __restrict__ anc, int anc_ld,
                                                                const int* __restrict__ step_ptr, int max_len,
                                                                elem_t* __restrict__ out, int rows, int heads) {
  extern __shared__ int sa_slots_all[];  // [4][max_len] ancestor slots
  __shared__ __align__(16) elem_t s_new[4][3][HD];
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
  const int r = blockIdx.x;
  const int h = blockIdx.y * 4 + warp;
  if (h >= heads) return;
  const int dim = heads * HD;
  int* slots = sa_slots_all + warp * max_len;
  // ---- round 1
  const int step = *step_ptr;
  const int* arow = anc + (long long)r * anc_ld;
  int sl_reg[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) sl_reg[j] = (lane + 32 * j < max_len) ? arow[lane + 32 * j] : 0;
  float2 acc[3];
  const float* pp = part + (long long)r * 3 * dim + h * HD + 2 * lane;
  const long long zs = slice_rows * 3LL * dim;
#pragma unroll
  for (int t = 0; t < 3; ++t) acc[t] = *reinterpret_cast<const float2*>(bias + t * dim + h * HD + 2 * lane);
  for (int z0 = 0; z0 < splits; z0 += 4) {
    float2 p[4][3];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int t = 0; t < 3; ++t)
        p[u][t] = (z0 + u < splits) ? *reinterpret_cast<const float2*>(pp + (z0 + u) * zs + t * dim) : make_float2(0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int t = 0; t < 3; ++t) { acc[t].x += p[u][t].x; acc[t].y += p[u][t].y; }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (lane + 32 * j < max_len) slots[lane + 32 * j] = sl_reg[j];
  for (int t = lane + 128; t < step; t += 32) slots[t] = arow[t];  // max_len > 128
#pragma unroll
  for (int t = 0; t < 3; ++t) reinterpret_cast<__half2*>(s_new[warp][t])[lane] = __floats2half2_rn(acc[t].x, acc[t].y);
  __syncwarp();
  const elem_t *qp = s_new[warp][0], *knew = s_new[warp][1], *vnew = s_new[warp][2];
  {  // persist the new K/V (slot r, position step)
    elem_t* kd = kcache + ((long long)step * rows + r) * dim + h * HD;
    elem_t* vd = vcache + ((long long)step * rows + r) * dim + h * HD;
    reinterpret_cast<__half2*>(kd)[lane] = reinterpret_cast<const __half2*>(knew)[lane];
    reinterpret_cast<__half2*>(vd)[lane] = reinterpret_cast<const __half2*>(vnew)[lane];
  }
  float q[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(qp + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); q[2 * e] = f.x; q[2 * e + 1] = f.y; }
  }
  const long long hoff = (long long)h * HD + dc * 8;
  const int nkeys = step + 1;
  float m = -INFINITY, l = 0.f, o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;
  for (int t0 = 0; t0 < nkeys; t0 += 32) {
    uint4 ku[8], vu[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + 4 * i + kg;
      if (t < step) {
        const long long off = ((long long)t * rows + slots[t]) * dim + hoff;
        ku[i] = *reinterpret_cast<const uint4*>(kcache + off);
        vu[i] = *reinterpret_cast<const uint4*>(vcache + off);
      } else if (t == step) {
        ku[i] = *reinterpret_cast<const uint4*>(knew + dc * 8);
        vu[i] = *reinterpret_cast<const uint4*>(vnew + dc * 8);
      } else {
        ku[i] = make_uint4(0, 0, 0, 0);
        vu[i] = make_uint4(0, 0, 0, 0);
      }
    }
    float sc[8], cm = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __half2* hh = reinterpret_cast<const __half2*>(&ku[i]);
      float a = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); a += q[2 * e] * f.x + q[2 * e + 1] * f.y; }
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      a += __shfl_xor_sync(0xffffffffu, a, 4);
      sc[i] = (t0 + 4 * i + kg < nkeys) ? a * 0.125f : -INFINITY;
      cm = fmaxf(cm, sc[i]);
    }
    cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 8));
    cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 16));
    const float m_new = fmaxf(m, cm);  // finite: every round holds at least one valid key
    const float scale = __expf(m - m_new);
    m = m_new;
    l *= scale;
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] *= scale;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float pw = __expf(sc[i] - m);
      l += pw;
      const __half2* hh = reinterpret_cast<const __half2*>(&vu[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); o[2 * e] += pw * f.x; o[2 * e + 1] += pw * f.y; }
    }
  }
  l += __shfl_xor_sync(0xffffffffu, l, 8);
  l += __shfl_xor_sync(0xffffffffu, l, 16);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 8);
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 16);
  }
  if (kg == 0) {
    const float inv = l > 0.f ? 1.f / l : 0.f;
    uint4 w;
    __half2* hh = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) hh[e] = __floats2half2_rn(o[2 * e] * inv, o[2 * e + 1] * inv);
    *reinterpret_cast<uint4*>(out + (long long)r * dim + (long long)h * HD + dc * 8) = w;
  }
}

__global__ void __launch_bounds__(128) decode_cross_attn_kernel(const elem_t* __restrict__ q, const float* __restrict__ part,
                                                                int splits, long long slice_rows, const float* __restrict__ bias,
                                                                const elem_t* __restrict__ k,
                                                                const elem_t* __restrict__ v, long long kv_ld,
                                                                const int* __restrict__ enc_lens, int s_enc,
                                                                elem_t* __restrict__ out, int rows, int beam, int heads) {
  extern __shared__ float sc_all[];  // [4][s_enc]
  __shared__ __align__(16) elem_t s_q[4][HD];
  pdl_sync();
  const int warp = threadIdx.x >> 5;
  const int r = blockIdx.x;
  const int h = blockIdx.y * 4 + warp;
  if (h >= heads) return;
  const int dim = heads * HD;
  const int b = r / beam;
  const int len = enc_lens ? min(enc_lens[b], s_enc) : s_enc;
  float* sc = sc_all + warp * s_enc;
  const elem_t* kb = k + (long long)b * s_enc * kv_ld + h * HD;
  const elem_t* vb = v + (long long)b * s_enc * kv_ld + h * HD;
  auto kptr = [&](int t) -> const elem_t* { return kb + (long long)t * kv_ld; };
  auto vptr = [&](int t) -> const elem_t* { return vb + (long long)t * kv_ld; };
  const elem_t* qp = q + (long long)r * dim + h * HD;
  if (part != nullptr) {
    gather_head_vec(part, splits, slice_rows, dim, bias, r, h * HD, s_q[warp]);
    __syncwarp();
    qp = s_q[warp];
  }
  attend_one(qp, len, kptr, vptr, sc, out + (long long)r * dim + h * HD);
}

// Cross-attention of ALL hypotheses of one sentence in one CTA (grid: sentence x head, one warp per hypothesis).  The beams
// of a sentence attend the same encoder keys: the CTA stages K and V of its (sentence, head) in shared memory once instead
// of every (row, head) warp streaming them from L2 (160 rows x 16 heads x 63 keys x 256 B = 41 MB per layer and step against
// 8 MB unique).  Scores -> probabilities (shared memory) -> values:
// no dependent global round trip after the staging.  Lane = (key group kg, dim chunk dc) as in attend_one.
__global__ void __launch_bounds__(256) decode_cross_attn_shared_kernel(const float* __restrict__ part, int splits, long long slice_rows,
                                                                       const float* __restrict__ bias, const elem_t* __restrict__ k,
                                                                       const elem_t* __restrict__ v, long long kv_ld,
                                                                       const int* __restrict__ enc_lens, int s_enc,
                                                                       elem_t* __restrict__ out, int beam, int heads) {
  extern __shared__ __align__(16) unsigned char cs_smem[];
  pdl_sync();
  const int b = blockIdx.x, h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, kg = lane >> 3, dc = lane & 7;
  const int dim = heads * HD;
  elem_t* ks = reinterpret_cast<elem_t*>(cs_smem);
  elem_t* vs = ks + (size_t)s_enc * HD;
  float* ps = reinterpret_cast<float*>(vs + (size_t)s_enc * HD) + warp * s_enc;
  elem_t* qs = reinterpret_cast<elem_t*>(reinterpret_cast<float*>(vs + (size_t)s_enc * HD) + (blockDim.x >> 5) * s_enc) + warp * HD;
  const elem_t* kb = k + (long long)b * s_enc * kv_ld + h * HD;
  const elem_t* vb = v + (long long)b * s_enc * kv_ld + h * HD;
  const long long r = (long long)b * beam + warp;
  // Every global read of the kernel is independent of the others: request them all before the first use (a kernel of this
  // size costs one L2 round trip per DEPENDENT access; the valid length only masks the arithmetic, rows past it are read too).
  const int n16 = s_enc * 8;
  uint4 kreg[2], vreg[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = threadIdx.x + j * blockDim.x;
    if (i < n16) {
      kreg[j] = *reinterpret_cast<const uint4*>(kb + (long long)(i >> 3) * kv_ld + (i & 7) * 8);
      vreg[j] = *reinterpret_cast<const uint4*>(vb + (long long)(i >> 3) * kv_ld + (i & 7) * 8);
    }
  }
  const int len = enc_lens ? min(enc_lens[b], s_enc) : s_enc;
  if (warp < beam) gather_head_vec(part, splits, slice_rows, dim, bias, r, h * HD, qs);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = threadIdx.x + j * blockDim.x;
    if (i < n16) {
      reinterpret_cast<uint4*>(ks)[i] = kreg[j];
      reinterpret_cast<uint4*>(vs)[i] = vreg[j];
    }
  }
  for (int i = threadIdx.x + 2 * blockDim.x; i < n16; i += blockDim.x) {  // encoders longer than 64 (32) frames
    reinterpret_cast<uint4*>(ks)[i] = *reinterpret_cast<const uint4*>(kb + (long long)(i >> 3) * kv_ld + (i & 7) * 8);
    reinterpret_cast<uint4*>(vs)[i] = *reinterpret_cast<const uint4*>(vb + (long long)(i >> 3) * kv_ld + (i & 7) * 8);
  }
  __syncthreads();
  if (warp >= beam) return;
  float q[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(qs + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); q[2 * e] = f.x; q[2 * e + 1] = f.y; }
  }
  float mx = -INFINITY;
  for (int t0 = 0; t0 < len; t0 += 4) {  // warp-uniform trip count
    const int t = t0 + kg;
    const bool ok = t < len;
    const uint4 u = ok ? *reinterpret_cast<const uint4*>(ks + (size_t)t * HD + dc * 8) : make_uint4(0, 0, 0, 0);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); a += q[2 * e] * f.x + q[2 * e + 1] * f.y; }
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    a += __shfl_xor_sync(0xffffffffu, a, 4);
    a *= 0.125f;
    if (ok) {
      if (dc == 0) ps[t] = a;
      mx = fmaxf(mx, a);
    }
  }
  mx = warp_max(mx);
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < len; t += 32) {
    const float p = __expf(ps[t] - mx);
    ps[t] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;
  for (int t = kg; t < len; t += 4) {
    const float p = ps[t];
    const uint4 u = *reinterpret_cast<const uint4*>(vs + (size_t)t * HD + dc * 8);
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); o[2 * e] += p * f.x; o[2 * e + 1] += p * f.y; }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 8);
    o[e] += __shfl_xor_sync(0xffffffffu, o[e], 16);
  }
  if (kg == 0) {
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    uint4 w;
    __half2* hh = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) hh[e] = __floats2half2_rn(o[2 * e] * inv, o[2 * e + 1] * inv);
    *reinterpret_cast<uint4*>(out + r * dim + h * HD + dc * 8) = w;
  }
}

// ------------------------------------------------------------------------------------------- log-softmax stats + top-K
// One CTA per row, two streaming passes (the second one hits L2):
//   pass 1: online max / sum-exp over the raw logits, plus each thread's single best candidate;
//           tau = K-th largest of the per-thread bests is a lower bound of the K-th largest candidate overall;
//   pass 2: every candidate >= tau (a few dozen at most, barring massive ties) is appended to a shared list;
//   a single warp then extracts the top K in (value desc, index asc) order.
constexpr int TK_MAX = 16;
constexpr int TK_THREADS = 512;
constexpr int TK_CAP = 2048;

__device__ __forceinline__ float tk_cand(float x, int i, int pad_idx, int unk_idx, float unk_penalty) {
  if (i == pad_idx) return -INFINITY;            // never allow PAD (fairseq2.cpp:1293-1296)
  if (i == unk_idx) return x - unk_penalty;      // UNK penalty (fairseq2.cpp:1298-1305)
  return x;
}

__global__ void __launch_bounds__(TK_THREADS) logits_topk_kernel(const float* __restrict__ logits, long long ld, int vocab,
                                                                 int pad_idx, int eos_idx, int unk_idx, float unk_penalty, int K,
                                                                 float* __restrict__ cand_val, int* __restrict__ cand_idx,
                                                                 float* __restrict__ eos_lprob) {
  pdl_sync();
  const int r = blockIdx.x;
  const float* row = logits + (long long)r * ld;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float s_m[TK_THREADS / 32], s_s[TK_THREADS / 32];
  __shared__ float s_best[TK_THREADS];
  __shared__ float s_lse, s_tau;
  __shared__ int s_count;
  __shared__ float s_cv[TK_CAP];
  __shared__ int s_ci[TK_CAP];
  const int nvec = vocab >> 2;
  // ---- pass 1
  float mx = -INFINITY, sum = 0.f, best = -INFINITY;
  for (int i = threadIdx.x; i < nvec; i += TK_THREADS) {
    const float4 v = *reinterpret_cast<const float4*>(row + 4 * i);
    const float xs[4] = {v.x, v.y, v.z, v.w};
    const float m4 = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
    if (m4 > mx) { sum *= __expf(mx - m4); mx = m4; }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sum += __expf(xs[e] - mx);
      best = fmaxf(best, tk_cand(xs[e], 4 * i + e, pad_idx, unk_idx, unk_penalty));
    }
  }
  for (int i = 4 * nvec + threadIdx.x; i < vocab; i += TK_THREADS) {
    const float x = row[i];
    if (x > mx) { sum *= __expf(mx - x); mx = x; }
    sum += __expf(x - mx);
    best = fmaxf(best, tk_cand(x, i, pad_idx, unk_idx, unk_penalty));
  }
  s_best[threadIdx.x] = best;
  {
    const float m2 = warp_max(mx);
    const float s2 = warp_sum(mx == -INFINITY ? 0.f : sum * __expf(mx - m2));
    if (lane == 0) { s_m[warp] = m2; s_s[warp] = s2; }
  }
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  if (warp == 0) {
    float M = -INFINITY;
    for (int i = 0; i < TK_THREADS / 32; ++i) M = fmaxf(M, s_m[i]);
    float S = 0.f;
    for (int i = 0; i < TK_THREADS / 32; ++i) S += s_s[i] * __expf(s_m[i] - M);
    if (lane == 0) {
      s_lse = M + logf(S);
      eos_lprob[r] = row[eos_idx] - (M + logf(S));
    }
    // K-th largest of the 512 per-thread bests: each lane owns 16 of them
    float loc[TK_THREADS / 32];
#pragma unroll
    for (int i = 0; i < TK_THREADS / 32; ++i) loc[i] = s_best[lane * (TK_THREADS / 32) + i];
    float tau = -INFINITY;
    for (int round = 0; round < K; ++round) {
      float lm = -INFINITY; int li = 0;
#pragma unroll
      for (int i = 0; i < TK_THREADS / 32; ++i) if (loc[i] > lm) { lm = loc[i]; li = i; }
      const float wm = warp_max(lm);
      tau = wm;
      // the first lane holding the maximum removes one copy
      const unsigned ball = __ballot_sync(0xffffffffu, lm == wm);
      if (lane == __ffs(ball) - 1) {
#pragma unroll
        for (int i = 0; i < TK_THREADS / 32; ++i) if (i == li) loc[i] = -INFINITY;
      }
    }
    if (lane == 0) s_tau = tau;
  }
  __syncthreads();
  const float tau = s_tau, lse = s_lse;
  // ---- pass 2: gather candidates >= tau
  for (int i = threadIdx.x; i < nvec; i += TK_THREADS) {
    const float4 v = *reinterpret_cast<const float4*>(row + 4 * i);
    const float xs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float cv = tk_cand(xs[e], 4 * i + e, pad_idx, unk_idx, unk_penalty);
      if (cv >= tau && cv > -INFINITY) {
        const int slot = atomicAdd(&s_count, 1);
        if (slot < TK_CAP) { s_cv[slot] = cv; s_ci[slot] = 4 * i + e; }
      }
    }
  }
  for (int i = 4 * nvec + threadIdx.x; i < vocab; i += TK_THREADS) {
    const float cv = tk_cand(row[i], i, pad_idx, unk_idx, unk_penalty);
    if (cv >= tau && cv > -INFINITY) {
      const int slot = atomicAdd(&s_count, 1);
      if (slot < TK_CAP) { s_cv[slot] = cv; s_ci[slot] = i; }
    }
  }
  __syncthreads();
  // ---- top-K of the candidate list, one warp
  if (warp == 0) {
    const int n = min(s_count, TK_CAP);
    for (int round = 0; round < K; ++round) {
      float bv = -INFINITY; int bi = 0x7fffffff, bs = -1;
      for (int j = lane; j < n; j += 32) {
        const float v = s_cv[j]; const int id = s_ci[j];
        if (v > bv || (v == bv && id < bi)) { bv = v; bi = id; bs = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        const int s2 = __shfl_xor_sync(0xffffffffu, bs, o);
        if (v2 > bv || (v2 == bv && i2 < bi)) { bv = v2; bi = i2; bs = s2; }
      }
      if (lane == 0) {
        cand_val[(long long)r * K + round] = bs >= 0 ? bv - lse : -INFINITY;
        cand_idx[(long long)r * K + round] = bs >= 0 ? bi : 0;
        if (bs >= 0) s_cv[bs] = -INFINITY;
      }
      __syncwarp();
    }
  }
}

// Top-K from per-tile statistics (written by the projection GEMM's epilogue, sb_gemm tile_stats): one CTA per row.
//   1. log-sum-exp of the row from the (max, sum-exp) pairs of its tiles;
//   2. tau = (K+2)-th largest tile maximum: at least K+2 elements are >= tau, so at least K CANDIDATES are (PAD is never a
//      candidate and the UNK penalty can push one more below);
//   3. only the tiles whose maximum reaches tau are read back (one warp per tile, 512 B) and their elements >= tau collected;
//   4. the same (value desc, index asc) extraction as logits_topk_kernel.
constexpr int TKT_THREADS = 256;
constexpr int TKT_TILE = 128;

__global__ void __launch_bounds__(TKT_THREADS) logits_topk_tiles_kernel(const float* __restrict__ logits, long long ld,
                                                                        const float2* __restrict__ stats, int rows, int vocab,
                                                                        int pad_idx, int eos_idx, int unk_idx, float unk_penalty, int K,
                                                                        float* __restrict__ cand_val, int* __restrict__ cand_idx,
                                                                        float* __restrict__ eos_lprob) {
  extern __shared__ float tk_sm[];  // tile maxima [n_tiles]
  pdl_sync();
  const int r = blockIdx.x;
  const float* row = logits + (long long)r * ld;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = TKT_THREADS / 32;
  const int n_tiles = (vocab + TKT_TILE - 1) / TKT_TILE;
  __shared__ float s_red[TKT_THREADS / 32];
  __shared__ int s_redi[TKT_THREADS / 32];
  __shared__ float s_lse, s_tau;
  __shared__ int s_count;
  __shared__ float s_cv[TK_CAP];
  __shared__ int s_ci[TK_CAP];
  // ---- 1. row log-sum-exp
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n_tiles; i += TKT_THREADS) {
    const float m = stats[(long long)i * rows + r].x;
    tk_sm[i] = m;
    mx = fmaxf(mx, m);
  }
  mx = warp_max(mx);
  if (lane == 0) s_red[warp] = mx;
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  float M = -INFINITY;
  for (int i = 0; i < nwarp; ++i) M = fmaxf(M, s_red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < n_tiles; i += TKT_THREADS) {
    const float2 ms = stats[(long long)i * rows + r];
    sum += ms.y * __expf(ms.x - M);
  }
  sum = warp_sum(sum);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float S = 0.f;
    for (int i = 0; i < nwarp; ++i) S += s_red[i];
    s_lse = M + logf(S);
    eos_lprob[r] = row[eos_idx] - (M + logf(S));
  }
  __syncthreads();
  // ---- 2. tau = (K+2)-th largest tile maximum (block-wide arg-max, K+2 rounds; the found tile is marked by negating into
  // a side copy: tk_sm keeps the maxima, the removal is tracked in the sign-safe way below)
  // a removed maximum is remembered as NaN in a second array to keep tk_sm intact for step 3
  float* live = tk_sm + n_tiles;
  for (int i = threadIdx.x; i < n_tiles; i += TKT_THREADS) live[i] = tk_sm[i];
  __syncthreads();
  const int rounds = min(K + 2, n_tiles);
  float tau = -INFINITY;
  for (int round = 0; round < rounds; ++round) {
    float bm = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n_tiles; i += TKT_THREADS) {
      const float m = live[i];
      if (m > bm || (m == bm && i < bi)) { bm = m; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, bm, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (m2 > bm || (m2 == bm && i2 < bi)) { bm = m2; bi = i2; }
    }
    if (lane == 0) { s_red[warp] = bm; s_redi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = s_red[0];
      int ix = s_redi[0];
      for (int i = 1; i < nwarp; ++i)
        if (s_red[i] > m || (s_red[i] == m && s_redi[i] < ix)) { m = s_red[i]; ix = s_redi[i]; }
      if (ix < n_tiles) live[ix] = -INFINITY;
      s_tau = m;
    }
    __syncthreads();
    tau = s_tau;
  }
  // ---- 3. gather candidates >= tau from the tiles that can hold one
  for (int t = warp; t < n_tiles; t += nwarp) {
    if (!(tk_sm[t] >= tau)) continue;  // warp-uniform
    const int i0 = t * TKT_TILE + lane * 4;
    float xs[4];
    if (i0 + 3 < vocab) {
      const float4 v4 = *reinterpret_cast<const float4*>(row + i0);
      xs[0] = v4.x; xs[1] = v4.y; xs[2] = v4.z; xs[3] = v4.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) xs[e] = (i0 + e < vocab) ? row[i0 + e] : -INFINITY;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (i0 + e >= vocab) continue;
      const float cv = tk_cand(xs[e], i0 + e, pad_idx, unk_idx, unk_penalty);
      if (cv >= tau && cv > -INFINITY) {
        const int slot = atomicAdd(&s_count, 1);
        if (slot < TK_CAP) { s_cv[slot] = cv; s_ci[slot] = i0 + e; }
      }
    }
  }
  __syncthreads();
  // ---- 4. top-K of the candidate list, one warp
  if (warp == 0) {
    const float lse = s_lse;
    const int n = min(s_count, TK_CAP);
    for (int round = 0; round < K; ++round) {
      float bv = -INFINITY; int bi = 0x7fffffff, bs = -1;
      for (int j = lane; j < n; j += 32) {
        const float v = s_cv[j]; const int id = s_ci[j];
        if (v > bv || (v == bv && id < bi)) { bv = v; bi = id; bs = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        const int s2 = __shfl_xor_sync(0xffffffffu, bs, o);
        if (v2 > bv || (v2 == bv && i2 < bi)) { bv = v2; bi = i2; bs = s2; }
      }
      if (lane == 0) {
        cand_val[(long long)r * K + round] = bs >= 0 ? bv - lse : -INFINITY;
        cand_idx[(long long)r * K + round] = bs >= 0 ? bi : 0;
        if (bs >= 0) s_cv[bs] = -INFINITY;
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------- beam bookkeeping
// one CTA per sentence; the step index is read from device memory so that one captured CUDA graph serves every step
__global__ void __launch_bounds__(128) beam_step_kernel(const sb_beam_t p) {
  pdl_sync();
  const int b = blockIdx.x;
  const int beam = p.beam, K = p.K, ML = p.max_len;  // ML: row stride of the state arrays
  const int step = *p.step_ptr;
  const int budget = p.len_budget != nullptr ? min(*p.len_budget, ML) : ML;
  __shared__ int s_parent[16];
  __shared__ int s_tok[16];
  __shared__ float s_score[16];
  __shared__ int s_active;
  if (step + 1 >= budget) return;  // search exhausted (graph replays beyond the last step are no-ops)
  if (threadIdx.x == 0) {
    int active = p.active[b];
    if (active) {
      const bool first_step = (step == p.prefix_len - 1);
      const int nsrc = first_step ? 1 : beam;  // first step: all beams are identical, use beam 0 (fairseq2.cpp:1499-1510)
      int used[16];
      bool forced_taken[16];
      for (int i = 0; i < nsrc; ++i) { used[i] = 0; forced_taken[i] = false; }
      const bool force_eos = (step == budget - 2);  // _tweak_lprobs fairseq2.cpp:1280-1291
      const bool block_eos = (step < p.min_len); // fairseq2.cpp:1273-1278
      int n_ongoing = 0, fin = p.fin_count[b];
      const int want = 2 * beam;
      for (int pick = 0; pick < want && n_ongoing < beam && active; ++pick) {
        float best = -INFINITY; int bb = -1, tok = -1;
        for (int i = 0; i < nsrc; ++i) {
          const int row = b * beam + i;
          const float base = p.scores[(long long)row * ML + step];
          float v; int t;
          if (force_eos) {
            if (forced_taken[i]) continue;
            v = p.eos_lprob[row] + base; t = p.eos_idx;
          } else {
            int u = used[i];
            while (u < K && block_eos && p.cand_idx[(long long)row * K + u] == p.eos_idx) ++u;
            used[i] = u;
            if (u >= K) continue;
            v = p.cand_val[(long long)row * K + u] + base; t = p.cand_idx[(long long)row * K + u];
          }
          // order: higher value first; ties by lower flat index (beam*V + token)
          if (bb < 0 || v > best || (v == best && ((long long)i * p.vocab + t) < ((long long)bb * p.vocab + tok))) {
            best = v; bb = i; tok = t;
          }
        }
        if (bb < 0) break;
        if (force_eos) forced_taken[bb] = true; else used[bb]++;
        if (tok == p.eos_idx && best != -INFINITY) {
          // _finalize_hypothesis (fairseq2.cpp:1310-1350)
          const int row = b * beam + bb;
          int* dst = p.fin_seqs + ((long long)b * beam + fin) * ML;
          for (int t = 0; t <= step; ++t) dst[t] = p.seqs[(long long)row * ML + t];
          dst[step + 1] = tok;
          if (p.fin_anc != nullptr) {  // cache slots holding the decoder states of this hypothesis, position by position
            int* fa = p.fin_anc + ((long long)b * beam + fin) * ML;
            for (int t = 0; t < step; ++t) fa[t] = p.anc[(long long)row * ML + t];
            fa[step] = row;
          }
          p.fin_len[b * beam + fin] = step + 2;
          p.fin_score[b * beam + fin] = best / powf((float)(step + 1), p.len_penalty);
          ++fin;
          if (fin == beam) active = 0;
          continue;
        }
        s_parent[n_ongoing] = bb; s_tok[n_ongoing] = tok; s_score[n_ongoing] = best;
        ++n_ongoing;
      }
      p.fin_count[b] = fin;
      if (!active) {
        p.active[b] = 0;
        if (p.n_active) atomicSub(p.n_active, 1);
      } else {
        // fewer than `beam` continuations can only happen with -inf scores; pad by repeating the last one
        for (int i = n_ongoing; i < beam; ++i) {
          s_parent[i] = n_ongoing > 0 ? s_parent[n_ongoing - 1] : 0;
          s_tok[i] = n_ongoing > 0 ? s_tok[n_ongoing - 1] : p.eos_idx;
          s_score[i] = -INFINITY;
        }
      }
    }
    s_active = active;
  }
  __syncthreads();
  if (!s_active) return;
  // in-place beam reorder, column by column: thread t reads column t of every parent row, then writes it back
  for (int t = threadIdx.x; t <= step + 1; t += blockDim.x) {
    int sv[16]; float cv[16]; int av[16];
    for (int i = 0; i < beam; ++i) {
      const long long src = (long long)(b * beam + s_parent[i]) * ML + t;
      sv[i] = p.seqs[src]; cv[i] = p.scores[src]; av[i] = p.anc[src];
      if (t == step) av[i] = b * beam + s_parent[i];  // K/V of position `step` live in the parent's slot
      if (t == step + 1) { sv[i] = s_tok[i]; cv[i] = s_score[i]; }
    }
    for (int i = 0; i < beam; ++i) {
      const long long dst = (long long)(b * beam + i) * ML + t;
      p.seqs[dst] = sv[i]; p.scores[dst] = cv[i]; p.anc[dst] = av[i];
    }
  }
}

// hist[step][...] = h: keeps the final-LayerNorm decoder state of every search step so that the states of the winning
// hypothesis can be gathered afterwards instead of re-running the decoder teacher-forced (inference/generator.py:294-299)
__global__ void store_step_kernel(const uint4* __restrict__ h, uint4* __restrict__ hist, const int* __restrict__ step_ptr, long long n16) {
  pdl_sync();
  uint4* dst = hist + (long long)(*step_ptr) * n16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (long long)gridDim.x * blockDim.x) dst[i] = h[i];
}

__global__ void step_advance_kernel(int* step_ptr) {
  pdl_sync();
  *step_ptr += 1;
}

}  // namespace sb

extern "C" int sb_embed_step(const int32_t* seqs, int32_t seq_ld, const int32_t* step_ptr, const void* embed,
                             const void* pos_table, float scale, void* x, int32_t rows, int32_t dim, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(seqs && step_ptr && embed && pos_table && x && rows > 0 && dim % 2 == 0, SB_EINVAL, "sb_embed_step: bad args");
  SB_CUDA_OK(launch_k(embed_kernel, dim3(rows, 1), dim3(128), 0, (cudaStream_t)stream, (const int*)seqs, (long long)seq_ld,
                       (const int*)step_ptr, 1, (const elem_t*)embed, (const float*)pos_table, scale, (elem_t*)x, (int)dim));
  count_launch();
  return SB_OK;
}

extern "C" int sb_embed_seq(const int32_t* ids, int32_t ids_ld, int32_t L, const void* embed, const void* pos_table,
                            float scale, void* x, int32_t rows, int32_t dim, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(ids && embed && pos_table && x && rows > 0 && L > 0 && dim % 2 == 0, SB_EINVAL, "sb_embed_seq: bad args");
  embed_kernel<<<dim3(rows, L), 128, 0, (cudaStream_t)stream>>>(ids, ids_ld, nullptr, L, (const elem_t*)embed,
                                                                (const float*)pos_table, scale, (elem_t*)x, dim);
  SB_LAUNCH_OK();
  return SB_OK;
}

// A launch whose dynamic plus static shared memory exceeds 48 KB needs the kernel's opt-in attribute (set per device, so
// it is set on every such launch; the self-attention kernels hold 1.5 KB of static staging next to their dynamic scratch)
template <typename Kernel>
static cudaError_t allow_dynamic_smem(Kernel kernel, size_t dyn) {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, kernel);
  if (e != cudaSuccess || dyn + a.sharedSizeBytes <= 48 * 1024) return e;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
}

extern "C" int sb_decode_self_attn(const void* qkv, const float* qkv_partials, int32_t splits, int64_t slice_rows,
                                   const float* qkv_bias, void* kcache, void* vcache, const int32_t* anc, int32_t anc_ld,
                                   const int32_t* step_ptr, int32_t max_len, void* out, int32_t rows, int32_t heads,
                                   sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE((qkv || (qkv_partials && qkv_bias && splits >= 1)) && kcache && vcache && anc && out && step_ptr && rows > 0 &&
                 heads > 0 && max_len > 0,
             SB_EINVAL, "sb_decode_self_attn: bad args");
  static int v2 = -1;
  if (v2 < 0) { const char* e = getenv("SB_SELF_ATTN_V2"); v2 = (e == nullptr || atoi(e) != 0) ? 1 : 0; }
  if (v2 && qkv == nullptr && (size_t)4 * max_len * sizeof(int) <= 48 * 1024) {
    if (max_len > 2048) SB_CUDA_OK(allow_dynamic_smem(decode_self_attn2_kernel, (size_t)4 * max_len * sizeof(int)));
    SB_CUDA_OK(launch_k(decode_self_attn2_kernel, dim3(rows, (heads + 3) / 4), dim3(128), (size_t)4 * max_len * sizeof(int),
                         (cudaStream_t)stream, qkv_partials, (int)splits, (long long)slice_rows, qkv_bias, (elem_t*)kcache, (elem_t*)vcache,
                         (const int*)anc, (int)anc_ld, (const int*)step_ptr, (int)max_len, (elem_t*)out, (int)rows, (int)heads));
    count_launch();
    return SB_OK;
  }
  size_t smem = (size_t)8 * max_len * sizeof(float);
  SB_REQUIRE(smem <= 48 * 1024, SB_ENOSUP, "sb_decode_self_attn: max_len %d too large", max_len);
  if (max_len > 1024) SB_CUDA_OK(allow_dynamic_smem(decode_self_attn_kernel, smem));
  SB_CUDA_OK(launch_k(decode_self_attn_kernel, dim3(rows, (heads + 3) / 4), dim3(128), smem, (cudaStream_t)stream,
                       (const elem_t*)qkv, qkv_partials, (int)splits, (long long)slice_rows, qkv_bias, (elem_t*)kcache,
                       (elem_t*)vcache, (const int*)anc, (int)anc_ld, (const int*)step_ptr,
                       (int)max_len, (elem_t*)out, (int)rows, (int)heads));
  count_launch();
  return SB_OK;
}

extern "C" int sb_decode_cross_attn(const void* q, const float* q_partials, int32_t splits, int64_t slice_rows,
                                    const float* q_bias, const void* k, const void* v, int64_t kv_ld, const int32_t* enc_lens,
                                    int32_t s_enc, void* out, int32_t rows, int32_t beam, int32_t heads, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE((q || (q_partials && q_bias && splits >= 1)) && k && v && out && rows > 0 && heads > 0 && s_enc > 0 && beam > 0,
             SB_EINVAL, "sb_decode_cross_attn: bad args");
  static int shared_ok = -1;
  if (shared_ok < 0) { const char* e = getenv("SB_CROSS_ATTN_SHARED"); shared_ok = (e == nullptr || atoi(e) != 0) ? 1 : 0; }
  if (shared_ok && q_partials != nullptr && beam <= 8 && rows % beam == 0) {
    const int nw = beam <= 4 ? 4 : 8;
    const size_t sm = (size_t)2 * s_enc * HD * sizeof(elem_t) + (size_t)nw * s_enc * sizeof(float) + (size_t)nw * HD * sizeof(elem_t);
    if (sm <= 200 * 1024) {
      static size_t configured = 0;
      if (sm > 48 * 1024 && sm > configured) {
        SB_CUDA_OK(cudaFuncSetAttribute(decode_cross_attn_shared_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        configured = sm;
      }
      SB_CUDA_OK(launch_k(decode_cross_attn_shared_kernel, dim3(rows / beam, heads), dim3(nw * 32), sm, (cudaStream_t)stream, q_partials,
                           (int)splits, (long long)slice_rows, q_bias, (const elem_t*)k, (const elem_t*)v, (long long)kv_ld,
                           (const int*)enc_lens, (int)s_enc, (elem_t*)out, (int)beam, (int)heads));
      count_launch();
      return SB_OK;
    }
  }
  size_t smem = (size_t)4 * s_enc * sizeof(float);
  SB_REQUIRE(smem <= 48 * 1024, SB_ENOSUP, "sb_decode_cross_attn: s_enc %d too large", s_enc);
  SB_CUDA_OK(launch_k(decode_cross_attn_kernel, dim3(rows, (heads + 3) / 4), dim3(128), smem, (cudaStream_t)stream,
                       (const elem_t*)q, q_partials, (int)splits, (long long)slice_rows, q_bias, (const elem_t*)k,
                       (const elem_t*)v, (long long)kv_ld, (const int*)enc_lens, (int)s_enc,
                       (elem_t*)out, (int)rows, (int)beam, (int)heads));
  count_launch();
  return SB_OK;
}

extern "C" int sb_logits_topk(const float* logits, int64_t ld, int32_t rows, int32_t vocab, int32_t pad_idx, int32_t eos_idx,
                              int32_t unk_idx, float unk_penalty, int32_t K, float* cand_val, int32_t* cand_idx,
                              float* eos_lprob, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(logits && cand_val && cand_idx && eos_lprob && rows > 0 && vocab > 0, SB_EINVAL, "sb_logits_topk: bad args");
  SB_REQUIRE(K > 0 && K <= TK_MAX, SB_ENOSUP, "sb_logits_topk: K=%d unsupported (<= %d)", K, TK_MAX);
  SB_CUDA_OK(launch_k(logits_topk_kernel, dim3(rows), dim3(TK_THREADS), 0, (cudaStream_t)stream, logits, (long long)ld,
                       (int)vocab, (int)pad_idx, (int)eos_idx, (int)unk_idx, unk_penalty, (int)K, cand_val, (int*)cand_idx,
                       eos_lprob));
  count_launch();
  return SB_OK;
}

extern "C" int sb_logits_topk_tiles(const float* logits, int64_t ld, const float* tile_stats, int32_t rows, int32_t vocab,
                                    int32_t pad_idx, int32_t eos_idx, int32_t unk_idx, float unk_penalty, int32_t K, float* cand_val,
                                    int32_t* cand_idx, float* eos_lprob, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(logits && tile_stats && cand_val && cand_idx && eos_lprob && rows > 0 && vocab > 0, SB_EINVAL, "sb_logits_topk_tiles: bad args");
  SB_REQUIRE(K > 0 && K <= TK_MAX, SB_ENOSUP, "sb_logits_topk_tiles: K=%d unsupported (<= %d)", K, TK_MAX);
  SB_REQUIRE(ld % 4 == 0 && ((uintptr_t)logits % 16) == 0, SB_EINVAL, "sb_logits_topk_tiles: logits must be 16-byte aligned rows");
  const int n_tiles = (vocab + TKT_TILE - 1) / TKT_TILE;
  const size_t smem = (size_t)2 * n_tiles * sizeof(float);
  SB_REQUIRE(smem <= 40 * 1024, SB_ENOSUP, "sb_logits_topk_tiles: vocabulary of %d too large", vocab);
  SB_CUDA_OK(launch_k(logits_topk_tiles_kernel, dim3(rows), dim3(TKT_THREADS), smem, (cudaStream_t)stream, logits, (long long)ld,
                       (const float2*)tile_stats, (int)rows, (int)vocab, (int)pad_idx, (int)eos_idx, (int)unk_idx, unk_penalty, (int)K,
                       cand_val, (int*)cand_idx, eos_lprob));
  count_launch();
  return SB_OK;
}

extern "C" int sb_beam_step(const sb_beam_t* p, sb_stream_t stream) {
  using namespace sb;
  SB_REQUIRE(p && p->batch > 0 && p->beam > 0 && p->beam <= 16 && p->K > 0, SB_EINVAL, "sb_beam_step: bad args");
  SB_REQUIRE(p->step_ptr != nullptr, SB_EINVAL, "sb_beam_step: step_ptr is null");
  SB_CUDA_OK(launch_k(beam_step_kernel, dim3(p->batch), dim3(128), 0, (cudaStream_t)stream, *p));
  count_launch();
  return SB_OK;
}

extern "C" int sb_step_advance(int32_t* step_ptr, sb_stream_t stream) {
  SB_REQUIRE(step_ptr != nullptr, SB_EINVAL, "sb_step_advance: null");
  SB_CUDA_OK(sb::launch_k(sb::step_advance_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, (int*)step_ptr));
  sb::count_launch();
  return SB_OK;
}

extern "C" int sb_store_step(const void* h, void* hist, const int32_t* step_ptr, int64_t bytes_per_step, sb_stream_t stream) {
  SB_REQUIRE(h && hist && step_ptr && bytes_per_step > 0 && bytes_per_step % 16 == 0, SB_EINVAL, "sb_store_step: bad args");
  const long long n16 = bytes_per_step / 16;
  SB_CUDA_OK(sb::launch_k(sb::store_step_kernel, dim3((unsigned)((n16 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream,
                          (const uint4*)h, (uint4*)hist, (const int*)step_ptr, n16));
  sb::count_launch();
  return SB_OK;
}
