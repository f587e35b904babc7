// libhgb.so -- tensor-core flash attention for head_dim 8 (GPS global attention, hydragnn/globalAtt/gps.py:126-133,
// quirk Q1: the whole mini-batch is ONE dense sequence; C5: 8 heads x 8 dims over ~10^4 atoms).
//
// head_dim 8 is exactly one k-step of mma.sync.m16n8k8 (TF32 in, fp32 accumulate): a score block S[16 queries x 8 keys] is
// ONE instruction, P V another.  The softmax exponentials then bound the kernel (SFU), not the FMAs as in the SIMT kernels of
// hgb_attn.cu.  SPLIT = 3 runs every product as hi*hi + hi*lo + lo*hi of a TF32 split ("3xTF32": the dropped lo*lo term is
// 2^-22 |a||b|, below the fp32 rounding of the sums -- measured 1e-6 against fp64; C5 is an fp32 config, parity tolerance 1e-5;
// SPLIT = 4 adds lo*lo); SPLIT = 1 is plain TF32 for precision="bf16".  Scores are kept in base 2 (log2 e folded
// into the query scale) so that the exponentials are bare ex2.approx with no argument-scaling error.
//
// Fragment trick: the accumulator layout of S (thread holds keys 2t, 2t+1 of rows g, g+8) is fed back as the A operand of
// P V by declaring that k-slot t of the second product IS key 2t and k-slot t+4 IS key 2t+1 -- the B operand (V rows) is
// loaded in the same permuted order, so no shuffle is needed between the two products.  No [N, N] matrix reaches HBM; the
// forward saves one log-sum-exp per (query, head); the backward recomputes P twice (query-major for dQ, key-major for dK/dV).
#include "hgb_common.cuh"

namespace {

constexpr int D = 8;          // head dim
constexpr int CH = 64;        // keys (or queries) per shared-memory chunk
constexpr int RS = 12;        // row stride of a staged [CH][8] tile (floats): conflict-free for both fragment patterns
constexpr int WARPS = 4;
constexpr int ROWS = 16 * WARPS;
constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

__device__ __forceinline__ float tf32_hi(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ void mma8(float (&c)[4], const float (&a)[4], float b0, float b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}

// c = (c +) A B with A, B given as fp32 fragments (a_lo precomputed by the caller).  NOTE: the tensor core adds into its C operand
// with truncation, so a LONG chain of accumulating mma's drifts (measured: 3e-5 relative after 512 key blocks).  Long sums are
// therefore kept in registers with round-to-nearest FADDs: callers use mma_add, which runs the 1-4 products of ONE block through a
// zeroed temporary and adds it.
template <int SPLIT>
__device__ __forceinline__ void mma_acc(float (&c)[4], const float (&ahi)[4], const float (&alo)[4], float b0, float b1) {
  const float b0h = tf32_hi(b0), b1h = tf32_hi(b1);
  if (SPLIT >= 3) {
    const float b0l = tf32_hi(b0 - b0h), b1l = tf32_hi(b1 - b1h);
    if (SPLIT == 4) mma8(c, alo, b0l, b1l);      // the lo*lo term too: the product is then exact to ~2^-22 of |a||b|
    mma8(c, alo, b0h, b1h);
    mma8(c, ahi, b0l, b1l);
  }
  mma8(c, ahi, b0h, b1h);
}

template <int SPLIT>
__device__ __forceinline__ void mma_add(float (&c)[4], const float (&ahi)[4], const float (&alo)[4], float b0, float b1) {
  float d[4] = {0.f, 0.f, 0.f, 0.f};
  mma_acc<SPLIT>(d, ahi, alo, b0, b1);
  c[0] += d[0]; c[1] += d[1]; c[2] += d[2]; c[3] += d[3];
}

template <int SPLIT>
__device__ __forceinline__ void split4(const float (&x)[4], float (&hi)[4], float (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    hi[i] = tf32_hi(x[i]);
    lo[i] = SPLIT >= 3 ? tf32_hi(x[i] - hi[i]) : 0.f;
  }
}

// stage rows [r0, r0 + CH) of one 8-wide column block of a row-major matrix into shared memory (zero beyond n), already split into
// the TF32 hi part (dst) and the lo remainder (dst + TILE): the split is done once per element here instead of once per warp and use
constexpr int TILE = CH * RS;
template <int SPLIT>
__device__ __forceinline__ void stage(float* dst, const float* __restrict__ src, int ld, int col, int r0, int n, float mul) {
  for (int i = threadIdx.x; i < CH * 2; i += WARPS * 32) {
    const int r = i >> 1, half = i & 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + r < n) v = __ldg(reinterpret_cast<const float4*>(src + (int64_t)(r0 + r) * ld + col) + half);
    v.x *= mul; v.y *= mul; v.z *= mul; v.w *= mul;
    float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    *reinterpret_cast<float4*>(dst + r * RS + 4 * half) = h;
    if (SPLIT >= 3)
      *reinterpret_cast<float4*>(dst + TILE + r * RS + 4 * half) =
          make_float4(tf32_hi(v.x - h.x), tf32_hi(v.y - h.y), tf32_hi(v.z - h.z), tf32_hi(v.w - h.w));
  }
}

// c (+)= A B with the B fragment read from a pre-split shared-memory tile: element offsets o0 / o1 into the hi tile, lo tile at + TILE
template <int SPLIT>
__device__ __forceinline__ void mma_sm(float (&c)[4], const float (&ahi)[4], const float (&alo)[4], const float* tile, int o0, int o1) {
  const float b0h = tile[o0], b1h = tile[o1];
  if (SPLIT >= 3) {
    const float b0l = tile[TILE + o0], b1l = tile[TILE + o1];
    if (SPLIT == 4) mma8(c, alo, b0l, b1l);
    mma8(c, alo, b0h, b1h);
    mma8(c, ahi, b0l, b1l);
  }
  mma8(c, ahi, b0h, b1h);
}
template <int SPLIT>
__device__ __forceinline__ void mma_sm_add(float (&c)[4], const float (&ahi)[4], const float (&alo)[4], const float* tile, int o0, int o1) {
  float d[4] = {0.f, 0.f, 0.f, 0.f};
  mma_sm<SPLIT>(d, ahi, alo, tile, o0, o1);
  c[0] += d[0]; c[1] += d[1]; c[2] += d[2]; c[3] += d[3];
}

// A-operand fragment of rows [r0 + g, r0 + g + 8] of an 8-wide block, straight from global memory (zero beyond n)
__device__ __forceinline__ void load_a(float (&a)[4], const float* __restrict__ src, int ld, int col, int r0, int n, float mul) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ra = r0 + g, rb = r0 + g + 8;
  a[0] = ra < n ? src[(int64_t)ra * ld + col + t] * mul : 0.f;
  a[1] = rb < n ? src[(int64_t)rb * ld + col + t] * mul : 0.f;
  a[2] = ra < n ? src[(int64_t)ra * ld + col + t + 4] * mul : 0.f;
  a[3] = rb < n ? src[(int64_t)rb * ld + col + t + 4] * mul : 0.f;
}

// ------------------------------------------------------------------------------------------------------------------
template <int SPLIT>
__global__ void __launch_bounds__(WARPS * 32) mha_tc_fwd_kernel(const float* __restrict__ qkv, int n, int f, float scale,
                                                                float* __restrict__ out, float* __restrict__ lse) {
  __shared__ __align__(16) float sk[2 * TILE], sv[2 * TILE];      // hi | lo
  const int h = blockIdx.y, nh = gridDim.y, f3 = 3 * f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = blockIdx.x * ROWS + warp * 16;
  float q[4], qh[4], ql[4];
  load_a(q, qkv, f3, h * D, r0, n, scale * LOG2E);        // scores in base 2
  split4<SPLIT>(q, qh, ql);
  float o[4] = {0.f, 0.f, 0.f, 0.f};
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int j0 = 0; j0 < n; j0 += CH) {
    __syncthreads();
    stage<SPLIT>(sk, qkv, f3, f + h * D, j0, n, 1.f);
    stage<SPLIT>(sv, qkv, f3, 2 * f + h * D, j0, n, 1.f);
    __syncthreads();
    float s[CH / 8][4];
#pragma unroll
    for (int kb = 0; kb < CH / 8; ++kb) {
      s[kb][0] = s[kb][1] = s[kb][2] = s[kb][3] = 0.f;
      mma_sm<SPLIT>(s[kb], qh, ql, sk, (kb * 8 + g) * RS + t, (kb * 8 + g) * RS + t + 4);
      const int key = j0 + kb * 8 + 2 * t;
      if (key >= n) s[kb][0] = s[kb][2] = -INFINITY;
      if (key + 1 >= n) s[kb][1] = s[kb][3] = -INFINITY;
    }
    float a0 = -INFINITY, a1 = -INFINITY;
#pragma unroll
    for (int kb = 0; kb < CH / 8; ++kb) {
      a0 = fmaxf(a0, fmaxf(s[kb][0], s[kb][1]));
      a1 = fmaxf(a1, fmaxf(s[kb][2], s[kb][3]));
    }
    a0 = fmaxf(a0, __shfl_xor_sync(0xffffffffu, a0, 1)); a0 = fmaxf(a0, __shfl_xor_sync(0xffffffffu, a0, 2));
    a1 = fmaxf(a1, __shfl_xor_sync(0xffffffffu, a1, 1)); a1 = fmaxf(a1, __shfl_xor_sync(0xffffffffu, a1, 2));
    const float n0 = fmaxf(m0, a0), n1 = fmaxf(m1, a1);          // finite: every chunk holds at least one valid key
    const float c0 = exp2f(m0 - n0), c1 = exp2f(m1 - n1);
    m0 = n0; m1 = n1;
    l0 *= c0; l1 *= c1;
    o[0] *= c0; o[1] *= c0; o[2] *= c1; o[3] *= c1;
#pragma unroll
    for (int kb = 0; kb < CH / 8; ++kb) {
      float p[4], ph[4], pl[4];
      // A-operand order of the permuted product: (row g, key 2t), (row g+8, key 2t), (row g, key 2t+1), (row g+8, key 2t+1)
      p[0] = exp2f(s[kb][0] - m0); p[1] = exp2f(s[kb][2] - m1); p[2] = exp2f(s[kb][1] - m0); p[3] = exp2f(s[kb][3] - m1);
      l0 += p[0] + p[2];
      l1 += p[1] + p[3];
      split4<SPLIT>(p, ph, pl);
      mma_sm_add<SPLIT>(o, ph, pl, sv, (kb * 8 + 2 * t) * RS + g, (kb * 8 + 2 * t + 1) * RS + g);
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const int ra = r0 + g, rb = r0 + g + 8;
  if (ra < n) {
    const float inv = 1.f / l0;
    *reinterpret_cast<float2*>(out + (int64_t)ra * f + h * D + 2 * t) = make_float2(o[0] * inv, o[1] * inv);
    if (t == 0) lse[(int64_t)ra * nh + h] = m0 * LN2 + logf(l0);      // natural-log lse (the contract of hgb_mha_fwd)
  }
  if (rb < n) {
    const float inv = 1.f / l1;
    *reinterpret_cast<float2*>(out + (int64_t)rb * f + h * D + 2 * t) = make_float2(o[2] * inv, o[3] * inv);
    if (t == 0) lse[(int64_t)rb * nh + h] = m1 * LN2 + logf(l1);
  }
}

// delta[i, h] = sum_d gout[i, h*8 + d] * out[i, h*8 + d]
__global__ void mha_tc_delta_kernel(const float* __restrict__ out, const float* __restrict__ gout, int n, int f, int nh,
                                    float* __restrict__ delta) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n * nh) return;
  const int64_t i = idx / nh;
  const int h = (int)(idx % nh);
  const float4* a = reinterpret_cast<const float4*>(out + i * f + h * D);
  const float4* b = reinterpret_cast<const float4*>(gout + i * f + h * D);
  const float4 a0 = __ldg(a), a1 = __ldg(a + 1), b0 = __ldg(b), b1 = __ldg(b + 1);
  delta[idx] = a0.x * b0.x + a0.y * b0.y + a0.z * b0.z + a0.w * b0.w + a1.x * b1.x + a1.y * b1.y + a1.z * b1.z + a1.w * b1.w;
}

// dQ: a warp owns 16 query rows and walks every key
template <int SPLIT>
__global__ void __launch_bounds__(WARPS * 32) mha_tc_bwd_q_kernel(const float* __restrict__ qkv, const float* __restrict__ lse,
                                                                  const float* __restrict__ delta, const float* __restrict__ gout,
                                                                  int n, int f, float scale, float* __restrict__ gqkv) {
  __shared__ __align__(16) float sk[2 * TILE], sv[2 * TILE];
  const int h = blockIdx.y, nh = gridDim.y, f3 = 3 * f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = blockIdx.x * ROWS + warp * 16;
  const int ra = r0 + g, rb = r0 + g + 8;
  float q[4], qh[4], ql[4], go[4], goh[4], gol[4];
  load_a(q, qkv, f3, h * D, r0, n, scale * LOG2E);
  split4<SPLIT>(q, qh, ql);
  load_a(go, gout, f, h * D, r0, n, 1.f);
  split4<SPLIT>(go, goh, gol);
  const float ls0 = ra < n ? lse[(int64_t)ra * nh + h] * LOG2E : 0.f, ls1 = rb < n ? lse[(int64_t)rb * nh + h] * LOG2E : 0.f;
  const float dl0 = ra < n ? delta[(int64_t)ra * nh + h] : 0.f, dl1 = rb < n ? delta[(int64_t)rb * nh + h] : 0.f;
  float dq[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j0 = 0; j0 < n; j0 += CH) {
    __syncthreads();
    stage<SPLIT>(sk, qkv, f3, f + h * D, j0, n, 1.f);
    stage<SPLIT>(sv, qkv, f3, 2 * f + h * D, j0, n, 1.f);
    __syncthreads();
#pragma unroll
    for (int kb = 0; kb < CH / 8; ++kb) {
      float s[4] = {0.f, 0.f, 0.f, 0.f}, dp[4] = {0.f, 0.f, 0.f, 0.f};
      mma_sm<SPLIT>(s, qh, ql, sk, (kb * 8 + g) * RS + t, (kb * 8 + g) * RS + t + 4);
      mma_sm<SPLIT>(dp, goh, gol, sv, (kb * 8 + g) * RS + t, (kb * 8 + g) * RS + t + 4);
      const int key = j0 + kb * 8 + 2 * t;
      const bool v0 = key < n, v1 = key + 1 < n;
      float ds[4], dsh[4], dsl[4];
      // permuted A order: (row g, key 2t), (row g+8, key 2t), (row g, key 2t+1), (row g+8, key 2t+1)
      ds[0] = v0 ? exp2f(s[0] - ls0) * (dp[0] - dl0) : 0.f;
      ds[1] = v0 ? exp2f(s[2] - ls1) * (dp[2] - dl1) : 0.f;
      ds[2] = v1 ? exp2f(s[1] - ls0) * (dp[1] - dl0) : 0.f;
      ds[3] = v1 ? exp2f(s[3] - ls1) * (dp[3] - dl1) : 0.f;
      split4<SPLIT>(ds, dsh, dsl);
      mma_sm_add<SPLIT>(dq, dsh, dsl, sk, (kb * 8 + 2 * t) * RS + g, (kb * 8 + 2 * t + 1) * RS + g);
    }
  }
  if (ra < n) *reinterpret_cast<float2*>(gqkv + (int64_t)ra * f3 + h * D + 2 * t) = make_float2(dq[0] * scale, dq[1] * scale);
  if (rb < n) *reinterpret_cast<float2*>(gqkv + (int64_t)rb * f3 + h * D + 2 * t) = make_float2(dq[2] * scale, dq[3] * scale);
}

// dK, dV: a warp owns 16 key rows and walks every query.  Q is staged with the forward's base-2 scale, so S^T is built from the
// same split operands as the forward's S and P = exp2(s - lse log2 e) matches the forward's p to a few ulp of the score; Q
// staged with 1/sqrt(d) alone would round differently and, at the TF32 split, shift p by ~2^-11 |s| (15 % at |s| = 600).
// dK = dS^T Q / sqrt(d) is then the accumulated dS^T (Q scale log2 e) times ln 2.
template <int SPLIT>
__global__ void __launch_bounds__(WARPS * 32) mha_tc_bwd_kv_kernel(const float* __restrict__ qkv, const float* __restrict__ lse,
                                                                   const float* __restrict__ delta, const float* __restrict__ gout,
                                                                   int n, int f, float scale, float* __restrict__ gqkv) {
  __shared__ __align__(16) float sq[2 * TILE], sg[2 * TILE];
  __shared__ float sl[CH], sd[CH];
  const int h = blockIdx.y, nh = gridDim.y, f3 = 3 * f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = blockIdx.x * ROWS + warp * 16;
  const int ra = r0 + g, rb = r0 + g + 8;
  float k[4], kh[4], kl[4], v[4], vh[4], vl[4];
  load_a(k, qkv, f3, f + h * D, r0, n, 1.f);
  split4<SPLIT>(k, kh, kl);
  load_a(v, qkv, f3, 2 * f + h * D, r0, n, 1.f);
  split4<SPLIT>(v, vh, vl);
  float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i0 = 0; i0 < n; i0 += CH) {
    __syncthreads();
    stage<SPLIT>(sq, qkv, f3, h * D, i0, n, scale * LOG2E);
    stage<SPLIT>(sg, gout, f, h * D, i0, n, 1.f);
    for (int i = threadIdx.x; i < CH; i += WARPS * 32) {
      sl[i] = i0 + i < n ? lse[(int64_t)(i0 + i) * nh + h] * LOG2E : 0.f;
      sd[i] = i0 + i < n ? delta[(int64_t)(i0 + i) * nh + h] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int qb = 0; qb < CH / 8; ++qb) {
      float st[4] = {0.f, 0.f, 0.f, 0.f}, dpt[4] = {0.f, 0.f, 0.f, 0.f};      // S^T (base 2), dP^T: rows = keys, cols = queries
      mma_sm<SPLIT>(st, kh, kl, sq, (qb * 8 + g) * RS + t, (qb * 8 + g) * RS + t + 4);
      mma_sm<SPLIT>(dpt, vh, vl, sg, (qb * 8 + g) * RS + t, (qb * 8 + g) * RS + t + 4);
      const int qi = qb * 8 + 2 * t;
      const bool v0 = i0 + qi < n, v1 = i0 + qi + 1 < n;
      const float lq0 = sl[qi], lq1 = sl[qi + 1], dq0 = sd[qi], dq1 = sd[qi + 1];
      float p[4], ds[4], ph[4], pl[4], dsh[4], dsl[4];
      // permuted A order: (key g, query 2t), (key g+8, query 2t), (key g, query 2t+1), (key g+8, query 2t+1)
      p[0] = v0 ? exp2f(st[0] - lq0) : 0.f; p[1] = v0 ? exp2f(st[2] - lq0) : 0.f;
      p[2] = v1 ? exp2f(st[1] - lq1) : 0.f; p[3] = v1 ? exp2f(st[3] - lq1) : 0.f;
      ds[0] = p[0] * (dpt[0] - dq0); ds[1] = p[1] * (dpt[2] - dq0);
      ds[2] = p[2] * (dpt[1] - dq1); ds[3] = p[3] * (dpt[3] - dq1);
      split4<SPLIT>(p, ph, pl);
      split4<SPLIT>(ds, dsh, dsl);
      mma_sm_add<SPLIT>(dv, ph, pl, sg, (qb * 8 + 2 * t) * RS + g, (qb * 8 + 2 * t + 1) * RS + g);
      mma_sm_add<SPLIT>(dk, dsh, dsl, sq, (qb * 8 + 2 * t) * RS + g, (qb * 8 + 2 * t + 1) * RS + g);
    }
  }
  if (ra < n) {
    *reinterpret_cast<float2*>(gqkv + (int64_t)ra * f3 + f + h * D + 2 * t) = make_float2(dk[0] * LN2, dk[1] * LN2);
    *reinterpret_cast<float2*>(gqkv + (int64_t)ra * f3 + 2 * f + h * D + 2 * t) = make_float2(dv[0], dv[1]);
  }
  if (rb < n) {
    *reinterpret_cast<float2*>(gqkv + (int64_t)rb * f3 + f + h * D + 2 * t) = make_float2(dk[2] * LN2, dk[3] * LN2);
    *reinterpret_cast<float2*>(gqkv + (int64_t)rb * f3 + 2 * f + h * D + 2 * t) = make_float2(dv[2], dv[3]);
  }
}

}  // namespace

extern "C" int32_t hgb_mha_tc_supported(int32_t f, int32_t heads) {
  return (heads > 0 && f % heads == 0 && f / heads == D && f % 4 == 0) ? 1 : 0;
}

static bool aligned(const void* p, uintptr_t bytes) { return ((uintptr_t)p & (bytes - 1)) == 0; }

// Sizes are checked first, pointers only when there is a row: the data pointer of an empty tensor may be NULL.  Rows are read
// with float4 loads (stage, delta) and written with float2 stores; the row strides 3f and f are multiples of 4 floats, so the
// base pointers decide the alignment.
extern "C" int hgb_mha_tc_fwd(const float* qkv, int32_t n, int32_t f, int32_t heads, int32_t exact, float* out, float* lse,
                              hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && hgb_mha_tc_supported(f, heads), "mha_tc_fwd: bad sizes (n %d, f %d, heads %d; head_dim must be 8)",
              n, f, heads);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(qkv && out && lse, "mha_tc_fwd: NULL pointer");
  HGB_REQUIRE(aligned(qkv, 16) && aligned(out, 8), "mha_tc_fwd: qkv must be 16-byte and out 8-byte aligned");
  const float scale = 1.f / sqrtf((float)D);
  dim3 grid((n + ROWS - 1) / ROWS, heads);
  cudaStream_t st = (cudaStream_t)stream;
  if (exact) mha_tc_fwd_kernel<3><<<grid, WARPS * 32, 0, st>>>(qkv, n, f, scale, out, lse);
  else mha_tc_fwd_kernel<1><<<grid, WARPS * 32, 0, st>>>(qkv, n, f, scale, out, lse);
  HGB_LAUNCH_CHECK("mha_tc_fwd");
  return HGB_OK;
}

extern "C" int hgb_mha_tc_bwd(const float* qkv, const float* out, const float* lse, const float* gout, int32_t n, int32_t f,
                              int32_t heads, int32_t exact, float* delta_ws, float* gqkv, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && hgb_mha_tc_supported(f, heads), "mha_tc_bwd: bad sizes (n %d, f %d, heads %d; head_dim must be 8)",
              n, f, heads);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(qkv && out && lse && gout && gqkv && delta_ws, "mha_tc_bwd: NULL pointer");
  HGB_REQUIRE(aligned(qkv, 16) && aligned(out, 16) && aligned(gout, 16) && aligned(gqkv, 8),
              "mha_tc_bwd: qkv, out and gout must be 16-byte and gqkv 8-byte aligned");
  const float scale = 1.f / sqrtf((float)D);
  dim3 grid((n + ROWS - 1) / ROWS, heads);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cnt = (int64_t)n * heads;
  mha_tc_delta_kernel<<<(int)((cnt + 255) / 256), 256, 0, st>>>(out, gout, n, f, heads, delta_ws);
  HGB_LAUNCH_CHECK("mha_tc_delta");
  if (exact) {
    mha_tc_bwd_q_kernel<3><<<grid, WARPS * 32, 0, st>>>(qkv, lse, delta_ws, gout, n, f, scale, gqkv);
    HGB_LAUNCH_CHECK("mha_tc_bwd_q");
    mha_tc_bwd_kv_kernel<3><<<grid, WARPS * 32, 0, st>>>(qkv, lse, delta_ws, gout, n, f, scale, gqkv);
  } else {
    mha_tc_bwd_q_kernel<1><<<grid, WARPS * 32, 0, st>>>(qkv, lse, delta_ws, gout, n, f, scale, gqkv);
    HGB_LAUNCH_CHECK("mha_tc_bwd_q");
    mha_tc_bwd_kv_kernel<1><<<grid, WARPS * 32, 0, st>>>(qkv, lse, delta_ws, gout, n, f, scale, gqkv);
  }
  HGB_LAUNCH_CHECK("mha_tc_bwd_kv");
  return HGB_OK;
}
