// libhgb.so -- dense multi-head self-attention over one sequence (GPS global attention,
// hydragnn/globalAtt/gps.py:126-133 with quirk Q1: the whole mini-batch is ONE sequence).
//
// Head dims on this path are tiny (hidden 64 / 8 heads = 8), so attention here is exp/FMA-bound SIMT work, not a
// tensor-core GEMM: four lanes share one (query, head) row (each walks every 4th key, partial online-softmax states
// combined with shuffles), q, the output accumulator and the softmax state live in registers; K/V tiles of the same head are staged in shared memory and broadcast to the block.
// No [N,N] matrix ever reaches HBM (flash-style), forward saves only the log-sum-exp per (query, head).
#include "hgb_common.cuh"

#define ATT_TK 64    // keys per shared-memory tile
#define ATT_TQ 128   // threads per block
#define ATT_KS 4     // lanes that share one (row, head): each walks every 4th key of a tile; combined with shuffles.
#define ATT_QPB (ATT_TQ / ATT_KS)   // rows per block.  (Sequences here are a few thousand atoms: one thread per row would
                                    // leave most of the 132 SMs idle and serialise the whole key loop in one dependency chain.)

// qkv [n, 3f]: row = [ q (f) | k (f) | v (f) ], head h owns columns h*D .. h*D+D-1 of each part
template <int D>
__global__ void __launch_bounds__(ATT_TQ) mha_fwd_kernel(const float* __restrict__ qkv, int n, int f, float scale,
                                                         float* __restrict__ out, float* __restrict__ lse) {
  __shared__ float sk[ATT_TK][D], sv[ATT_TK][D];
  const int h = blockIdx.y, nh = gridDim.y;
  const int ks = threadIdx.x & (ATT_KS - 1);
  const int i = blockIdx.x * ATT_QPB + (threadIdx.x >> 2);
  const int f3 = 3 * f;
  float q[D], o[D];
  float m = -INFINITY, l = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) { q[d] = i < n ? qkv[(int64_t)i * f3 + h * D + d] * scale : 0.f; o[d] = 0.f; }
  for (int j0 = 0; j0 < n; j0 += ATT_TK) {
    __syncthreads();
    for (int t = threadIdx.x; t < ATT_TK * D; t += ATT_TQ) {
      const int jj = t / D, d = t % D;
      const int j = j0 + jj;
      sk[jj][d] = j < n ? qkv[(int64_t)j * f3 + f + h * D + d] : 0.f;
      sv[jj][d] = j < n ? qkv[(int64_t)j * f3 + 2 * f + h * D + d] : 0.f;
    }
    __syncthreads();
    const int jn = min(ATT_TK, n - j0);
    for (int jj = ks; jj < jn; jj += ATT_KS) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) s = fmaf(q[d], sk[jj][d], s);
      if (s > m) {                       // rescale only when the running maximum moves
        const float c = __expf(m - s);
        l *= c;
#pragma unroll
        for (int d = 0; d < D; ++d) o[d] *= c;
        m = s;
      }
      const float p = __expf(s - m);
      l += p;
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] = fmaf(p, sv[jj][d], o[d]);
    }
  }
  // combine the ATT_KS partial softmax states of this row
#pragma unroll
  for (int off = 1; off < ATT_KS; off <<= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
    const float mn = fmaxf(m, m2);
    const float c1 = m == -INFINITY ? 0.f : __expf(m - mn), c2 = m2 == -INFINITY ? 0.f : __expf(m2 - mn);
    l = l * c1 + l2 * c2;
#pragma unroll
    for (int d = 0; d < D; ++d) o[d] = o[d] * c1 + __shfl_xor_sync(0xffffffffu, o[d], off) * c2;
    m = mn;
  }
  if (i < n && ks == 0) {
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < D; ++d) out[(int64_t)i * f + h * D + d] = o[d] * inv;
    lse[(int64_t)i * nh + h] = m + __logf(l);
  }
}

// dq: ATT_KS lanes per (query, head).  delta_i = dO_i . O_i
template <int D>
__global__ void __launch_bounds__(ATT_TQ) mha_bwd_q_kernel(const float* __restrict__ qkv, const float* __restrict__ out,
                                                           const float* __restrict__ lse, const float* __restrict__ gout, int n, int f,
                                                           float scale, float* __restrict__ gqkv) {
  __shared__ float sk[ATT_TK][D], sv[ATT_TK][D];
  const int h = blockIdx.y, nh = gridDim.y;
  const int ks = threadIdx.x & (ATT_KS - 1);
  const int i = blockIdx.x * ATT_QPB + (threadIdx.x >> 2);
  const int f3 = 3 * f;
  float q[D], go[D], dq[D];
  float delta = 0.f, li = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    q[d] = i < n ? qkv[(int64_t)i * f3 + h * D + d] * scale : 0.f;
    go[d] = i < n ? gout[(int64_t)i * f + h * D + d] : 0.f;
    delta += go[d] * (i < n ? out[(int64_t)i * f + h * D + d] : 0.f);
    dq[d] = 0.f;
  }
  if (i < n) li = lse[(int64_t)i * nh + h];
  for (int j0 = 0; j0 < n; j0 += ATT_TK) {
    __syncthreads();
    for (int t = threadIdx.x; t < ATT_TK * D; t += ATT_TQ) {
      const int jj = t / D, d = t % D;
      const int j = j0 + jj;
      sk[jj][d] = j < n ? qkv[(int64_t)j * f3 + f + h * D + d] : 0.f;
      sv[jj][d] = j < n ? qkv[(int64_t)j * f3 + 2 * f + h * D + d] : 0.f;
    }
    __syncthreads();
    const int jn = min(ATT_TK, n - j0);
    for (int jj = ks; jj < jn; jj += ATT_KS) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) { s = fmaf(q[d], sk[jj][d], s); dp = fmaf(go[d], sv[jj][d], dp); }
      const float ds = __expf(s - li) * (dp - delta);
#pragma unroll
      for (int d = 0; d < D; ++d) dq[d] = fmaf(ds, sk[jj][d], dq[d]);
    }
  }
#pragma unroll
  for (int off = 1; off < ATT_KS; off <<= 1)
#pragma unroll
    for (int d = 0; d < D; ++d) dq[d] += __shfl_xor_sync(0xffffffffu, dq[d], off);
  if (i < n && ks == 0) {
#pragma unroll
    for (int d = 0; d < D; ++d) gqkv[(int64_t)i * f3 + h * D + d] = dq[d] * scale;
  }
}

// dk, dv: ATT_KS lanes per (key, head); tiles of (q, dO, lse, delta) staged in shared memory
template <int D>
__global__ void __launch_bounds__(ATT_TQ) mha_bwd_kv_kernel(const float* __restrict__ qkv, const float* __restrict__ out,
                                                            const float* __restrict__ lse, const float* __restrict__ gout, int n, int f,
                                                            float scale, float* __restrict__ gqkv) {
  __shared__ float sq[ATT_TK][D], sg[ATT_TK][D], sl[ATT_TK], sd[ATT_TK];
  const int h = blockIdx.y, nh = gridDim.y;
  const int ks = threadIdx.x & (ATT_KS - 1);
  const int j = blockIdx.x * ATT_QPB + (threadIdx.x >> 2);
  const int f3 = 3 * f;
  float k[D], v[D], dk[D], dv[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    k[d] = j < n ? qkv[(int64_t)j * f3 + f + h * D + d] : 0.f;
    v[d] = j < n ? qkv[(int64_t)j * f3 + 2 * f + h * D + d] : 0.f;
    dk[d] = 0.f; dv[d] = 0.f;
  }
  for (int i0 = 0; i0 < n; i0 += ATT_TK) {
    __syncthreads();
    for (int t = threadIdx.x; t < ATT_TK * D; t += ATT_TQ) {
      const int ii = t / D, d = t % D;
      const int i = i0 + ii;
      sq[ii][d] = i < n ? qkv[(int64_t)i * f3 + h * D + d] * scale : 0.f;
      sg[ii][d] = i < n ? gout[(int64_t)i * f + h * D + d] : 0.f;
    }
    for (int ii = threadIdx.x; ii < ATT_TK; ii += ATT_TQ) {
      const int i = i0 + ii;
      float dl = 0.f;
      if (i < n)
        for (int d = 0; d < D; ++d) dl += gout[(int64_t)i * f + h * D + d] * out[(int64_t)i * f + h * D + d];
      sd[ii] = dl;
      sl[ii] = i < n ? lse[(int64_t)i * nh + h] : INFINITY;   // exp(s - inf) = 0 for padded queries
    }
    __syncthreads();
    for (int ii = ks; ii < ATT_TK; ii += ATT_KS) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) { s = fmaf(sq[ii][d], k[d], s); dp = fmaf(sg[ii][d], v[d], dp); }
      const float p = __expf(s - sl[ii]);
      const float ds = p * (dp - sd[ii]);
#pragma unroll
      for (int d = 0; d < D; ++d) { dv[d] = fmaf(p, sg[ii][d], dv[d]); dk[d] = fmaf(ds, sq[ii][d], dk[d]); }
    }
  }
#pragma unroll
  for (int off = 1; off < ATT_KS; off <<= 1)
#pragma unroll
    for (int d = 0; d < D; ++d) {
      dk[d] += __shfl_xor_sync(0xffffffffu, dk[d], off);
      dv[d] += __shfl_xor_sync(0xffffffffu, dv[d], off);
    }
  if (j < n && ks == 0) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      gqkv[(int64_t)j * f3 + f + h * D + d] = dk[d];          // sq already carries the 1/sqrt(D) scale
      gqkv[(int64_t)j * f3 + 2 * f + h * D + d] = dv[d];
    }
  }
}

#define ATT_DISPATCH(KERNEL, ...)                                                   \
  switch (d) {                                                                      \
    case 1: KERNEL<1><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;                 \
    case 2: KERNEL<2><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;                 \
    case 4: KERNEL<4><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;                 \
    case 8: KERNEL<8><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;                 \
    case 16: KERNEL<16><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;               \
    case 32: KERNEL<32><<<grid, ATT_TQ, 0, st>>>(__VA_ARGS__); break;               \
    default: hgb_set_error("mha: head_dim %d not supported (1,2,4,8,16,32)", d); return HGB_EINVAL; \
  }

static bool mha_head_dim_ok(int d) { return d == 1 || d == 2 || d == 4 || d == 8 || d == 16 || d == 32; }

// Sizes are checked first, pointers only when there is a row: the data pointer of an empty tensor may be NULL.
extern "C" int hgb_mha_fwd(const float* qkv, int32_t n, int32_t f, int32_t heads, float* out, float* lse, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && heads > 0 && f % heads == 0 && mha_head_dim_ok(f / heads),
              "mha_fwd: bad sizes (n %d, f %d, heads %d; head_dim must be 1, 2, 4, 8, 16 or 32)", n, f, heads);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(qkv && out && lse, "mha_fwd: NULL pointer");
  const int d = f / heads;
  const float scale = 1.f / sqrtf((float)d);
  dim3 grid((n + ATT_QPB - 1) / ATT_QPB, heads);
  cudaStream_t st = (cudaStream_t)stream;
  ATT_DISPATCH(mha_fwd_kernel, qkv, n, f, scale, out, lse)
  HGB_LAUNCH_CHECK("mha_fwd");
  return HGB_OK;
}

extern "C" int hgb_mha_bwd(const float* qkv, const float* out, const float* lse, const float* gout, int32_t n, int32_t f,
                           int32_t heads, float* gqkv, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && heads > 0 && f % heads == 0 && mha_head_dim_ok(f / heads),
              "mha_bwd: bad sizes (n %d, f %d, heads %d; head_dim must be 1, 2, 4, 8, 16 or 32)", n, f, heads);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(qkv && out && lse && gout && gqkv, "mha_bwd: NULL pointer");
  const int d = f / heads;
  const float scale = 1.f / sqrtf((float)d);
  dim3 grid((n + ATT_QPB - 1) / ATT_QPB, heads);
  cudaStream_t st = (cudaStream_t)stream;
  ATT_DISPATCH(mha_bwd_q_kernel, qkv, out, lse, gout, n, f, scale, gqkv)
  HGB_LAUNCH_CHECK("mha_bwd_q");
  ATT_DISPATCH(mha_bwd_kv_kernel, qkv, out, lse, gout, n, f, scale, gqkv)
  HGB_LAUNCH_CHECK("mha_bwd_kv");
  return HGB_OK;
}
