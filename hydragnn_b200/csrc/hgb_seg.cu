// libhgb.so -- row gather, atomics-free segmented sum over a CSR view, graph pooling.
//
// All three are HBM-bound.  Thread mapping: a group of LANES = min(32, pow2 >= C/4) threads owns one
// output row and walks the row with float4 loads (16 B per thread, consecutive lanes -> consecutive
// 16 B, i.e. fully coalesced 128 B lines when C*4 >= 128), so narrow rows (C = 1..16) do not waste
// a whole warp per row.  Summation order inside a segment is the CSR order: deterministic.
#include "hgb_common.cuh"

template <int VEC>
struct VecT;
template <>
struct VecT<4> { using type = float4; };
template <>
struct VecT<1> { using type = float; };

__device__ __forceinline__ void vadd(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void vadd(float& a, const float& b) { a += b; }
__device__ __forceinline__ void vzero(float4& a) { a = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void vzero(float& a) { a = 0.f; }

// picks the sub-warp group width for rows of `cv` vector elements
static inline int group_lanes(int cv) {
  int l = 1;
  while (l < cv && l < 32) l <<= 1;
  return l;
}

// ---- gather -----------------------------------------------------------------------------------
template <int VEC>
__global__ void gather_rows_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t e, int cv,
                                   int lanes, float* __restrict__ out) {
  using V = typename VecT<VEC>::type;
  const int gpb = blockDim.x / lanes;
  const int sub = threadIdx.x % lanes;
  for (int64_t row = (int64_t)blockIdx.x * gpb + threadIdx.x / lanes; row < e; row += (int64_t)gridDim.x * gpb) {
    const V* src = reinterpret_cast<const V*>(x) + (int64_t)idx[row] * cv;
    V* dst = reinterpret_cast<V*>(out) + row * cv;
    for (int c = sub; c < cv; c += lanes) dst[c] = __ldg(src + c);
  }
}

extern "C" int hgb_gather_rows(const float* x, const int32_t* idx, int64_t e, int32_t c, float* out, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && c > 0 && x && idx && out, "gather_rows: bad arguments");
  if (e == 0) return HGB_OK;
  const bool v4 = (c % 4 == 0) && ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
  const int cv = v4 ? c / 4 : c;
  const int lanes = group_lanes(cv);
  const int gpb = 256 / lanes;
  const int grid = hgb_grid_for(e, gpb);
  if (v4) gather_rows_kernel<4><<<grid, 256, 0, (cudaStream_t)stream>>>(x, idx, e, cv, lanes, out);
  else gather_rows_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(x, idx, e, cv, lanes, out);
  HGB_LAUNCH_CHECK("gather_rows");
  return HGB_OK;
}

// ---- segmented sum ------------------------------------------------------------------------------
template <int VEC>
__global__ void segment_sum_kernel(const float* __restrict__ m, const int32_t* __restrict__ rowptr,
                                   const int32_t* __restrict__ perm, int n, int cv, int lanes, float* __restrict__ out,
                                   int ldo_v /* output row stride in V units */) {
  using V = typename VecT<VEC>::type;
  const int gpb = blockDim.x / lanes;
  const int sub = threadIdx.x % lanes;
  for (int row = blockIdx.x * gpb + threadIdx.x / lanes; row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    for (int c = sub; c < cv; c += lanes) {
      V acc;
      vzero(acc);
      int p = lo;
      // two independent loads in flight per lane
      for (; p + 1 < hi; p += 2) {
        const int e0 = perm ? perm[p] : p, e1 = perm ? perm[p + 1] : p + 1;
        V a = __ldg(reinterpret_cast<const V*>(m) + (int64_t)e0 * cv + c);
        V b = __ldg(reinterpret_cast<const V*>(m) + (int64_t)e1 * cv + c);
        vadd(acc, a);
        vadd(acc, b);
      }
      if (p < hi) {
        const int e0 = perm ? perm[p] : p;
        vadd(acc, __ldg(reinterpret_cast<const V*>(m) + (int64_t)e0 * cv + c));
      }
      reinterpret_cast<V*>(out)[(int64_t)row * ldo_v + c] = acc;
    }
  }
}

extern "C" int hgb_segment_sum_strided(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c,
                                       float* out, int32_t ldo, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && c > 0 && rowptr && out && ldo >= c, "segment_sum: bad arguments");
  if (n == 0) return HGB_OK;
  const bool v4 = (c % 4 == 0) && (ldo % 4 == 0) && ((uintptr_t)m % 16 == 0) && ((uintptr_t)out % 16 == 0);
  const int cv = v4 ? c / 4 : c;
  const int lanes = group_lanes(cv);
  const int gpb = 256 / lanes;
  const int grid = hgb_grid_for(n, gpb);
  if (v4) segment_sum_kernel<4><<<grid, 256, 0, (cudaStream_t)stream>>>(m, rowptr, perm, n, cv, lanes, out, ldo / 4);
  else segment_sum_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(m, rowptr, perm, n, cv, lanes, out, ldo);
  HGB_LAUNCH_CHECK("segment_sum");
  return HGB_OK;
}

extern "C" int hgb_segment_sum(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c,
                               float* out, hgb_stream_t stream) {
  return hgb_segment_sum_strided(m, rowptr, perm, n, c, out, c, stream);
}

// ---- graph pooling (batch is sorted: a graph is a contiguous run of rows) -------------------------
__global__ void pool_fwd_kernel(const float* __restrict__ x, const int32_t* __restrict__ gptr, int g, int c, int mode,
                                float* __restrict__ out, int32_t* __restrict__ argmax) {
  // one warp per graph, lanes stride over channels (rows of a graph are contiguous -> coalesced)
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (int k = blockIdx.x * wpb + (threadIdx.x >> 5); k < g; k += gridDim.x * wpb) {
    const int lo = gptr[k], hi = gptr[k + 1];
    for (int ch = lane; ch < c; ch += 32) {
      if (mode == HGB_POOL_MAX) {
        float best = -INFINITY;
        int arg = -1;
        for (int i = lo; i < hi; ++i) {
          float v = x[(int64_t)i * c + ch];
          if (v > best || arg < 0) { if (v > best || arg < 0) { best = v; arg = i; } }
        }
        out[(int64_t)k * c + ch] = arg < 0 ? 0.f : best;
        if (argmax) argmax[(int64_t)k * c + ch] = arg;
      } else {
        float acc = 0.f;
        for (int i = lo; i < hi; ++i) acc += x[(int64_t)i * c + ch];
        if (mode == HGB_POOL_MEAN) acc /= (float)max(hi - lo, 1);
        out[(int64_t)k * c + ch] = acc;
      }
    }
  }
}

// one warp zeroes gx rows [lo, hi)
__device__ __forceinline__ void pool_zero_rows(float* __restrict__ gx, int lo, int hi, int c, int lane) {
  for (int64_t t = lane; t < (int64_t)(hi - lo) * c; t += 32) gx[(int64_t)lo * c + t] = 0.f;
}

// relu_y (add / mean, may be NULL): the pooled rows were ReLU outputs, gx is masked by hgb_relu_select on the way out.
// Rows outside [gptr[0], gptr[g]) belong to no graph: the warps of the first and last graph zero them.
__global__ void pool_bwd_kernel(const float* __restrict__ gout, const int32_t* __restrict__ gptr, const int32_t* __restrict__ argmax,
                                const float* __restrict__ relu_y, int n, int g, int c, int mode, float* __restrict__ gx) {
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  if (g == 0 && blockIdx.x == 0 && threadIdx.x < 32) pool_zero_rows(gx, 0, n, c, lane);
  for (int k = blockIdx.x * wpb + (threadIdx.x >> 5); k < g; k += gridDim.x * wpb) {
    const int lo = gptr[k], hi = gptr[k + 1];
    if (k == 0) pool_zero_rows(gx, 0, lo, c, lane);
    if (k == g - 1) pool_zero_rows(gx, hi, n, c, lane);
    const float scale = mode == HGB_POOL_MEAN ? 1.f / (float)max(hi - lo, 1) : 1.f;
    for (int ch = lane; ch < c; ch += 32) {
      const float gv = gout[(int64_t)k * c + ch] * scale;
      if (mode == HGB_POOL_MAX) {
        const int arg = argmax[(int64_t)k * c + ch];
        for (int i = lo; i < hi; ++i) gx[(int64_t)i * c + ch] = (i == arg) ? gv : 0.f;
      } else if (relu_y) {
        for (int i = lo; i < hi; ++i) gx[(int64_t)i * c + ch] = hgb_relu_select(gv, relu_y[(int64_t)i * c + ch]);
      } else {
        for (int i = lo; i < hi; ++i) gx[(int64_t)i * c + ch] = gv;
      }
    }
  }
}

extern "C" int hgb_pool_fwd(const float* x, const int32_t* graph_ptr, int32_t g, int32_t c, int32_t mode, float* out,
                            int32_t* argmax, hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && c > 0 && graph_ptr && out && mode >= 0 && mode <= 2, "pool_fwd: bad arguments");
  HGB_REQUIRE(mode != HGB_POOL_MAX || argmax, "pool_fwd: max pooling needs an argmax buffer");
  if (g == 0) return HGB_OK;
  pool_fwd_kernel<<<hgb_grid_for(g, 8), 256, 0, (cudaStream_t)stream>>>(x, graph_ptr, g, c, mode, out, argmax);
  HGB_LAUNCH_CHECK("pool_fwd");
  return HGB_OK;
}

extern "C" int hgb_pool_bwd(const float* gout, const int32_t* graph_ptr, const int32_t* argmax, const float* relu_y, int32_t n,
                            int32_t g, int32_t c, int32_t mode, float* gx, hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && c > 0 && graph_ptr && gx && mode >= 0 && mode <= 2, "pool_bwd: bad arguments");
  HGB_REQUIRE(mode != HGB_POOL_MAX || argmax, "pool_bwd: max pooling needs the argmax buffer");
  HGB_REQUIRE(mode != HGB_POOL_MAX || !relu_y, "pool_bwd: the ReLU mask is for add / mean pooling");
  HGB_REQUIRE(n >= 0, "pool_bwd: bad row count");
  if (g == 0 && n == 0) return HGB_OK;
  pool_bwd_kernel<<<hgb_grid_for(g, 8), 256, 0, (cudaStream_t)stream>>>(gout, graph_ptr, argmax, relu_y, n, g, c, mode, gx);
  HGB_LAUNCH_CHECK("pool_bwd");
  return HGB_OK;
}

// ---- segmented arg-min / arg-max (PNA aggregators, hydragnn/models/PNAEqStack.py:396-400) ---------------------
// For every (node, channel): the EDGE id holding the minimum / maximum over the node's CSR segment (first one wins
// on ties, -1 for an empty segment).  Values and gradients are then plain gathers at those ids.
__global__ void segment_argminmax_kernel(const float* __restrict__ m, const int32_t* __restrict__ rowptr,
                                         const int32_t* __restrict__ perm, int n, int c, int lanes, int64_t* __restrict__ amin,
                                         int64_t* __restrict__ amax) {
  const int gpb = blockDim.x / lanes;
  const int sub = threadIdx.x % lanes;
  for (int row = blockIdx.x * gpb + threadIdx.x / lanes; row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    for (int ch = sub; ch < c; ch += lanes) {
      float vmin = INFINITY, vmax = -INFINITY;
      int64_t imin = -1, imax = -1;
      for (int p = lo; p < hi; ++p) {
        const int e = perm ? perm[p] : p;
        const float v = m[(int64_t)e * c + ch];
        if (imin < 0 || v < vmin) { vmin = v; imin = e; }
        if (imax < 0 || v > vmax) { vmax = v; imax = e; }
      }
      amin[(int64_t)row * c + ch] = imin;
      amax[(int64_t)row * c + ch] = imax;
    }
  }
}

extern "C" int hgb_segment_argminmax(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c,
                                     int64_t* argmin, int64_t* argmax, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && c > 0 && rowptr && argmin && argmax, "segment_argminmax: bad arguments");
  if (n == 0) return HGB_OK;
  const int lanes = group_lanes(c);
  segment_argminmax_kernel<<<hgb_grid_for(n, 256 / lanes), 256, 0, (cudaStream_t)stream>>>(m, rowptr, perm, n, c, lanes, argmin, argmax);
  HGB_LAUNCH_CHECK("segment_argminmax");
  return HGB_OK;
}

// ---- PNA aggregation: mean | min | max | std of every CSR segment in ONE pass (PNAEqStack.py:396-400; PyG 2.6.1
// MeanAggregation / MinAggregation / MaxAggregation / StdAggregation).  out [n, 4c]; amin / amax [n, c] hold the EDGE id
// of the first minimum / maximum (-1 for an empty segment) for the backward.  std = sqrt(clamp(E[x^2] - E[x]^2, 1e-5)),
// reported as 0 where it equals sqrt(1e-5) (PyG masks the clamped entries).
#define PNA_EPS 1e-5f

// The four aggregators of one (segment, channel), fed one value per edge in CSR order.  Shared by pna_aggregate_fwd (messages
// read from memory) and pna_conv_fwd (messages formed on the fly), so both apply the same tie and std rules.
struct PnaAcc {
  float s1 = 0.f, s2 = 0.f, vmin = 0.f, vmax = 0.f;
  int imin = -1, imax = -1;

  __device__ __forceinline__ void push(float v, int e) {
    s1 += v;
    s2 = fmaf(v, v, s2);
    if (imin < 0 || v < vmin) { vmin = v; imin = e; }
    if (imax < 0 || v > vmax) { vmax = v; imax = e; }
  }

  // o: the channel's column in an [.., 4c] output row; inv = 1 / max(segment length, 1)
  __device__ __forceinline__ void store(float inv, float* o, int c, int32_t* arg_min, int32_t* arg_max) const {
    const float mean = s1 * inv;
    float sd = sqrtf(fmaxf(s2 * inv - mean * mean, PNA_EPS));
    if (sd <= sqrtf(PNA_EPS)) sd = 0.f;
    o[0] = mean;
    o[c] = vmin;
    o[2 * c] = vmax;
    o[3 * c] = sd;
    *arg_min = imin;
    *arg_max = imax;
  }
};

__global__ void pna_aggregate_fwd_kernel(const float* __restrict__ m, const int32_t* __restrict__ rowptr,
                                         const int32_t* __restrict__ perm, int n, int c, int lanes, float* __restrict__ out,
                                         int32_t* __restrict__ amin, int32_t* __restrict__ amax) {
  const int gpb = blockDim.x / lanes;
  const int sub = threadIdx.x % lanes;
  for (int row = blockIdx.x * gpb + threadIdx.x / lanes; row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    const float inv = 1.f / (float)max(hi - lo, 1);
    for (int ch = sub; ch < c; ch += lanes) {
      PnaAcc acc;
      for (int p = lo; p < hi; ++p) {
        const int e = perm ? perm[p] : p;
        acc.push(__ldg(m + (int64_t)e * c + ch), e);
      }
      acc.store(inv, out + (int64_t)row * 4 * c + ch, c, amin + (int64_t)row * c + ch, amax + (int64_t)row * c + ch);
    }
  }
}

// g_m[e, ch] = g_mean/cnt + [e == amin] g_min + [e == amax] g_max + g_std (m - mean) / (cnt std)
__global__ void pna_aggregate_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ m, const float* __restrict__ out,
                                         const int32_t* __restrict__ idx, const int32_t* __restrict__ rowptr,
                                         const int32_t* __restrict__ amin, const int32_t* __restrict__ amax, int64_t total, int c,
                                         float* __restrict__ gm) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(t / c);
    const int ch = (int)(t - (int64_t)e * c);
    const int i = idx[e];
    const float inv = 1.f / (float)max(rowptr[i + 1] - rowptr[i], 1);
    const float* g = gout + (int64_t)i * 4 * c;
    const float* o = out + (int64_t)i * 4 * c;
    float acc = g[ch] * inv;
    if (amin[(int64_t)i * c + ch] == e) acc += g[c + ch];
    if (amax[(int64_t)i * c + ch] == e) acc += g[2 * c + ch];
    const float sd = o[3 * c + ch];
    if (sd > 0.f) acc = fmaf(g[3 * c + ch] * inv / sd, m[t] - o[ch], acc);
    gm[t] = acc;
  }
}

extern "C" int hgb_pna_aggregate_fwd(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c, float* out,
                                     int32_t* argmin, int32_t* argmax, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && c > 0 && rowptr && out && argmin && argmax, "pna_aggregate_fwd: bad arguments");
  if (n == 0) return HGB_OK;
  const int lanes = group_lanes(c);
  pna_aggregate_fwd_kernel<<<hgb_grid_for(n, 256 / lanes), 256, 0, (cudaStream_t)stream>>>(m, rowptr, perm, n, c, lanes, out, argmin, argmax);
  HGB_LAUNCH_CHECK("pna_aggregate_fwd");
  return HGB_OK;
}

extern "C" int hgb_pna_aggregate_bwd(const float* g_out, const float* m, const float* out, const int32_t* idx, const int32_t* rowptr,
                                     const int32_t* argmin, const int32_t* argmax, int64_t e, int32_t c, float* g_m, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && c > 0 && g_out && out && idx && rowptr && argmin && argmax && g_m, "pna_aggregate_bwd: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(m, "pna_aggregate_bwd: null messages");
  pna_aggregate_bwd_kernel<<<hgb_grid_for(e * c, 256), 256, 0, (cudaStream_t)stream>>>(g_out, m, out, idx, rowptr, argmin, argmax, e * c, c, g_m);
  HGB_LAUNCH_CHECK("pna_aggregate_bwd");
  return HGB_OK;
}

// ---- PNAConv message + aggregation in one pass (torch_geometric 2.6.1 PNAConv with towers = pre_layers = post_layers = 1,
// hydragnn/models/PNAStack.py:42-53).  The pre_nn Linear is affine in its blocks, so for the edge e = (j -> i)
//   h_e = P[i] + Q[j] + M a_e + c,   [P | Q] = x [W_a; W_b]^T (one per-node Linear), M = W_c W_enc [f, d], c = W_c b_enc + b_pre,
// and h_e is formed in registers and reduced straight into [mean | min | max | std]: no [E, f] tensor is written.
//
// Thread mapping: a group of `lanes` threads (a power of two <= 256) owns one target node; every thread owns a FIXED set of
// VEC consecutive channels (blockIdx.y selects the channel tile when f needs more than 256 * VEC), so M's rows for those
// channels stay in registers and the backward's parameter sums accumulate per thread across every node the thread visits.
#define PNA_MAX_D 16
#define PNA_BLOCK 256
#define PNA_BWD_MAX_BLOCKS (HGB_NUM_SMS * 4)

template <int VEC, int MAXD>
struct PnaChan {
  float m[MAXD > 0 ? MAXD : 1][VEC];   // M[ch, k] of the thread's channels
  float c[VEC];

  __device__ __forceinline__ void load(const float* __restrict__ mt, const float* __restrict__ cvec, int d, int f, int ch0) {
#pragma unroll
    for (int j = 0; j < VEC; ++j) c[j] = cvec ? __ldg(cvec + ch0 + j) : 0.f;
#pragma unroll
    for (int k = 0; k < MAXD; ++k)
#pragma unroll
      for (int j = 0; j < VEC; ++j) m[k][j] = k < d ? __ldg(mt + (int64_t)k * f + ch0 + j) : 0.f;
  }
};

template <int VEC>
__device__ __forceinline__ void pna_load(const float* __restrict__ p, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = __ldg(p);
  }
}

// h_e for the thread's channels: base = P[i] + c (per node), then + Q[src] + sum_k M[., k] a_e[k].  The forward and the
// backward both call this, so the backward sees the forward's h_e bit for bit (its argmin / argmax / std mask agree).
template <int VEC, int MAXD>
__device__ __forceinline__ void pna_message(const PnaChan<VEC, MAXD>& ch, const float (&base)[VEC], const float* __restrict__ q_row,
                                            const float* __restrict__ a_row, int d, float (&h)[VEC]) {
  pna_load<VEC>(q_row, h);
#pragma unroll
  for (int j = 0; j < VEC; ++j) h[j] += base[j];
  if (MAXD > 0 && d > 0) {
#pragma unroll
    for (int k = 0; k < MAXD; ++k) {
      if (k < d) {
        const float a = __ldg(a_row + k);
#pragma unroll
        for (int j = 0; j < VEC; ++j) h[j] = fmaf(ch.m[k][j], a, h[j]);
      }
    }
  }
}

template <int VEC, int MAXD>
__global__ void __launch_bounds__(PNA_BLOCK, 1) pna_conv_fwd_kernel(
    const float* __restrict__ pq, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm,
    const int32_t* __restrict__ src, const float* __restrict__ eattr, int d, const float* __restrict__ mt,
    const float* __restrict__ cvec, int n, int f, int lanes, float* __restrict__ out, int32_t* __restrict__ amin,
    int32_t* __restrict__ amax) {
  const int gpb = blockDim.x / lanes;
  const int ch0 = (blockIdx.y * lanes + threadIdx.x % lanes) * VEC;
  if (ch0 >= f) return;                                  // no block-wide synchronisation below
  PnaChan<VEC, MAXD> chan;
  chan.load(mt, cvec, d, f, ch0);
  for (int row = blockIdx.x * gpb + threadIdx.x / lanes; row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    const float inv = 1.f / (float)max(hi - lo, 1);
    float base[VEC];
    pna_load<VEC>(pq + (int64_t)row * 2 * f + ch0, base);
#pragma unroll
    for (int j = 0; j < VEC; ++j) base[j] += chan.c[j];
    PnaAcc acc[VEC];
    for (int p = lo; p < hi; ++p) {
      const int e = perm ? perm[p] : p;
      float h[VEC];
      pna_message<VEC, MAXD>(chan, base, pq + (int64_t)src[p] * 2 * f + f + ch0, eattr + (int64_t)e * d, d, h);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j].push(h[j], e);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      acc[j].store(inv, out + (int64_t)row * 4 * f + ch0 + j, f, amin + (int64_t)row * f + ch0 + j, amax + (int64_t)row * f + ch0 + j);
  }
}

// g_h_e = g_mean / deg + [e = amin] g_min + [e = amax] g_max + g_std (h_e - mean) / (deg std)   (std term 0 where std was masked),
// the same rule as pna_aggregate_bwd_kernel.  g_p[i] = sum over i's segment; g_h written once per edge (Q was gathered by the
// source, so g_Q is a segment sum over the by-source CSR).  part [gridDim.x, 1 + d, f]: per-CTA sum_e g_h_e and sum_e g_h_e a_e^T.
template <int VEC, int MAXD>
__global__ void __launch_bounds__(PNA_BLOCK, 1) pna_conv_bwd_kernel(
    const float* __restrict__ g_out, const float* __restrict__ pq, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ src, const float* __restrict__ eattr, int d,
    const float* __restrict__ mt, const float* __restrict__ cvec, const float* __restrict__ agg,
    const int32_t* __restrict__ amin, const int32_t* __restrict__ amax, int n, int f, int lanes, float* __restrict__ g_p,
    int ldgp, float* __restrict__ g_h, float* __restrict__ part) {
  __shared__ float red[PNA_BLOCK * VEC];
  const int gpb = blockDim.x / lanes;
  const int sub = threadIdx.x % lanes;
  const int ch0 = (blockIdx.y * lanes + sub) * VEC;
  const bool active = ch0 < f;
  PnaChan<VEC, MAXD> chan;
  float gc[VEC], gm[MAXD > 0 ? MAXD : 1][VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    gc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXD; ++k) gm[k][j] = 0.f;
  }
  if (active) {
    chan.load(mt, cvec, d, f, ch0);
    for (int row = blockIdx.x * gpb + threadIdx.x / lanes; row < n; row += gridDim.x * gpb) {
      const int lo = rowptr[row], hi = rowptr[row + 1];
      const float inv = 1.f / (float)max(hi - lo, 1);
      const float* g = g_out + (int64_t)row * 4 * f + ch0;
      const float* o = agg + (int64_t)row * 4 * f + ch0;
      float base[VEC], gmean[VEC], gmin[VEC], gmax[VEC], kstd[VEC], mean[VEC], gp[VEC];
      int imin[VEC], imax[VEC];
      pna_load<VEC>(pq + (int64_t)row * 2 * f + ch0, base);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        base[j] += chan.c[j];
        gmean[j] = g[j] * inv;
        gmin[j] = g[f + j];
        gmax[j] = g[2 * f + j];
        mean[j] = o[j];
        const float sd = o[3 * f + j];
        kstd[j] = sd > 0.f ? g[3 * f + j] * inv / sd : 0.f;
        imin[j] = amin[(int64_t)row * f + ch0 + j];
        imax[j] = amax[(int64_t)row * f + ch0 + j];
        gp[j] = 0.f;
      }
      for (int p = lo; p < hi; ++p) {
        const int e = perm ? perm[p] : p;
        const float* a_row = eattr + (int64_t)e * d;
        float h[VEC];
        pna_message<VEC, MAXD>(chan, base, pq + (int64_t)src[p] * 2 * f + f + ch0, a_row, d, h);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          float acc = gmean[j];
          if (imin[j] == e) acc += gmin[j];
          if (imax[j] == e) acc += gmax[j];
          if (kstd[j] != 0.f) acc = fmaf(kstd[j], h[j] - mean[j], acc);
          h[j] = acc;                                      // h now holds g_h_e
          gp[j] += acc;
          gc[j] += acc;
        }
        if (MAXD > 0 && d > 0) {
#pragma unroll
          for (int k = 0; k < MAXD; ++k) {
            if (k < d) {
              const float a = __ldg(a_row + k);
#pragma unroll
              for (int j = 0; j < VEC; ++j) gm[k][j] = fmaf(h[j], a, gm[k][j]);
            }
          }
        }
        float* gh = g_h + (int64_t)e * f + ch0;
        if constexpr (VEC == 4) *reinterpret_cast<float4*>(gh) = make_float4(h[0], h[1], h[2], h[3]);
        else gh[0] = h[0];
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j) g_p[(int64_t)row * ldgp + ch0 + j] = gp[j];
    }
  }
  // fixed-order reduction over the CTA's node groups, one parameter row (c, then M[:, k]) at a time
#pragma unroll
  for (int k = 0; k <= MAXD; ++k) {
    if (k <= d) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) red[threadIdx.x * VEC + j] = k == 0 ? gc[j] : gm[k > 0 ? k - 1 : 0][j];
      __syncthreads();
      if (threadIdx.x < lanes && active) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          float s = 0.f;
          for (int grp = 0; grp < gpb; ++grp) s += red[(grp * lanes + sub) * VEC + j];
          part[((int64_t)blockIdx.x * (d + 1) + k) * f + ch0 + j] = s;
        }
      }
      __syncthreads();
    }
  }
}

// out[r] = sum over the CTAs in index order (fp64) of part[b, r]
__global__ void pna_conv_reduce_kernel(const float* __restrict__ part, int nblk, int rows, float* __restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += (double)part[(int64_t)b * rows + r];
    out[r] = (float)s;
  }
}

namespace {
struct PnaLaunch {
  bool v4;
  int lanes, gpb;
  dim3 grid;
};

PnaLaunch pna_launch(const float* pq, int32_t n, int32_t f, int max_blocks, const void* extra_aligned = nullptr) {
  PnaLaunch L;
  L.v4 = (f % 4 == 0) && ((uintptr_t)pq % 16 == 0) && ((uintptr_t)extra_aligned % 16 == 0);
  const int cv = L.v4 ? f / 4 : f;
  L.lanes = 1;
  while (L.lanes < cv && L.lanes < PNA_BLOCK) L.lanes <<= 1;
  L.gpb = PNA_BLOCK / L.lanes;
  L.grid = dim3(hgb_grid_for(n, L.gpb, max_blocks), (cv + L.lanes - 1) / L.lanes);
  return L;
}
}  // namespace

// instantiations by vector width and edge-attribute capacity (0, 4 or 16): the registers holding M and the backward's
// g_M accumulators are sized by the capacity, so narrow or absent edge attributes do not pay for d = 16
#define PNA_DISPATCH(LAUNCH)                           \
  do {                                                 \
    if (L.v4) {                                        \
      if (d == 0) LAUNCH(4, 0);                        \
      else if (d <= 4) LAUNCH(4, 4);                   \
      else LAUNCH(4, 16);                              \
    } else {                                           \
      if (d == 0) LAUNCH(1, 0);                        \
      else if (d <= 4) LAUNCH(1, 4);                   \
      else LAUNCH(1, 16);                              \
    }                                                  \
  } while (0)

extern "C" int64_t hgb_pna_conv_workspace_bytes(int32_t f, int32_t d) {
  if (f <= 0 || d < 0 || d > PNA_MAX_D) return -1;
  return (int64_t)PNA_BWD_MAX_BLOCKS * (d + 1) * f * (int64_t)sizeof(float);
}

extern "C" int hgb_pna_conv_fwd(const float* pq, const int32_t* rowptr, const int32_t* perm, const int32_t* src,
                                const float* eattr, int32_t d, const float* mt, const float* cvec, int32_t n, int32_t f,
                                float* out, int32_t* argmin, int32_t* argmax, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && f > 0 && d >= 0 && d <= PNA_MAX_D, "pna_conv_fwd: bad sizes (n %d, f %d, d %d; d <= %d)", n, f, d, PNA_MAX_D);
  HGB_REQUIRE(pq && rowptr && src && out && argmin && argmax, "pna_conv_fwd: null argument");
  HGB_REQUIRE(d == 0 || (eattr && mt), "pna_conv_fwd: d > 0 needs edge attributes and M");
  if (n == 0) return HGB_OK;
  const PnaLaunch L = pna_launch(pq, n, f, HGB_NUM_SMS * 16);
#define PNA_FWD(V, D)                                                                                                        \
  pna_conv_fwd_kernel<V, D><<<L.grid, PNA_BLOCK, 0, (cudaStream_t)stream>>>(pq, rowptr, perm, src, eattr, d, mt, cvec, n, f, \
                                                                           L.lanes, out, argmin, argmax)
  PNA_DISPATCH(PNA_FWD);
#undef PNA_FWD
  HGB_LAUNCH_CHECK("pna_conv_fwd");
  return HGB_OK;
}

extern "C" int hgb_pna_conv_bwd(const float* g_out, const float* pq, const int32_t* rowptr, const int32_t* perm,
                                const int32_t* src, const float* eattr, int32_t d, const float* mt, const float* cvec,
                                const float* out, const int32_t* argmin, const int32_t* argmax, int32_t n, int32_t f,
                                float* g_p, int32_t ldgp, float* g_h, float* g_cm, void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && f > 0 && d >= 0 && d <= PNA_MAX_D && ldgp >= f,
              "pna_conv_bwd: bad sizes (n %d, f %d, d %d, ldgp %d)", n, f, d, ldgp);
  HGB_REQUIRE(g_out && pq && rowptr && src && out && argmin && argmax && g_p && g_h && g_cm && workspace,
              "pna_conv_bwd: null argument");
  HGB_REQUIRE(d == 0 || (eattr && mt), "pna_conv_bwd: d > 0 needs edge attributes and M");
  if (n == 0) {
    cudaMemsetAsync(g_cm, 0, sizeof(float) * (size_t)(d + 1) * f, (cudaStream_t)stream);
    HGB_LAUNCH_CHECK("pna_conv_bwd");
    return HGB_OK;
  }
  // the float4 path also stores g_h with float4 writes, so g_h must be 16-byte aligned as well
  const PnaLaunch L = pna_launch(pq, n, f, PNA_BWD_MAX_BLOCKS, g_h);
  float* part = static_cast<float*>(workspace);
#define PNA_BWD(V, D)                                                                                                         \
  pna_conv_bwd_kernel<V, D><<<L.grid, PNA_BLOCK, 0, (cudaStream_t)stream>>>(g_out, pq, rowptr, perm, src, eattr, d, mt, cvec, \
                                                                           out, argmin, argmax, n, f, L.lanes, g_p, ldgp, g_h, part)
  PNA_DISPATCH(PNA_BWD);
#undef PNA_BWD
  HGB_LAUNCH_CHECK("pna_conv_bwd");
  const int rows = (d + 1) * f;
  pna_conv_reduce_kernel<<<hgb_grid_for(rows, 256), 256, 0, (cudaStream_t)stream>>>(part, (int)L.grid.x, rows, g_cm);
  HGB_LAUNCH_CHECK("pna_conv_reduce");
  return HGB_OK;
}

// ---- PNAPlus: PNAConv with a Bessel-gated message (hydragnn/models/PNAPlusStack.py:144-279, torch_geometric 2.6.1
// BesselBasisLayer / Envelope), message and four-way aggregation in one pass.  For the edge e = (j -> i) with length d_e:
//   x = d_e / radius,  rbf_k = env(x) sin(freq_k x)  (0 for x >= 1),  u_e = relu(W_r rbf + b_r),
//   h_e = P[i] + Q[j] + M_r u_e + M_a a_e + c,  m_e = h_e * (W_l rbf),
// reduced straight into [mean | min | max | std] by the PnaAcc of pna_conv_fwd.  Only d_e [E] is read per edge: the [E, R]
// basis, the [E, F] embedding u and the message are formed on chip.
//
// Thread mapping: one warp owns one target node, lane l the channels l and l + 32 (F <= 64).  The per-edge F x F product
// M_r u_e is SIMT: u_e goes through a per-warp shared row, M_r sits in shared memory with an odd row stride, so both the
// row-wise read of the forward and the column-wise read of the backward are free of bank conflicts.
#define PNAP_MAX_F 64
#define PNAP_MAX_R 16
#define PNAP_MAX_D 16
#define PNAP_BWD_MAX_BLOCKS (HGB_NUM_SMS * 2)

static __host__ __device__ __forceinline__ int pnap_stride(int f) { return f | 1; }

// parameters staged in shared memory once per CTA: mr [f][s] (s odd), wr / wl [r][f], ma [d][f], br, cv [f], fr [r]
struct PnapParams {
  float *mr, *wr, *wl, *ma, *br, *cv, *fr, *end;

  static __host__ __device__ int64_t floats(int f, int r, int d) { return (int64_t)f * pnap_stride(f) + 2 * r * f + d * f + 2 * f + r; }

  __device__ void stage(float* base, int f, int r, int d, const float* __restrict__ g_mr, const float* __restrict__ g_wr,
                        const float* __restrict__ g_wl, const float* __restrict__ g_mat, const float* __restrict__ g_br,
                        const float* __restrict__ g_cv, const float* __restrict__ g_fr) {
    const int s = pnap_stride(f);
    mr = base;
    wr = mr + f * s;
    wl = wr + r * f;
    ma = wl + r * f;
    br = ma + d * f;
    cv = br + f;
    fr = cv + f;
    end = fr + r;
    for (int t = threadIdx.x; t < f * f; t += blockDim.x) mr[(t / f) * s + t % f] = __ldg(g_mr + t);
    for (int t = threadIdx.x; t < r * f; t += blockDim.x) {
      const int k = t / f, c = t % f;
      wr[t] = __ldg(g_wr + c * r + k);
      wl[t] = __ldg(g_wl + c * r + k);
    }
    for (int t = threadIdx.x; t < d * f; t += blockDim.x) ma[t] = __ldg(g_mat + t);
    for (int t = threadIdx.x; t < f; t += blockDim.x) {
      br[t] = __ldg(g_br + t);
      cv[t] = g_cv ? __ldg(g_cv + t) : 0.f;
    }
    for (int t = threadIdx.x; t < r; t += blockDim.x) fr[t] = __ldg(g_fr + t);
    __syncthreads();
  }
};

// x = d / radius, env(x) and d env / dx (both 0 for x >= 1), rb[k] = env sin(freq_k x)
__device__ __forceinline__ void pnap_basis(float dist, float radius, int expo, const float* fr, int r, float (&rb)[PNAP_MAX_R],
                                           float& x, float& env, float& denv) {
  x = dist / radius;
  const int p = expo + 1;
  const float a = -(float)((p + 1) * (p + 2)) / 2.f, b = (float)(p * (p + 2)), c = -(float)(p * (p + 1)) / 2.f;
  float xp0 = 1.f;
  for (int q = 0; q < p - 1; ++q) xp0 *= x;
  const float xp1 = xp0 * x, xp2 = xp1 * x;
  const bool in = x < 1.f;
  env = in ? 1.f / x + a * xp0 + b * xp1 + c * xp2 : 0.f;
  denv = in ? -1.f / (x * x) + a * (float)(p - 1) * (xp0 / x) + b * (float)p * xp0 + c * (float)(p + 1) * xp1 : 0.f;
#pragma unroll
  for (int k = 0; k < PNAP_MAX_R; ++k) rb[k] = (k < r && in) ? env * sinf(fr[k] * x) : 0.f;
}

// upre = W_r rb + b_r, gate = W_l rb, h = base + Q[j] + M_r relu(upre) + M_a a for the lane's channels.  The forward and the
// backward both call this, so the backward sees the forward's m_e = h * gate bit for bit.  u_s: the warp's [f] row.
template <int NC>
__device__ __forceinline__ void pnap_message(const PnapParams& s, int f, int r, int d, int lane, float* u_s, const float (&base)[NC],
                                             const float* __restrict__ q_row, const float* __restrict__ a_row,
                                             const float (&rb)[PNAP_MAX_R], float (&upre)[NC], float (&gate)[NC], float (&h)[NC]) {
  const int sr = pnap_stride(f);
  __syncwarp();                                           // the previous edge's reads of u_s are done
#pragma unroll
  for (int t = 0; t < NC; ++t) {
    const int c = lane + 32 * t;
    float ub = 0.f, g = 0.f;
    if (c < f) {
      ub = s.br[c];
#pragma unroll
      for (int k = 0; k < PNAP_MAX_R; ++k) {
        if (k < r) {
          ub = fmaf(s.wr[k * f + c], rb[k], ub);
          g = fmaf(s.wl[k * f + c], rb[k], g);
        }
      }
      u_s[c] = fmaxf(ub, 0.f);
    }
    upre[t] = ub;
    gate[t] = g;
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < NC; ++t) {
    const int c = lane + 32 * t;
    float acc = 0.f;
    if (c < f) {
      acc = base[t] + __ldg(q_row + c);
      const float* mrow = s.mr + c * sr;
      for (int m = 0; m < f; ++m) acc = fmaf(mrow[m], u_s[m], acc);
      for (int k = 0; k < d; ++k) acc = fmaf(s.ma[k * f + c], __ldg(a_row + k), acc);
    }
    h[t] = acc;
  }
}

template <int NC>
__global__ void __launch_bounds__(256) pnaplus_conv_fwd_kernel(
    const float* __restrict__ pq, const float* __restrict__ dist, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ src, const float* __restrict__ eattr, int d,
    const float* __restrict__ freq, int r, float radius, int expo, const float* __restrict__ wr, const float* __restrict__ br,
    const float* __restrict__ wl, const float* __restrict__ mr, const float* __restrict__ mat, const float* __restrict__ cvec,
    int n, int f, float* __restrict__ out, int32_t* __restrict__ amin, int32_t* __restrict__ amax) {
  extern __shared__ float smem[];
  PnapParams s;
  s.stage(smem, f, r, d, mr, wr, wl, mat, br, cvec, freq);
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* u_s = s.end + warp * f;
  for (int row = blockIdx.x * warps + warp; row < n; row += gridDim.x * warps) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    const float inv = 1.f / (float)max(hi - lo, 1);
    float base[NC];
#pragma unroll
    for (int t = 0; t < NC; ++t) {
      const int c = lane + 32 * t;
      base[t] = c < f ? __ldg(pq + (int64_t)row * 2 * f + c) + s.cv[c] : 0.f;
    }
    PnaAcc acc[NC];
    for (int p = lo; p < hi; ++p) {
      const int e = perm ? perm[p] : p;
      float rb[PNAP_MAX_R], x, env, denv, upre[NC], gate[NC], h[NC];
      pnap_basis(__ldg(dist + e), radius, expo, s.fr, r, rb, x, env, denv);
      pnap_message<NC>(s, f, r, d, lane, u_s, base, pq + (int64_t)src[p] * 2 * f + f, eattr + (int64_t)e * d, rb, upre, gate, h);
#pragma unroll
      for (int t = 0; t < NC; ++t)
        if (lane + 32 * t < f) acc[t].push(h[t] * gate[t], e);
    }
#pragma unroll
    for (int t = 0; t < NC; ++t) {
      const int c = lane + 32 * t;
      if (c < f) acc[t].store(inv, out + (int64_t)row * 4 * f + c, f, amin + (int64_t)row * f + c, amax + (int64_t)row * f + c);
    }
  }
}

// Parameter-gradient layout (the order of g_params): c [f] | M_a^T [d][f] | M_r [f][f] | W_r^T [r][f] | b_r [f] | W_l^T [r][f] |
// freq [r].  Per warp the accumulators live in shared memory in the same order, M_r with the odd row stride.
struct PnapGrad {
  float *c, *ma, *mr, *wr, *br, *wl, *fr;
  static __host__ __device__ int64_t floats(int f, int r, int d) { return (int64_t)f + d * f + (int64_t)f * f + 2 * r * f + f + r; }
  static __host__ __device__ int64_t smem_floats(int f, int r, int d) { return floats(f, r, d) + (int64_t)f * (pnap_stride(f) - f); }
  __device__ void carve(float* base, int f, int r, int d) {
    c = base;
    ma = c + f;
    mr = ma + d * f;
    wr = mr + f * pnap_stride(f);
    br = wr + r * f;
    wl = br + f;
    fr = wl + r * f;
  }
};

// g_m = g_mean / deg + [e = amin] g_min + [e = amax] g_max + g_std (m - mean) / (deg std), as pna_conv_bwd_kernel; then
// g_h = g_m * gate, g_gate = g_m * h, g_u = M_r^T g_h, g_upre = [upre > 0] g_u, g_rbf = W_r^T g_upre + W_l^T g_gate.
// g_p[i] summed in registers; g_h written once per edge; g_dist / g_eattr per edge when asked; with `grads` the parameter
// sums go to per-warp shared accumulators, summed over the CTA's warps in order into part [gridDim.x, PnapGrad::floats].
template <int NC>
__global__ void __launch_bounds__(256) pnaplus_conv_bwd_kernel(
    const float* __restrict__ g_out, const float* __restrict__ pq, const float* __restrict__ dist, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ src, const float* __restrict__ eattr, int d,
    const float* __restrict__ freq, int r, float radius, int expo, const float* __restrict__ wr, const float* __restrict__ br,
    const float* __restrict__ wl, const float* __restrict__ mr, const float* __restrict__ mat, const float* __restrict__ cvec,
    const float* __restrict__ agg, const int32_t* __restrict__ amin, const int32_t* __restrict__ amax, int n, int f,
    float* __restrict__ g_p, int ldgp, float* __restrict__ g_h, float* __restrict__ g_dist, float* __restrict__ g_eattr,
    bool grads, float* __restrict__ part) {
  extern __shared__ float smem[];
  PnapParams s;
  s.stage(smem, f, r, d, mr, wr, wl, mat, br, cvec, freq);
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sr = pnap_stride(f);
  const int64_t per_warp = 2 * f + (grads ? PnapGrad::smem_floats(f, r, d) : 0);
  float* u_s = s.end + warp * per_warp;
  float* gh_s = u_s + f;
  PnapGrad A;
  A.carve(gh_s + f, f, r, d);
  if (grads)
    for (int64_t q = lane; q < PnapGrad::smem_floats(f, r, d); q += 32) A.c[q] = 0.f;
  const bool want_rbf = grads || g_dist;
  float gfreq = 0.f;                                      // lane k < r: sum of g_freq[k]
  for (int row = blockIdx.x * warps + warp; row < n; row += gridDim.x * warps) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    const float inv = 1.f / (float)max(hi - lo, 1);
    float base[NC], gmean[NC], gmin[NC], gmax[NC], kstd[NC], mean[NC], gp[NC];
    int imin[NC], imax[NC];
#pragma unroll
    for (int t = 0; t < NC; ++t) {
      const int c = lane + 32 * t;
      const bool on = c < f;
      const float* g = g_out + (int64_t)row * 4 * f + c;
      const float* o = agg + (int64_t)row * 4 * f + c;
      base[t] = on ? __ldg(pq + (int64_t)row * 2 * f + c) + s.cv[c] : 0.f;
      gmean[t] = on ? g[0] * inv : 0.f;
      gmin[t] = on ? g[f] : 0.f;
      gmax[t] = on ? g[2 * f] : 0.f;
      mean[t] = on ? o[0] : 0.f;
      const float sd = on ? o[3 * f] : 0.f;
      kstd[t] = sd > 0.f ? g[3 * f] * inv / sd : 0.f;
      imin[t] = on ? amin[(int64_t)row * f + c] : -1;
      imax[t] = on ? amax[(int64_t)row * f + c] : -1;
      gp[t] = 0.f;
    }
    for (int p = lo; p < hi; ++p) {
      const int e = perm ? perm[p] : p;
      const float* a_row = eattr + (int64_t)e * d;
      float rb[PNAP_MAX_R], x, env, denv, upre[NC], gate[NC], h[NC], gh[NC], gg[NC];
      pnap_basis(__ldg(dist + e), radius, expo, s.fr, r, rb, x, env, denv);
      pnap_message<NC>(s, f, r, d, lane, u_s, base, pq + (int64_t)src[p] * 2 * f + f, a_row, rb, upre, gate, h);
#pragma unroll
      for (int t = 0; t < NC; ++t) {
        const int c = lane + 32 * t;
        gh[t] = gg[t] = 0.f;
        if (c < f) {
          float gm = gmean[t];
          if (imin[t] == e) gm += gmin[t];
          if (imax[t] == e) gm += gmax[t];
          if (kstd[t] != 0.f) gm = fmaf(kstd[t], h[t] * gate[t] - mean[t], gm);
          gh[t] = gm * gate[t];
          gg[t] = gm * h[t];
          gp[t] += gh[t];
          g_h[(int64_t)e * f + c] = gh[t];
          gh_s[c] = gh[t];
          if (grads) {
            A.c[c] += gh[t];
            for (int k = 0; k < d; ++k) A.ma[k * f + c] = fmaf(gh[t], __ldg(a_row + k), A.ma[k * f + c]);
#pragma unroll
            for (int k = 0; k < PNAP_MAX_R; ++k)
              if (k < r) A.wl[k * f + c] = fmaf(gg[t], rb[k], A.wl[k * f + c]);
            float* arow = A.mr + c * sr;
            for (int m = 0; m < f; ++m) arow[m] = fmaf(gh[t], u_s[m], arow[m]);
          }
        }
      }
      __syncwarp();                                       // gh_s complete
      float grbf[PNAP_MAX_R];
#pragma unroll
      for (int k = 0; k < PNAP_MAX_R; ++k) grbf[k] = 0.f;
#pragma unroll
      for (int t = 0; t < NC; ++t) {
        const int c = lane + 32 * t;
        if (c < f) {
          float gu = 0.f;
          for (int q = 0; q < f; ++q) gu = fmaf(s.mr[q * sr + c], gh_s[q], gu);
          const float gpre = upre[t] > 0.f ? gu : 0.f;
          if (grads) {
            A.br[c] += gpre;
#pragma unroll
            for (int k = 0; k < PNAP_MAX_R; ++k)
              if (k < r) A.wr[k * f + c] = fmaf(gpre, rb[k], A.wr[k * f + c]);
          }
          if (want_rbf) {
#pragma unroll
            for (int k = 0; k < PNAP_MAX_R; ++k)
              if (k < r) grbf[k] = fmaf(s.wr[k * f + c], gpre, fmaf(s.wl[k * f + c], gg[t], grbf[k]));
          }
        }
      }
      if (want_rbf) {
        float gx = 0.f;
#pragma unroll
        for (int k = 0; k < PNAP_MAX_R; ++k) {
          if (k < r) {
            const float gk = hgb_warp_sum(grbf[k]);
            if (x < 1.f) {
              float sn, cs;
              sincosf(s.fr[k] * x, &sn, &cs);
              gx = fmaf(gk, fmaf(denv, sn, env * s.fr[k] * cs), gx);
              if (lane == k) gfreq = fmaf(gk, env * x * cs, gfreq);
            }
          }
        }
        if (g_dist && lane == 0) g_dist[e] = gx / radius;
      }
      if (g_eattr) {
        for (int k = 0; k < d; ++k) {
          float v = 0.f;
#pragma unroll
          for (int t = 0; t < NC; ++t)
            if (lane + 32 * t < f) v = fmaf(s.ma[k * f + lane + 32 * t], gh[t], v);
          v = hgb_warp_sum(v);
          if (lane == 0) g_eattr[(int64_t)e * d + k] = v;
        }
      }
    }
#pragma unroll
    for (int t = 0; t < NC; ++t) {
      const int c = lane + 32 * t;
      if (c < f) g_p[(int64_t)row * ldgp + c] = gp[t];
    }
  }
  if (!grads) return;                                     // grid-uniform: no CTA skips the barrier below alone
  if (lane < r) A.fr[lane] = gfreq;
  __syncthreads();
  // fixed-order sum over the CTA's warps, written unpadded
  const int64_t total = PnapGrad::floats(f, r, d), mr0 = f + (int64_t)d * f, mr1 = mr0 + (int64_t)f * f;
  for (int64_t q = threadIdx.x; q < total; q += blockDim.x) {
    const int64_t qs = q < mr0 ? q : (q < mr1 ? mr0 + ((q - mr0) / f) * sr + (q - mr0) % f : q + (int64_t)f * (sr - f));
    float v = 0.f;
    for (int w = 0; w < warps; ++w) v += s.end[w * per_warp + 2 * f + qs];
    part[(int64_t)blockIdx.x * total + q] = v;
  }
}

namespace {
// warps per CTA and dynamic shared bytes; the backward's per-warp accumulators grow as f^2, so wide rows run 4 warps
struct PnapLaunch {
  int warps;
  size_t fwd_smem, bwd_smem;
};

PnapLaunch pnap_launch(int f, int r, int d, bool grads) {
  PnapLaunch L;
  const int64_t params = PnapParams::floats(f, r, d);
  const int64_t per_warp = 2 * f + (grads ? PnapGrad::smem_floats(f, r, d) : 0);
  L.warps = (params + 8 * per_warp) * 4 <= 200 * 1024 ? 8 : 4;
  L.fwd_smem = (size_t)(params + 8 * f) * 4;
  L.bwd_smem = (size_t)(params + L.warps * per_warp) * 4;
  return L;
}
}  // namespace

extern "C" int hgb_pnaplus_conv_supported(int32_t f, int32_t r, int32_t d) {
  return f >= 1 && f <= PNAP_MAX_F && r >= 1 && r <= PNAP_MAX_R && d >= 0 && d <= PNAP_MAX_D;
}

extern "C" int64_t hgb_pnaplus_conv_workspace_bytes(int32_t f, int32_t r, int32_t d) {
  if (!hgb_pnaplus_conv_supported(f, r, d)) return -1;
  return (int64_t)PNAP_BWD_MAX_BLOCKS * PnapGrad::floats(f, r, d) * (int64_t)sizeof(float);
}

#define PNAP_CHECK_ARGS(name)                                                                                                \
  HGB_REQUIRE(n >= 0 && hgb_pnaplus_conv_supported(f, r, d) && radius > 0.f && expo >= 0,                                  \
              name ": bad sizes (n %d, f %d, r %d, d %d, radius %g, exponent %d; f <= %d, r <= %d, d <= %d)", n, f, r, d,     \
              (double)radius, expo, PNAP_MAX_F, PNAP_MAX_R, PNAP_MAX_D);                                                     \
  HGB_REQUIRE(pq && dist && rowptr && src && freq && wr && br && wl && mr && cvec, name ": null argument");                  \
  HGB_REQUIRE(d == 0 || (eattr && mat), name ": d > 0 needs edge attributes and M_a")

extern "C" int hgb_pnaplus_conv_fwd(const float* pq, const float* dist, const int32_t* rowptr, const int32_t* perm, const int32_t* src,
                                    const float* eattr, int32_t d, const float* freq, int32_t r, float radius, int32_t expo,
                                    const float* wr, const float* br, const float* wl, const float* mr, const float* mat,
                                    const float* cvec, int32_t n, int32_t f, float* out, int32_t* argmin, int32_t* argmax,
                                    hgb_stream_t stream) {
  PNAP_CHECK_ARGS("pnaplus_conv_fwd");
  HGB_REQUIRE(out && argmin && argmax, "pnaplus_conv_fwd: null output");
  if (n == 0) return HGB_OK;
  const PnapLaunch L = pnap_launch(f, r, d, false);
  const int grid = hgb_grid_for(n, 8);
#define PNAP_FWD(NC)                                                                                                         \
  do {                                                                                                                       \
    cudaFuncSetAttribute(pnaplus_conv_fwd_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.fwd_smem);        \
    pnaplus_conv_fwd_kernel<NC><<<grid, 256, L.fwd_smem, (cudaStream_t)stream>>>(pq, dist, rowptr, perm, src, eattr, d, freq, \
                                                                                 r, radius, expo, wr, br, wl, mr, mat, cvec, \
                                                                                 n, f, out, argmin, argmax);                 \
  } while (0)
  if (f <= 32) PNAP_FWD(1);
  else PNAP_FWD(2);
#undef PNAP_FWD
  HGB_LAUNCH_CHECK("pnaplus_conv_fwd");
  return HGB_OK;
}

extern "C" int hgb_pnaplus_conv_bwd(const float* g_out, const float* pq, const float* dist, const int32_t* rowptr, const int32_t* perm,
                                    const int32_t* src, const float* eattr, int32_t d, const float* freq, int32_t r, float radius,
                                    int32_t expo, const float* wr, const float* br, const float* wl, const float* mr, const float* mat,
                                    const float* cvec, const float* out, const int32_t* argmin, const int32_t* argmax, int32_t n,
                                    int32_t f, float* g_p, int32_t ldgp, float* g_h, float* g_dist, float* g_eattr, float* g_params,
                                    void* workspace, hgb_stream_t stream) {
  PNAP_CHECK_ARGS("pnaplus_conv_bwd");
  HGB_REQUIRE(ldgp >= f, "pnaplus_conv_bwd: ldgp %d < f %d", ldgp, f);
  HGB_REQUIRE(g_out && out && argmin && argmax && g_p && g_h, "pnaplus_conv_bwd: null argument");
  HGB_REQUIRE(!g_params || workspace, "pnaplus_conv_bwd: parameter gradients need the workspace");
  HGB_REQUIRE(!g_eattr || d > 0, "pnaplus_conv_bwd: g_eattr needs d > 0");
  const bool grads = g_params != nullptr;
  const int64_t rows = PnapGrad::floats(f, r, d);
  if (n == 0) {
    if (grads) cudaMemsetAsync(g_params, 0, sizeof(float) * (size_t)rows, (cudaStream_t)stream);
    HGB_LAUNCH_CHECK("pnaplus_conv_bwd");
    return HGB_OK;
  }
  const PnapLaunch L = pnap_launch(f, r, d, grads);
  const int grid = hgb_grid_for(n, L.warps, PNAP_BWD_MAX_BLOCKS);
  float* part = static_cast<float*>(workspace);
#define PNAP_BWD(NC)                                                                                                          \
  do {                                                                                                                        \
    cudaFuncSetAttribute(pnaplus_conv_bwd_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.bwd_smem);         \
    pnaplus_conv_bwd_kernel<NC><<<grid, L.warps * 32, L.bwd_smem, (cudaStream_t)stream>>>(                                    \
        g_out, pq, dist, rowptr, perm, src, eattr, d, freq, r, radius, expo, wr, br, wl, mr, mat, cvec, out, argmin, argmax, n, \
        f, g_p, ldgp, g_h, g_dist, g_eattr, grads, part);                                                                     \
  } while (0)
  if (f <= 32) PNAP_BWD(1);
  else PNAP_BWD(2);
#undef PNAP_BWD
  HGB_LAUNCH_CHECK("pnaplus_conv_bwd");
  if (grads) {
    pna_conv_reduce_kernel<<<hgb_grid_for(rows, 256), 256, 0, (cudaStream_t)stream>>>(part, grid, (int)rows, g_params);
    HGB_LAUNCH_CHECK("pnaplus_conv_reduce");
  }
  return HGB_OK;
}

// ---- CGConv (torch_geometric 2.6.1 CGConv(channels, dim, aggr="add", batch_norm=False, bias=True),
// hydragnn/models/CGCNNStack.py:60-80).  For the edge e = (j -> i), z_e = [x_i | x_j | a_e]:
//   m_e = sigmoid(W_f z_e + b_f) * softplus(W_s z_e + b_s),   out_i = x_i + sum_{e: target i} m_e.
// Both Linears are affine in the blocks of z, so with one per-node Linear [P_f | P_s | Q_f | Q_s] = x [A_f; A_s; B_f; B_s]^T
// the pre-activations are f_e = P_f[i] + Q_f[j] + C_f a_e + b_f (s_e alike) and are formed in registers: no [E, 2F + D] z,
// no [E, F] pre-activation and no message reach memory.
//
// Thread mapping: a group of G lanes owns one target node, G the power of two >= F up to 32, so a warp serves 32 / G targets
// at F <= 32 (at F = 1, the update_config shape without GPS, all 32 lanes work on 32 targets).  Above 32 a warp owns one
// target and lane l the channels l + 32 t, t < CPT.  A lane's channel set is fixed, so its sums run in CSR order (ascending
// edge id, as scatter_add_ does) with no atomics.  mt [d, 2F] and cvec [2F] are staged in shared memory once per CTA.
#define CGC_MAX_F 128
#define CGC_MAX_D 16
#define CGC_BWD_MAX_BLOCKS (HGB_NUM_SMS * 4)
#define CGC_BWD_WARPS 8

// torch's sigmoid and softplus (beta 1, threshold 20) with the accurate exp / log1p: the fp32 configs are held to fp64
__device__ __forceinline__ float cgc_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }
__device__ __forceinline__ float cgc_softplus(float z) { return z > 20.f ? z : log1pf(expf(z)); }

// f_e and s_e of the lane's channels cc[t] (clamped to f - 1 where the lane has no channel, so every load stays in range):
// base = P[i] + b per node, then + Q[j] + sum_k mt[k, .] a_e[k].  Forward and backward both call this, so the backward's
// softplus branch sees the forward's pre-activation bit for bit.
template <int CPT>
__device__ __forceinline__ void cgc_pre(const float* smt, int f, int d, const int (&cc)[CPT], const float (&bf)[CPT],
                                        const float (&bs)[CPT], const float* __restrict__ q, const float* __restrict__ a_row,
                                        float (&zf)[CPT], float (&zs)[CPT]) {
#pragma unroll
  for (int t = 0; t < CPT; ++t) {
    zf[t] = bf[t] + __ldg(q + cc[t]);
    zs[t] = bs[t] + __ldg(q + f + cc[t]);
  }
  for (int k = 0; k < d; ++k) {
    const float a = __ldg(a_row + k);
    const float* m = smt + k * 2 * f;
#pragma unroll
    for (int t = 0; t < CPT; ++t) {
      zf[t] = fmaf(m[cc[t]], a, zf[t]);
      zs[t] = fmaf(m[f + cc[t]], a, zs[t]);
    }
  }
}

__device__ __forceinline__ void cgc_stage(float* sm, const float* __restrict__ mt, const float* __restrict__ cvec, int f, int d) {
  const int nm = d * 2 * f;
  for (int t = threadIdx.x; t < nm + 2 * f; t += blockDim.x) sm[t] = t < nm ? __ldg(mt + t) : __ldg(cvec + t - nm);
}

template <int CPT>
__global__ void __launch_bounds__(256) cgconv_fwd_kernel(
    const float* __restrict__ pq, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm,
    const int32_t* __restrict__ src, const float* __restrict__ eattr, int d, const float* __restrict__ mt,
    const float* __restrict__ cvec, const float* __restrict__ x, int n, int f, int gl2, float* __restrict__ out) {
  extern __shared__ float cgc_sm[];
  const float* smt = cgc_sm;
  const float* scv = cgc_sm + d * 2 * f;
  cgc_stage(cgc_sm, mt, cvec, f, d);
  __syncthreads();
  const int sub = threadIdx.x & ((1 << gl2) - 1);
  const int gpb = blockDim.x >> gl2;
  const int64_t ld = 4 * (int64_t)f;
  int cc[CPT];
  bool ok[CPT];
#pragma unroll
  for (int t = 0; t < CPT; ++t) {
    ok[t] = sub + 32 * t < f;
    cc[t] = min(sub + 32 * t, f - 1);
  }
  for (int row = blockIdx.x * gpb + (threadIdx.x >> gl2); row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    float bf[CPT], bs[CPT], acc[CPT];
#pragma unroll
    for (int t = 0; t < CPT; ++t) {
      bf[t] = __ldg(pq + row * ld + cc[t]) + scv[cc[t]];
      bs[t] = __ldg(pq + row * ld + f + cc[t]) + scv[f + cc[t]];
      acc[t] = 0.f;
    }
    for (int p = lo; p < hi; ++p) {
      const int e = perm ? perm[p] : p;
      float zf[CPT], zs[CPT];
      cgc_pre<CPT>(smt, f, d, cc, bf, bs, pq + (int64_t)src[p] * ld + 2 * f, eattr + (int64_t)e * d, zf, zs);
#pragma unroll
      for (int t = 0; t < CPT; ++t) acc[t] += cgc_sigmoid(zf[t]) * cgc_softplus(zs[t]);
    }
#pragma unroll
    for (int t = 0; t < CPT; ++t)
      if (ok[t]) out[(int64_t)row * f + cc[t]] = acc[t] + __ldg(x + (int64_t)row * f + cc[t]);    // residual, as PyG adds it
  }
}

// Per edge, g = g_out[i]:  g_f = g softplus(s) sigma(f) (1 - sigma(f)),  g_s = g sigma(f) softplus'(s) with softplus'(s) = 1
// above the threshold and e^s / (e^s + 1) below (ATen's softplus_backward).  g_h [e, 2f] = [g_f | g_s] in edge order; g_p[i]
// its segment sum; g_eattr[e] = g_h mt^T (a fixed xor tree over the group) when non-NULL.  With part non-NULL the lane adds
// g_h and a_e g_h into its own shared slots (warp w, entry (k, half, t) at ((k * 2 + half) * CPT + t) * 32 + lane), which
// are then summed over the CTA's warps and groups in index order into part [gridDim.x, 1 + d, 2f].  The row loop and the
// edge loop are warp-uniform, so the g_eattr shuffles see every lane.
template <int CPT>
__global__ void __launch_bounds__(256) cgconv_bwd_kernel(
    const float* __restrict__ g_out, const float* __restrict__ pq, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ src, const float* __restrict__ eattr, int d,
    const float* __restrict__ mt, const float* __restrict__ cvec, int n, int f, int gl2, float* __restrict__ g_p, int ldgp,
    float* __restrict__ g_h, float* __restrict__ g_eattr, float* __restrict__ part) {
  extern __shared__ float cgc_sm[];
  const float* smt = cgc_sm;
  const float* scv = cgc_sm + d * 2 * f;
  float* sacc = cgc_sm + (d + 1) * 2 * f;
  const int slots = (d + 1) * 2 * CPT * 32;
  const int nwarps = blockDim.x >> 5;
  cgc_stage(cgc_sm, mt, cvec, f, d);
  if (part)
    for (int t = threadIdx.x; t < nwarps * slots; t += blockDim.x) sacc[t] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int G = 1 << gl2, sub = lane & (G - 1), gpw = 32 >> gl2;
  float* wacc = sacc + warp * slots + lane;
  const int64_t ld = 4 * (int64_t)f;
  int cc[CPT];
  bool ok[CPT];
#pragma unroll
  for (int t = 0; t < CPT; ++t) {
    ok[t] = sub + 32 * t < f;
    cc[t] = min(sub + 32 * t, f - 1);
  }
  for (int first = (blockIdx.x * nwarps + warp) * gpw; first < n; first += gridDim.x * nwarps * gpw) {
    const int row = first + (lane >> gl2);
    const bool rv = row < n;
    const int lo = rv ? rowptr[row] : 0, len = rv ? rowptr[row + 1] - lo : 0;
    const int maxlen = (int)__reduce_max_sync(0xffffffffu, (unsigned)len);
    float bf[CPT], bs[CPT], g[CPT], gpf[CPT], gps[CPT];
#pragma unroll
    for (int t = 0; t < CPT; ++t) {
      bf[t] = rv ? __ldg(pq + row * ld + cc[t]) + scv[cc[t]] : 0.f;
      bs[t] = rv ? __ldg(pq + row * ld + f + cc[t]) + scv[f + cc[t]] : 0.f;
      g[t] = (rv && ok[t]) ? __ldg(g_out + (int64_t)row * f + cc[t]) : 0.f;
      gpf[t] = gps[t] = 0.f;
    }
    for (int it = 0; it < maxlen; ++it) {
      const bool ev = it < len;
      const int p = lo + it;
      const int e = ev ? (perm ? perm[p] : p) : 0;
      const float* a_row = eattr + (int64_t)e * d;
      float gf[CPT], gs[CPT];
      if (ev) {
        float zf[CPT], zs[CPT];
        cgc_pre<CPT>(smt, f, d, cc, bf, bs, pq + (int64_t)src[p] * ld + 2 * f, a_row, zf, zs);
#pragma unroll
        for (int t = 0; t < CPT; ++t) {
          const float sg = cgc_sigmoid(zf[t]);
          float dsp = 1.f;
          if (!(zs[t] > 20.f)) {
            const float ez = expf(zs[t]);
            dsp = ez / (ez + 1.f);
          }
          gf[t] = g[t] * cgc_softplus(zs[t]) * (sg * (1.f - sg));
          gs[t] = g[t] * sg * dsp;
          gpf[t] += gf[t];
          gps[t] += gs[t];
          if (ok[t]) {
            g_h[(int64_t)e * 2 * f + cc[t]] = gf[t];
            g_h[(int64_t)e * 2 * f + f + cc[t]] = gs[t];
          }
        }
        if (part) {
#pragma unroll
          for (int t = 0; t < CPT; ++t) {
            wacc[(0 * CPT + t) * 32] += gf[t];
            wacc[(1 * CPT + t) * 32] += gs[t];
          }
          for (int k = 0; k < d; ++k) {
            const float a = __ldg(a_row + k);
#pragma unroll
            for (int t = 0; t < CPT; ++t) {
              float* s = wacc + ((k + 1) * 2 * CPT + t) * 32;
              s[0] = fmaf(a, gf[t], s[0]);
              s[CPT * 32] = fmaf(a, gs[t], s[CPT * 32]);
            }
          }
        }
      } else {
#pragma unroll
        for (int t = 0; t < CPT; ++t) gf[t] = gs[t] = 0.f;
      }
      if (g_eattr) {
        for (int k = 0; k < d; ++k) {
          const float* m = smt + k * 2 * f;
          float v = 0.f;
#pragma unroll
          for (int t = 0; t < CPT; ++t) v = fmaf(gf[t], m[cc[t]], fmaf(gs[t], m[f + cc[t]], v));
          for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (ev && sub == 0) g_eattr[(int64_t)e * d + k] = v;
        }
      }
    }
    if (rv) {
#pragma unroll
      for (int t = 0; t < CPT; ++t)
        if (ok[t]) {
          g_p[(int64_t)row * ldgp + cc[t]] = gpf[t];
          g_p[(int64_t)row * ldgp + f + cc[t]] = gps[t];
        }
    }
  }
  if (!part) return;
  __syncthreads();
  const int rows = (d + 1) * 2 * f;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    const int k = r / (2 * f), half = (r / f) & 1, c = r % f;
    const int slot = ((k * 2 + half) * CPT + (c >> 5)) * 32 + (c & 31);
    float s = 0.f;
    for (int w = 0; w < nwarps; ++w)
      for (int grp = 0; grp < gpw; ++grp) s += sacc[w * slots + slot + grp * G];
    part[(int64_t)blockIdx.x * rows + r] = s;
  }
}

namespace {
struct CgcLaunch {
  int cpt, gl2;
  size_t fwd_smem, bwd_smem;
};

// The backward always runs 8 warps: at the largest shape (f = 128, d = 16, CPT 4) the staged parameters and the 8 warps'
// accumulator slots take (17 * 256 + 8 * 17 * 2 * 4 * 32) * 4 = 156,672 bytes, within the 227 KB a CTA may opt into.
static_assert(((CGC_MAX_D + 1) * 2 * CGC_MAX_F + CGC_BWD_WARPS * (CGC_MAX_D + 1) * 2 * 4 * 32) * 4 <= 227 * 1024,
              "cgconv_bwd: the 8-warp shared memory must fit at every supported shape");

CgcLaunch cgc_launch(int f, int d, bool grads) {
  CgcLaunch L;
  L.cpt = f <= 32 ? 1 : (f <= 64 ? 2 : 4);
  L.gl2 = 0;
  while ((1 << L.gl2) < f && L.gl2 < 5) ++L.gl2;
  const size_t params = (size_t)(d + 1) * 2 * f;
  const size_t slots = grads ? (size_t)(d + 1) * 2 * L.cpt * 32 : 0;
  L.fwd_smem = params * 4;
  L.bwd_smem = (params + CGC_BWD_WARPS * slots) * 4;
  return L;
}
}  // namespace

extern "C" int hgb_cgconv_supported(int32_t f, int32_t d) { return f >= 1 && f <= CGC_MAX_F && d >= 0 && d <= CGC_MAX_D; }

extern "C" int64_t hgb_cgconv_workspace_bytes(int32_t f, int32_t d) {
  if (!hgb_cgconv_supported(f, d)) return -1;
  return (int64_t)CGC_BWD_MAX_BLOCKS * (d + 1) * 2 * f * (int64_t)sizeof(float);
}

#define CGC_CHECK_ARGS(name)                                                                                                 \
  HGB_REQUIRE(n >= 0 && e >= 0 && hgb_cgconv_supported(f, d),                                                               \
              name ": bad sizes (n %d, e %d, f %d, d %d; 1 <= f <= %d, 0 <= d <= %d)", n, e, f, d, CGC_MAX_F, CGC_MAX_D);      \
  HGB_REQUIRE(rowptr && (n == 0 || (pq && cvec)) && (e == 0 || src) && (d == 0 || (mt && (e == 0 || eattr))),               \
              name ": null argument")

extern "C" int hgb_cgconv_fwd(const float* pq, const int32_t* rowptr, const int32_t* perm, const int32_t* src, const float* eattr,
                              int32_t d, const float* mt, const float* cvec, const float* x, int32_t n, int32_t e, int32_t f,
                              float* out, hgb_stream_t stream) {
  CGC_CHECK_ARGS("cgconv_fwd");
  HGB_REQUIRE(n == 0 || (x && out), "cgconv_fwd: null argument");
  if (n == 0) return HGB_OK;
  if (e == 0) {                              // no messages: out = x
    cudaMemcpyAsync(out, x, sizeof(float) * (size_t)n * f, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    return cudaPeekAtLastError() == cudaSuccess ? HGB_OK : HGB_ECUDA;
  }
  const CgcLaunch L = cgc_launch(f, d, false);
  const int grid = hgb_grid_for(n, (256 >> L.gl2));
#define CGC_FWD(CPT)                                                                                                         \
  cgconv_fwd_kernel<CPT><<<grid, 256, L.fwd_smem, (cudaStream_t)stream>>>(pq, rowptr, perm, src, eattr, d, mt, cvec, x, n, f, \
                                                                          L.gl2, out)
  if (L.cpt == 1) CGC_FWD(1);
  else if (L.cpt == 2) CGC_FWD(2);
  else CGC_FWD(4);
#undef CGC_FWD
  HGB_LAUNCH_CHECK("cgconv_fwd");
  return HGB_OK;
}

extern "C" int hgb_cgconv_bwd(const float* g_out, const float* pq, const int32_t* rowptr, const int32_t* perm, const int32_t* src,
                              const float* eattr, int32_t d, const float* mt, const float* cvec, int32_t n, int32_t e, int32_t f,
                              float* g_p, int32_t ldgp, float* g_h, float* g_eattr, float* g_params, void* workspace,
                              hgb_stream_t stream) {
  CGC_CHECK_ARGS("cgconv_bwd");
  HGB_REQUIRE(ldgp >= 2 * f, "cgconv_bwd: ldgp %d < 2 f = %d", ldgp, 2 * f);
  HGB_REQUIRE((n == 0 || (g_out && g_p)) && (e == 0 || g_h), "cgconv_bwd: null argument");
  HGB_REQUIRE(!g_params || workspace, "cgconv_bwd: parameter gradients need the workspace");
  HGB_REQUIRE(!g_eattr || d > 0, "cgconv_bwd: g_eattr needs d > 0");
  const bool grads = g_params != nullptr;
  const int rows = (d + 1) * 2 * f;
  if (n == 0 || e == 0) {                    // no messages: every gradient the kernel writes is zero
    if (grads) cudaMemsetAsync(g_params, 0, sizeof(float) * (size_t)rows, (cudaStream_t)stream);
    if (n > 0) cudaMemset2DAsync(g_p, sizeof(float) * (size_t)ldgp, 0, sizeof(float) * 2 * (size_t)f, n, (cudaStream_t)stream);
    return cudaPeekAtLastError() == cudaSuccess ? HGB_OK : HGB_ECUDA;
  }
  const CgcLaunch L = cgc_launch(f, d, grads);
  const int grid = hgb_grid_for(n, CGC_BWD_WARPS * (32 >> L.gl2), CGC_BWD_MAX_BLOCKS);
  float* part = grads ? static_cast<float*>(workspace) : nullptr;
#define CGC_BWD(CPT)                                                                                                         \
  do {                                                                                                                       \
    cudaFuncSetAttribute(cgconv_bwd_kernel<CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.bwd_smem);             \
    cgconv_bwd_kernel<CPT><<<grid, CGC_BWD_WARPS * 32, L.bwd_smem, (cudaStream_t)stream>>>(                                        \
        g_out, pq, rowptr, perm, src, eattr, d, mt, cvec, n, f, L.gl2, g_p, ldgp, g_h, g_eattr, part);                       \
  } while (0)
  if (L.cpt == 1) CGC_BWD(1);
  else if (L.cpt == 2) CGC_BWD(2);
  else CGC_BWD(4);
#undef CGC_BWD
  HGB_LAUNCH_CHECK("cgconv_bwd");
  if (grads) {
    pna_conv_reduce_kernel<<<hgb_grid_for(rows, 256), 256, 0, (cudaStream_t)stream>>>(part, grid, rows, g_params);
    HGB_LAUNCH_CHECK("cgconv_reduce");
  }
  return HGB_OK;
}
