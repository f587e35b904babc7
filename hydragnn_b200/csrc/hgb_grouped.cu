// libhgb.so -- grouped dense layers for multi-branch decoding (hydragnn/models/Base.py:770-780 graph heads, :816-840 node heads,
// hydragnn/models/MultiTaskModelMP.py): every row (graph or atom) goes through the Linear of ITS dataset branch.  The reference
// loops over `dataset_name.unique()` with boolean masks (one host synchronisation and one set of small GEMMs per branch); here the
// rows are sorted by branch once (CSR over the branch ids, built on the device) and each layer is ONE launch of a grouped GEMM whose
// 64-row tiles pick their weight matrix by group:
//
//   fwd / dgrad   C[r, :] = act(A[r, :] op(W_g) + bias_g)      for r in [rowptr[g], rowptr[g+1])
//   wgrad         dW_g = sum_{r in g} dY[r, :]^T X[r, :],  db_g = sum_{r in g} dY[r, :]
//
// Exact fp32 FMAs (heads are small: 50 / 25 / 200-wide), no host read of the group sizes: the launch covers the worst case
// (ceil(M / 64) + groups tiles, strided over grid.y) and surplus tiles are skipped.
#include "hgb_common.cuh"

namespace {

constexpr int GBM = 64, GBN = 64, GBK = 16, GTM = 4, GTN = 4;

// tile -> (group, first row, rows) from the group offsets; returns false for surplus tiles
__device__ __forceinline__ bool locate_tile(const int32_t* __restrict__ rowptr, int groups, int tile, int& g, int& row0, int& rows) {
  int acc = 0;
  for (int q = 0; q < groups; ++q) {
    const int lo = rowptr[q], hi = rowptr[q + 1];
    const int nt = (hi - lo + GBM - 1) / GBM;
    if (tile < acc + nt) {
      g = q;
      row0 = lo + (tile - acc) * GBM;
      rows = min(GBM, hi - row0);
      return true;
    }
    acc += nt;
  }
  return false;
}

// TB = true : B_g(k, n) = w[g][n][k]  (forward, w [groups, n, k])
// TB = false: B_g(k, n) = w[g][k][n]  (data gradient: reduction over the layer's outputs, w [groups, k, n])
template <bool TB, bool PR>
__device__ __forceinline__ void grouped_rows_body(const float* __restrict__ a, int64_t lda, const float* __restrict__ w,
                                                  const float* __restrict__ bias, const int32_t* __restrict__ rowptr, int groups,
                                                  int tiles, int n, int k, int act, float act_param, float* __restrict__ c,
                                                  float* __restrict__ z, const float* __restrict__ slope) {
  __shared__ float As[GBK][GBM + 4];
  __shared__ float Bs[GBK][GBN + 4];
  const int tid = threadIdx.x, n0 = blockIdx.x * GBN;
  const int tx = tid % 16, ty = tid / 16;
  // tiles stride over grid.y, which holds at most 65,535 of them; each tile is summed as before
  for (int tile = blockIdx.y; tile < tiles; tile += gridDim.y) {
    int g, row0, rows;
    if (!locate_tile(rowptr, groups, tile, g, row0, rows)) continue;   // surplus tile (uniform across the block)
    const float* wg = w + (int64_t)g * n * k;
    float acc[GTM][GTN];
#pragma unroll
    for (int i = 0; i < GTM; ++i)
#pragma unroll
      for (int j = 0; j < GTN; ++j) acc[i][j] = 0.f;
    for (int kk = 0; kk < k; kk += GBK) {
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int l = tid + t * 256;
        const int ak = l % GBK, am = l / GBK;
        float v = 0.f;
        if (am < rows && kk + ak < k) v = a[(int64_t)(row0 + am) * lda + kk + ak];
        As[ak][am] = v;
        int bn, bk;
        if (TB) { bk = l % GBK; bn = l / GBK; } else { bn = l % GBN; bk = l / GBN; }
        float u = 0.f;
        if (n0 + bn < n && kk + bk < k) u = TB ? wg[(int64_t)(n0 + bn) * k + kk + bk] : wg[(int64_t)(kk + bk) * n + n0 + bn];
        Bs[bk][bn] = u;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < GBK; ++q) {
        float ra[GTM], rb[GTN];
#pragma unroll
        for (int i = 0; i < GTM; ++i) ra[i] = As[q][ty * GTM + i];
#pragma unroll
        for (int j = 0; j < GTN; ++j) rb[j] = Bs[q][tx * GTN + j];
#pragma unroll
        for (int i = 0; i < GTM; ++i)
#pragma unroll
          for (int j = 0; j < GTN; ++j) acc[i][j] = fmaf(ra[i], rb[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < GTM; ++i) {
      const int lm = ty * GTM + i;
      if (lm >= rows) continue;
#pragma unroll
      for (int j = 0; j < GTN; ++j) {
        const int gn = n0 + tx * GTN + j;
        if (gn >= n) continue;
        float v = acc[i][j];
        if (bias) v += bias[(int64_t)g * n + gn];
        if (z) z[(int64_t)(row0 + lm) * n + gn] = v;
        c[(int64_t)(row0 + lm) * n + gn] = hgb_epi_act<PR>(v, act, act_param, PR ? __ldg(slope) : 0.f);
      }
    }
  }
}

template <bool TB>
__global__ void __launch_bounds__(256) grouped_rows_kernel(const float* __restrict__ a, int64_t lda, const float* __restrict__ w,
                                                           const float* __restrict__ bias, const int32_t* __restrict__ rowptr,
                                                           int groups, int tiles, int n, int k, int act, float act_param,
                                                           float* __restrict__ c, float* __restrict__ z) {
  grouped_rows_body<TB, false>(a, lda, w, bias, rowptr, groups, tiles, n, k, act, act_param, c, z, nullptr);
}

// the forward (TB = true) with PReLU in the epilogue, slope read from device memory
__global__ void __launch_bounds__(256) grouped_rows_prelu_kernel(const float* __restrict__ a, int64_t lda, const float* __restrict__ w,
                                                                 const float* __restrict__ bias, const int32_t* __restrict__ rowptr,
                                                                 int groups, int tiles, int n, int k, float* __restrict__ c,
                                                                 float* __restrict__ z, const float* __restrict__ slope) {
  grouped_rows_body<true, true>(a, lda, w, bias, rowptr, groups, tiles, n, k, HGB_ACT_PRELU, 0.f, c, z, slope);
}

// dW_g[nn][kk] = sum_{r in g} dy[r][nn] x[r][kk];  grid = (ceil(k/64), ceil(n/64), groups)
__global__ void __launch_bounds__(256) grouped_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, int64_t ldx,
                                                            const int32_t* __restrict__ rowptr, int n, int k,
                                                            float* __restrict__ dw) {
  __shared__ float As[GBK][GBM + 4];   // dy^T tile: [row][out]
  __shared__ float Bs[GBK][GBN + 4];   // x tile:    [row][in]
  const int g = blockIdx.z;
  const int lo = rowptr[g], hi = rowptr[g + 1];
  const int tid = threadIdx.x, m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  const int tx = tid % 16, ty = tid / 16;
  float acc[GTM][GTN];
#pragma unroll
  for (int i = 0; i < GTM; ++i)
#pragma unroll
    for (int j = 0; j < GTN; ++j) acc[i][j] = 0.f;
  for (int r0 = lo; r0 < hi; r0 += GBK) {
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int l = tid + t * 256;
      const int am = l % GBM, ar = l / GBM;
      As[ar][am] = (r0 + ar < hi && m0 + am < n) ? dy[(int64_t)(r0 + ar) * n + m0 + am] : 0.f;
      const int bn = l % GBN, br = l / GBN;
      Bs[br][bn] = (r0 + br < hi && n0 + bn < k) ? x[(int64_t)(r0 + br) * ldx + n0 + bn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < GBK; ++q) {
      float ra[GTM], rb[GTN];
#pragma unroll
      for (int i = 0; i < GTM; ++i) ra[i] = As[q][ty * GTM + i];
#pragma unroll
      for (int j = 0; j < GTN; ++j) rb[j] = Bs[q][tx * GTN + j];
#pragma unroll
      for (int i = 0; i < GTM; ++i)
#pragma unroll
        for (int j = 0; j < GTN; ++j) acc[i][j] = fmaf(ra[i], rb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int gm = m0 + ty * GTM + i;
    if (gm >= n) continue;
#pragma unroll
    for (int j = 0; j < GTN; ++j) {
      const int gk = n0 + tx * GTN + j;
      if (gk < k) dw[((int64_t)g * n + gm) * k + gk] = acc[i][j];
    }
  }
}

// db_g[c] = sum_{r in g} dy[r][c]; one block per (group, 32 columns): 8 row-lanes x 32 columns, fixed-order tree
__global__ void grouped_colsum_kernel(const float* __restrict__ dy, const int32_t* __restrict__ rowptr, int n, float* __restrict__ db) {
  __shared__ float red[8][33];
  const int g = blockIdx.y, c = blockIdx.x * 32 + threadIdx.x;
  const int lo = rowptr[g], hi = rowptr[g + 1];
  float a = 0.f;
  if (c < n)
    for (int r = lo + threadIdx.y; r < hi; r += 8) a += dy[(int64_t)r * n + c];
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < n) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x];
    db[(int64_t)g * n + c] = t;
  }
}

}  // namespace

// y [m, n] = act(x [m, k] W_g^T + b_g) with w [groups, n, k] (trans_w = 0) or, for the data gradient, y [m, n] = x [m, k] W_g
// with w [groups, k, n] (trans_w = 1; bias / act must be off).  Rows are sorted by group: rowptr [groups + 1] (device).
extern "C" int hgb_grouped_linear(const float* x, int64_t ldx, const float* w, const float* bias, const int32_t* rowptr,
                                  int32_t groups, int32_t m, int32_t n, int32_t k, int32_t trans_w, int32_t act, float act_param,
                                  float* y, float* z, hgb_stream_t stream) {
  HGB_REQUIRE(x && w && rowptr && y && groups >= 1 && m >= 0 && n >= 1 && k >= 1 && ldx >= k, "grouped_linear: bad arguments");
  if (m == 0) return HGB_OK;
  const int tiles = (m + GBM - 1) / GBM + groups;
  dim3 grid((n + GBN - 1) / GBN, tiles < 65535 ? tiles : 65535);
  cudaStream_t st = (cudaStream_t)stream;
  if (trans_w) grouped_rows_kernel<false><<<grid, 256, 0, st>>>(x, ldx, w, bias, rowptr, groups, tiles, n, k, act, act_param, y, z);
  else grouped_rows_kernel<true><<<grid, 256, 0, st>>>(x, ldx, w, bias, rowptr, groups, tiles, n, k, act, act_param, y, z);
  HGB_LAUNCH_CHECK("grouped_linear");
  return HGB_OK;
}

extern "C" int hgb_grouped_linear_prelu(const float* x, int64_t ldx, const float* w, const float* bias, const int32_t* rowptr,
                                        int32_t groups, int32_t m, int32_t n, int32_t k, const float* slope, float* y, float* z,
                                        hgb_stream_t stream) {
  HGB_REQUIRE(x && w && rowptr && y && z && slope && groups >= 1 && m >= 0 && n >= 1 && k >= 1 && ldx >= k,
              "grouped_linear_prelu: bad arguments");
  if (m == 0) return HGB_OK;
  const int tiles = (m + GBM - 1) / GBM + groups;
  dim3 grid((n + GBN - 1) / GBN, tiles < 65535 ? tiles : 65535);
  grouped_rows_prelu_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, w, bias, rowptr, groups, tiles, n, k, y, z, slope);
  HGB_LAUNCH_CHECK("grouped_linear_prelu");
  return HGB_OK;
}

// dw [groups, n, k] = per-group dy^T x, db [groups, n] (optional) = per-group column sums of dy
extern "C" int hgb_grouped_wgrad(const float* dy, const float* x, int64_t ldx, const int32_t* rowptr, int32_t groups, int32_t m,
                                 int32_t n, int32_t k, float* dw, float* db, hgb_stream_t stream) {
  HGB_REQUIRE(dy && x && rowptr && dw && groups >= 1 && n >= 1 && k >= 1 && ldx >= k, "grouped_wgrad: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((k + GBN - 1) / GBN, (n + GBM - 1) / GBM, groups);
  grouped_wgrad_kernel<<<grid, 256, 0, st>>>(dy, x, ldx, rowptr, n, k, dw);
  HGB_LAUNCH_CHECK("grouped_wgrad");
  if (db) {
    grouped_colsum_kernel<<<dim3((n + 31) / 32, groups), dim3(32, 8), 0, st>>>(dy, rowptr, n, db);
    HGB_LAUNCH_CHECK("grouped_colsum");
  }
  return HGB_OK;
}
