// libhgb.so -- dense layers: generic fp32 GEMM (all transposes, split-K), fused linear+bias+act,
// activation backward, column sums.
//
// These are the fp32 "any shape" kernels used by every Linear on the path (M = nodes/edges/graphs is
// large, N and K are small: 1..192).  The bf16 tensor-core (wgmma) path for the hot shapes lives in
// hgb_tc_linear.cu; this file is the exact-fp32 path and the fallback for odd shapes.
#include "hgb_common.cuh"

#define BM 64
#define BN 64
#define BK 16
#define TM 4
#define TN 4

// C[m,n] (+)= sum_k A(m,k) B(k,n), A(m,k) = a[m*lda + k] or a[k*lda + m] (TA), same for B.
// grid.z = split-K slices; with splits > 1 each slice writes its partial to part[z, m, n].
// PR: PReLU epilogue with the slope at `slope` (gemm_prelu_kernel), else the runtime activation code (gemm_kernel)
template <bool TA, bool TB, bool PR>
__device__ __forceinline__ void gemm_body(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ c, int m,
                                          int n, int k, int64_t lda, int64_t ldb, int64_t ldc, int beta_one, int k_per_split,
                                          float* __restrict__ part, const float* __restrict__ bias, int act, float act_param,
                                          float* __restrict__ zout, const float* __restrict__ slope) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(k, kbeg + k_per_split);
  const int tx = tid % 16, ty = tid / 16;  // 16 x 16 threads, each TM x TN
  // row tiles stride over grid.y, which holds at most 65,535 of them (4,194,240 rows); each tile is summed as before
  for (int64_t mt = blockIdx.y; mt * BM < m; mt += gridDim.y) {
    const int m0 = (int)mt * BM;
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int kk = kbeg; kk < kend; kk += BK) {
      // load A tile (BM x BK) and B tile (BK x BN): 1024 elements each, 4 per thread
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int l = tid + t * 256;
        int am, ak;
        if (TA) { am = l % BM; ak = l / BM; } else { ak = l % BK; am = l / BK; }   // contiguous index fastest
        const int gm = m0 + am, gk = kk + ak;
        float v = 0.f;
        if (gm < m && gk < kend) v = TA ? a[(int64_t)gk * lda + gm] : a[(int64_t)gm * lda + gk];
        As[ak][am] = v;
        int bn, bk;
        if (TB) { bk = l % BK; bn = l / BK; } else { bn = l % BN; bk = l / BN; }
        const int gn = n0 + bn, gk2 = kk + bk;
        float w = 0.f;
        if (gn < n && gk2 < kend) w = TB ? b[(int64_t)gn * ldb + gk2] : b[(int64_t)gk2 * ldb + gn];
        Bs[bk][bn] = w;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < BK; ++q) {
        // one 16-byte shared-memory load per operand (TM = TN = 4; rows of As / Bs are 272 B apart: 16-byte aligned)
        const float4 a4 = *reinterpret_cast<const float4*>(&As[q][ty * TM]);
        const float4 b4 = *reinterpret_cast<const float4*>(&Bs[q][tx * TN]);
        const float ra[TM] = {a4.x, a4.y, a4.z, a4.w}, rb[TN] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(ra[i], rb[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int gm = m0 + ty * TM + i;
      if (gm >= m) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int gn = n0 + tx * TN + j;
        if (gn >= n) continue;
        if (part) {
          part[((int64_t)blockIdx.z * m + gm) * n + gn] = acc[i][j];
        } else {
          float v = acc[i][j];
          if (bias) v += bias[gn];
          if (zout) zout[(int64_t)gm * ldc + gn] = v;
          v = hgb_epi_act<PR>(v, act, act_param, PR ? __ldg(slope) : 0.f);
          if (beta_one) v += c[(int64_t)gm * ldc + gn];
          c[(int64_t)gm * ldc + gn] = v;
        }
      }
    }
  }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) gemm_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                   float* __restrict__ c, int m, int n, int k, int64_t lda, int64_t ldb,
                                                   int64_t ldc, int beta_one, int k_per_split, float* __restrict__ part,
                                                   const float* __restrict__ bias, int act, float act_param,
                                                   float* __restrict__ zout) {
  gemm_body<TA, TB, false>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, k_per_split, part, bias, act, act_param, zout, nullptr);
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) gemm_prelu_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                         float* __restrict__ c, int m, int n, int k, int64_t lda, int64_t ldb,
                                                         int64_t ldc, const float* __restrict__ bias, float* __restrict__ zout,
                                                         const float* __restrict__ slope) {
  gemm_body<TA, TB, true>(a, b, c, m, n, k, lda, ldb, ldc, 0, k, nullptr, bias, HGB_ACT_PRELU, 0.f, zout, slope);
}

// c[i] (+)= sum over split-K slices of part[s, i].  blockDim = (32, 8): x = output element, y = slice group (slices y, y+8, ...);
// the 8 group sums are added in a fixed order, so the result does not depend on scheduling.
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int64_t mn, int n, int64_t ldc,
                                     int beta_one, float* __restrict__ c) {
  __shared__ float red[8][33];
  for (int64_t base = (int64_t)blockIdx.x * 32; base < mn; base += (int64_t)gridDim.x * 32) {
    const int64_t i = base + threadIdx.x;
    float acc = 0.f;
    if (i < mn)
      for (int s = threadIdx.y; s < splits; s += 8) acc += part[(int64_t)s * mn + i];
    red[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && i < mn) {
      float t = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x];
      const int64_t o = (i / n) * ldc + (i % n);
      c[o] = beta_one ? c[o] + t : t;
    }
    __syncthreads();
  }
}

// ---- weight-gradient form with a long reduction:  C[mo, no] = sum_r A[r, mo]^T B[r, no],  r up to 10^6 rows ----------------------
// The generic kernel above splits K over hundreds of tiny CTAs (64 x 64 x 16 tiles, 4 x 4 register tiles: 2 FMA per shared-memory
// word).  Here every CTA streams 128-row chunks of both operands through shared memory with cp.async, keeps the WHOLE [mo, no]
// result in registers as 8 x 8 tiles (the (mo/8)(no/8) tiles take that many threads; the 128 threads form NSL slices of the chunk's
// rows), and writes one partial per (CTA, slice); a fixed-order reduce finishes.  Exact fp32 FMAs.
constexpr int TNF_ROWS = 64, TNF_THREADS = 128;      // rows per pipeline stage; two stages are in flight (cp.async double buffer)

__device__ __forceinline__ void tnf_cp16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}

__global__ void __launch_bounds__(TNF_THREADS) gemm_tn_fast_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                   int64_t lda, int64_t ldb, int r_total, int mo, int no,
                                                                   int chunks_per_cta, float* __restrict__ part) {
  extern __shared__ __align__(16) float tnf_smem[];
  const int stage_floats = TNF_ROWS * (mo + no);
  const int t = threadIdx.x;
  const int tps = (mo / 8) * (no / 8), nsl = TNF_THREADS / tps, ksl = TNF_ROWS / nsl;
  const int slice = t / tps, tt = t % tps;
  const int m0 = (tt / (no / 8)) * 8, n0 = (tt % (no / 8)) * 8;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int nchunks = (r_total + TNF_ROWS - 1) / TNF_ROWS;
  const int c_beg = blockIdx.x * chunks_per_cta, c_end = min(nchunks, c_beg + chunks_per_cta);
  const int ca = mo / 4, cb = no / 4;
  auto issue = [&](int ch, int buf) {
    float* sa = tnf_smem + buf * stage_floats;
    float* sb = sa + TNF_ROWS * mo;
    const int row0 = ch * TNF_ROWS;
    for (int i = t; i < TNF_ROWS * ca; i += TNF_THREADS) {
      const int r = i / ca, c4 = i - r * ca;
      float* dst = sa + r * mo + 4 * c4;
      if (row0 + r < r_total) tnf_cp16(dst, a + (int64_t)(row0 + r) * lda + 4 * c4);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int i = t; i < TNF_ROWS * cb; i += TNF_THREADS) {
      const int r = i / cb, c4 = i - r * cb;
      float* dst = sb + r * no + 4 * c4;
      if (row0 + r < r_total) tnf_cp16(dst, b + (int64_t)(row0 + r) * ldb + 4 * c4);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (c_beg < c_end) issue(c_beg, 0);
  for (int ch = c_beg; ch < c_end; ++ch) {
    const int buf = (ch - c_beg) & 1;
    if (ch + 1 < c_end) {
      issue(ch + 1, buf ^ 1);                       // the other buffer was released by the barrier at the end of the last iteration
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float* sa = tnf_smem + buf * stage_floats;
    const float* sb = sa + TNF_ROWS * mo;
#pragma unroll 4
    for (int kk = 0; kk < ksl; ++kk) {
      const int k = slice * ksl + kk;
      const float4 a0 = *reinterpret_cast<const float4*>(sa + k * mo + m0);
      const float4 a1 = *reinterpret_cast<const float4*>(sa + k * mo + m0 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(sb + k * no + n0);
      const float4 b1 = *reinterpret_cast<const float4*>(sb + k * no + n0 + 4);
      const float ra[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float rb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(ra[i], rb[j], acc[i][j]);
    }
    __syncthreads();                                // everyone is done with `buf` before the next iteration refills it
  }
  float* out = part + ((int64_t)blockIdx.x * nsl + slice) * mo * no;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    *reinterpret_cast<float4*>(out + (m0 + i) * no + n0) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    *reinterpret_cast<float4*>(out + (m0 + i) * no + n0 + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
  }
}

static bool tn_fast_ok(int m, int n, int k, int64_t lda, int64_t ldb, const void* a, const void* b) {
  if (k < 8192 || m % 8 || n % 8 || lda % 4 || ldb % 4) return false;
  if (((uintptr_t)a % 16) || ((uintptr_t)b % 16)) return false;
  const int tps = (m / 8) * (n / 8);
  if (tps < 1 || tps > TNF_THREADS || (TNF_THREADS % tps) != 0) return false;
  return (size_t)2 * TNF_ROWS * (m + n) * 4 <= 160 * 1024 && (TNF_ROWS % (TNF_THREADS / tps)) == 0;
}
static int tn_fast_grid(int k) {
  const int nchunks = (k + TNF_ROWS - 1) / TNF_ROWS;
  return nchunks < HGB_NUM_SMS * 3 ? nchunks : HGB_NUM_SMS * 3;
}

static int pick_splits(int m, int n, int k) {
  const int tiles = ((m + BM - 1) / BM) * ((n + BN - 1) / BN);
  if (tiles >= HGB_NUM_SMS || k < 4096) return 1;
  int s = (HGB_NUM_SMS * 4 + tiles - 1) / tiles;
  const int maxs = (k + 63) / 64;
  if (s > maxs) s = maxs;
  return s < 1 ? 1 : s;
}

extern "C" int64_t hgb_gemm_workspace_bytes(int32_t m, int32_t n, int32_t k, int32_t trans_a) {
  const int s = pick_splits(m, n, k);
  int64_t bytes = s > 1 ? (int64_t)s * m * n * 4 : 0;
  if (trans_a && m % 8 == 0 && n % 8 == 0 && m > 0 && n > 0) {
    const int tps = (m / 8) * (n / 8);
    if (tps >= 1 && tps <= TNF_THREADS && TNF_THREADS % tps == 0) {
      const int64_t fast = (int64_t)tn_fast_grid(k) * (TNF_THREADS / tps) * m * n * 4;
      if (fast > bytes) bytes = fast;
    }
  }
  return bytes;
}

template <bool TA, bool TB>
static int launch_gemm(const float* a, const float* b, float* c, int m, int n, int k, int64_t lda, int64_t ldb, int64_t ldc,
                       int beta_one, void* ws, int64_t ws_bytes, const float* bias, int act, float act_param, float* z,
                       cudaStream_t st) {
  int splits = (bias || act || z) ? 1 : pick_splits(m, n, k);
  if (splits > 1 && ((int64_t)splits * m * n * 4 > ws_bytes || !ws)) splits = 1;
  int kps = (k + splits - 1) / splits;
  kps = ((kps + BK - 1) / BK) * BK;
  splits = (k + kps - 1) / kps;
  if (splits < 1) splits = 1;
  const int mtiles = (m + BM - 1) / BM;
  dim3 grid((n + BN - 1) / BN, mtiles < 65535 ? mtiles : 65535, splits);
  gemm_kernel<TA, TB><<<grid, 256, 0, st>>>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, kps, splits > 1 ? (float*)ws : nullptr,
                                            bias, act, act_param, z);
  HGB_LAUNCH_CHECK("gemm");
  if (splits > 1) {
    splitk_reduce_kernel<<<hgb_grid_for((int64_t)m * n, 32), dim3(32, 8), 0, st>>>((const float*)ws, splits, (int64_t)m * n, n, ldc,
                                                                            beta_one, c);
    HGB_LAUNCH_CHECK("splitk_reduce");
  }
  return HGB_OK;
}

extern "C" int hgb_gemm(const float* a, const float* b, float* c, int32_t m, int32_t n, int32_t k, int32_t trans_a,
                        int32_t trans_b, int64_t lda, int64_t ldb, int64_t ldc, int32_t beta_one, void* workspace,
                        int64_t workspace_bytes, hgb_stream_t stream) {
  HGB_REQUIRE(m >= 0 && n >= 0 && k >= 0 && c, "gemm: bad arguments");
  if (m == 0 || n == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (k == 0) {
    if (!beta_one) cudaMemset2DAsync(c, ldc * 4, 0, (size_t)n * 4, m, st);
    return HGB_OK;
  }
  if (trans_a && trans_b) return launch_gemm<true, true>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, workspace, workspace_bytes, nullptr, 0, 0.f, nullptr, st);
  if (trans_a && tn_fast_ok(m, n, k, lda, ldb, a, b)) {
    const int tps = (m / 8) * (n / 8), nsl = TNF_THREADS / tps;
    const int grid0 = tn_fast_grid(k);
    if (workspace && workspace_bytes >= (int64_t)grid0 * nsl * m * n * 4) {
      const int nchunks = (k + TNF_ROWS - 1) / TNF_ROWS;
      const int cpc = (nchunks + grid0 - 1) / grid0;
      const int grid = (nchunks + cpc - 1) / cpc;
      const size_t smem = (size_t)2 * TNF_ROWS * (m + n) * 4;
      cudaFuncSetAttribute(gemm_tn_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      gemm_tn_fast_kernel<<<grid, TNF_THREADS, smem, st>>>(a, b, lda, ldb, k, m, n, cpc, (float*)workspace);
      HGB_LAUNCH_CHECK("gemm_tn_fast");
      splitk_reduce_kernel<<<hgb_grid_for((int64_t)m * n, 32), dim3(32, 8), 0, st>>>((const float*)workspace, grid * nsl, (int64_t)m * n, n,
                                                                              ldc, beta_one, c);
      HGB_LAUNCH_CHECK("splitk_reduce");
      return HGB_OK;
    }
  }
  if (trans_a) return launch_gemm<true, false>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, workspace, workspace_bytes, nullptr, 0, 0.f, nullptr, st);
  if (trans_b) return launch_gemm<false, true>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, workspace, workspace_bytes, nullptr, 0, 0.f, nullptr, st);
  return launch_gemm<false, false>(a, b, c, m, n, k, lda, ldb, ldc, beta_one, workspace, workspace_bytes, nullptr, 0, 0.f, nullptr, st);
}

extern "C" int hgb_linear_fwd(const float* x, const float* w, const float* b, int32_t m, int32_t n, int32_t k, int64_t ldx,
                              int64_t ldw, int32_t act, float act_param, float* y, float* z, hgb_stream_t stream) {
  HGB_REQUIRE(m >= 0 && n > 0 && k > 0 && x && w && y && ldx >= k && ldw >= k, "linear_fwd: bad arguments");
  if (m == 0) return HGB_OK;
  return launch_gemm<false, true>(x, w, y, m, n, k, ldx, ldw, n, 0, nullptr, 0, b, act, act_param, z, (cudaStream_t)stream);
}

extern "C" int hgb_linear_fwd_prelu(const float* x, const float* w, const float* b, int32_t m, int32_t n, int32_t k, int64_t ldx,
                                    int64_t ldw, const float* slope, float* y, float* z, hgb_stream_t stream) {
  HGB_REQUIRE(m >= 0 && n > 0 && k > 0 && x && w && y && z && slope && ldx >= k && ldw >= k, "linear_fwd_prelu: bad arguments");
  if (m == 0) return HGB_OK;
  const int mtiles = (m + BM - 1) / BM;
  dim3 grid((n + BN - 1) / BN, mtiles < 65535 ? mtiles : 65535, 1);      // one k slice: the epilogue needs the whole sum
  gemm_prelu_kernel<false, true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, y, m, n, k, ldx, ldw, n, b, z, slope);
  HGB_LAUNCH_CHECK("linear_fwd_prelu");
  return HGB_OK;
}

// ---- activation derivative kernels -----------------------------------------------------------------
__global__ void act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                               int64_t count, int act, float p, float* __restrict__ dz) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    dz[i] = act == HGB_ACT_RELU_SELECT ? hgb_relu_select(dy[i], y[i]) : dy[i] * hgb_act_grad(y ? y[i] : 0.f, z ? z[i] : 0.f, act, p);
}

extern "C" int hgb_act_bwd(const float* dy, const float* y, const float* z, int64_t count, int32_t act, float act_param,
                           float* dz, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && dy && dz, "act_bwd: bad arguments");
  HGB_REQUIRE((act != HGB_ACT_SILU && act != HGB_ACT_DERIV) || z, "act_bwd: SiLU needs the pre-activation z (HGB_ACT_DERIV: the stored derivative)");
  HGB_REQUIRE(act == HGB_ACT_SILU || act == HGB_ACT_DERIV || act == HGB_ACT_NONE || y, "act_bwd: needs the activation output y");
  if (count == 0) return HGB_OK;
  act_bwd_kernel<<<hgb_grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>(dy, y, z, count, act, act_param, dz);
  HGB_LAUNCH_CHECK("act_bwd");
  return HGB_OK;
}

// value (order 0) / first / second derivative of the activation at x
__device__ __forceinline__ float act_deriv(float x, int act, float p, int order) {
  if (order == 0) return hgb_act(x, act, p);
  const float a = 1.6732632423543772848170429916717f, sc = 1.0507009873554804934193349852946f;
  switch (act) {
    case HGB_ACT_RELU: return order == 1 ? (x > 0.f ? 1.f : 0.f) : 0.f;
    case HGB_ACT_LRELU: return order == 1 ? (x > 0.f ? 1.f : p) : 0.f;
    case HGB_ACT_SILU: {
      float s = hgb_sigmoid(x);
      if (order == 1) return s * (1.f + x * (1.f - s));
      return s * (1.f - s) * (2.f + x * (1.f - 2.f * s));
    }
    case HGB_ACT_TANH: {
      float t = tanhf(x);
      return order == 1 ? 1.f - t * t : -2.f * t * (1.f - t * t);
    }
    case HGB_ACT_SIGMOID: {
      float s = hgb_sigmoid(x);
      return order == 1 ? s * (1.f - s) : s * (1.f - s) * (1.f - 2.f * s);
    }
    case HGB_ACT_ELU: return x > 0.f ? (order == 1 ? 1.f : 0.f) : __expf(x);
    case HGB_ACT_SELU: return x > 0.f ? (order == 1 ? sc : 0.f) : sc * a * __expf(x);
    default: return order == 1 ? 1.f : 0.f;
  }
}

__global__ void act_deriv_kernel(const float* __restrict__ x, int64_t count, int act, float p, int order,
                                 float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = act_deriv(x[i], act, p, order);
}

extern "C" int hgb_act_deriv(const float* x, int64_t count, int32_t act, float act_param, int32_t order, float* out,
                             hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && x && out && order >= 0 && order <= 2, "act_deriv: bad arguments");
  if (count == 0) return HGB_OK;
  act_deriv_kernel<<<hgb_grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>(x, count, act, act_param, order, out);
  HGB_LAUNCH_CHECK("act_deriv");
  return HGB_OK;
}

// ---- column sums (bias gradients): two deterministic stages -------------------------------------
#define CS_ROWS 512  // rows per block in stage 1
__global__ void colsum_stage1(const float* __restrict__ x, int m, int n, float* __restrict__ part) {
  // block (32 x 8): lanes over columns, 8 row-walkers; partial [row block, n].  Row blocks stride over grid.y (at most 65,535).
  __shared__ float sm[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int nb = (m + CS_ROWS - 1) / CS_ROWS;
  for (int rb = blockIdx.y; rb < nb; rb += gridDim.y) {
    const int r0 = rb * CS_ROWS;
    const int r1 = min(m, r0 + CS_ROWS);
    float acc = 0.f;
    if (col < n)
      for (int r = r0 + threadIdx.y; r < r1; r += 8) acc += x[(int64_t)r * n + col];
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && col < n) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
      part[(int64_t)rb * n + col] = t;
    }
    __syncthreads();
  }
}
__global__ void colsum_stage2(const float* __restrict__ part, int nb, int n, float* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= n) return;
  float acc = 0.f;
  for (int b = 0; b < nb; ++b) acc += part[(int64_t)b * n + col];
  out[col] = acc;
}

extern "C" int64_t hgb_colsum_workspace_bytes(int32_t m, int32_t n) {
  return (int64_t)((m + CS_ROWS - 1) / CS_ROWS + 1) * n * 4;
}

extern "C" int hgb_colsum(const float* x, int32_t m, int32_t n, float* out, void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(m >= 0 && n > 0 && out && workspace, "colsum: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (m == 0) {
    cudaMemsetAsync(out, 0, (size_t)n * 4, st);
    return HGB_OK;
  }
  const int nb = (m + CS_ROWS - 1) / CS_ROWS;
  colsum_stage1<<<dim3((n + 31) / 32, nb < 65535 ? nb : 65535), dim3(32, 8), 0, st>>>(x, m, n, (float*)workspace);
  HGB_LAUNCH_CHECK("colsum_stage1");
  colsum_stage2<<<(n + 127) / 128, 128, 0, st>>>((const float*)workspace, nb, n, out);
  HGB_LAUNCH_CHECK("colsum_stage2");
  return HGB_OK;
}

// ---- tiny-K linear layers (K <= 8) ----------------------------------------------------------------------------
// The reference runs its first PaiNN / PNAEq layer at node_size = input_dim (often 1, quirk Q4), so Linear(1 -> F),
// Linear(2 -> 1), Linear(1 -> 3) ... appear at M = nodes (or 3*nodes).  They are outer products / column sums,
// purely HBM-bound; a tiled GEMM wastes almost all of its work on them.
#define SK_KMAX 8
#define SK_NPT 8   // outputs per lane -> n <= 256

template <bool PR>
__device__ __forceinline__ void linear_smallk_fwd_body(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w,
                                                       int64_t ldw, const float* __restrict__ b, int64_t total, int n, int k, int act,
                                                       float ap, float* __restrict__ y, float* __restrict__ z,
                                                       const float* __restrict__ slope) {
  extern __shared__ float sw[];  // [n][k] + [n]
  for (int i = threadIdx.x; i < n * k; i += blockDim.x) sw[i] = w[(int64_t)(i / k) * ldw + (i % k)];
  for (int i = threadIdx.x; i < n; i += blockDim.x) sw[n * k + i] = b ? b[i] : 0.f;
  __syncthreads();
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / n;
    const int c = (int)(t - r * n);
    float acc = sw[n * k + c];
    for (int q = 0; q < k; ++q) acc = fmaf(__ldg(x + r * ldx + q), sw[c * k + q], acc);
    if (z) z[t] = acc;
    y[t] = hgb_epi_act<PR>(acc, act, ap, PR ? __ldg(slope) : 0.f);
  }
}

__global__ void linear_smallk_fwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, int64_t ldw,
                                         const float* __restrict__ b, int64_t total, int n, int k, int act, float ap,
                                         float* __restrict__ y, float* __restrict__ z) {
  linear_smallk_fwd_body<false>(x, ldx, w, ldw, b, total, n, k, act, ap, y, z, nullptr);
}

__global__ void linear_smallk_fwd_prelu_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, int64_t ldw,
                                               const float* __restrict__ b, int64_t total, int n, int k, float* __restrict__ y,
                                               float* __restrict__ z, const float* __restrict__ slope) {
  linear_smallk_fwd_body<true>(x, ldx, w, ldw, b, total, n, k, HGB_ACT_PRELU, 0.f, y, z, slope);
}

// n % 4 == 0: a thread owns four consecutive output columns of a row (16-byte stores), its weights live in registers, rows are
// walked with a 2-D block (x: column group, y: row) -- no index division, no shared memory.
template <int KT, bool PR>
__device__ __forceinline__ void linear_smallk_fwd_vec4_body(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w,
                                                            int64_t ldw, const float* __restrict__ b, int m, int n, int k, int act,
                                                            float ap, float* __restrict__ y, float* __restrict__ z,
                                                            const float* __restrict__ slope) {
  const int c0 = threadIdx.x * 4;
  const float sl = PR ? __ldg(slope) : 0.f;
  float wr[4][KT], bias[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    bias[j] = b ? b[c0 + j] : 0.f;
#pragma unroll
    for (int q = 0; q < KT; ++q) wr[j][q] = q < k ? w[(int64_t)(c0 + j) * ldw + q] : 0.f;
  }
  for (int r = blockIdx.x * blockDim.y + threadIdx.y; r < m; r += gridDim.x * blockDim.y) {
    float xr[KT];
#pragma unroll
    for (int q = 0; q < KT; ++q) xr[q] = q < k ? __ldg(x + (int64_t)r * ldx + q) : 0.f;
    float acc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc[j] = bias[j];
#pragma unroll
      for (int q = 0; q < KT; ++q) acc[j] = fmaf(xr[q], wr[j][q], acc[j]);
    }
    const int64_t o = (int64_t)r * n + c0;
    if (z) *reinterpret_cast<float4*>(z + o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(y + o) = make_float4(hgb_epi_act<PR>(acc[0], act, ap, sl), hgb_epi_act<PR>(acc[1], act, ap, sl),
                                                    hgb_epi_act<PR>(acc[2], act, ap, sl), hgb_epi_act<PR>(acc[3], act, ap, sl));
  }
}

template <int KT>
__global__ void linear_smallk_fwd_vec4_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, int64_t ldw,
                                              const float* __restrict__ b, int m, int n, int k, int act, float ap,
                                              float* __restrict__ y, float* __restrict__ z) {
  linear_smallk_fwd_vec4_body<KT, false>(x, ldx, w, ldw, b, m, n, k, act, ap, y, z, nullptr);
}

template <int KT>
__global__ void linear_smallk_fwd_vec4_prelu_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w,
                                                    int64_t ldw, const float* __restrict__ b, int m, int n, int k,
                                                    float* __restrict__ y, float* __restrict__ z, const float* __restrict__ slope) {
  linear_smallk_fwd_vec4_body<KT, true>(x, ldx, w, ldw, b, m, n, k, HGB_ACT_PRELU, 0.f, y, z, slope);
}

// one pass over (dy, y|z, x): dz = dy * act'(.), dx[m,k] = dz . W, partial dW / db per block.
// KT = compile-time bound on k (1,2,4,8), NPT = outputs per lane (n <= 32*NPT): only the needed work is generated.
#define SK_RU 4   // rows per walker trip: independent loads / shuffles hide the latency
template <int KT, int NPT>
__global__ void __launch_bounds__(256)
linear_smallk_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                         const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, int64_t ldw, int m, int n, int k,
                         int act, float ap, int rows_per_block, float* __restrict__ dx, float* __restrict__ part) {
  __shared__ float red[8 * 32];
  const int lane = threadIdx.x, walker = threadIdx.y;
  float wr[NPT][KT], gw[NPT][KT + 1];
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const int c = lane + 32 * j;
#pragma unroll
    for (int q = 0; q < KT; ++q) { wr[j][q] = (c < n && q < k) ? w[(int64_t)c * ldw + q] : 0.f; gw[j][q] = 0.f; }
    gw[j][KT] = 0.f;
  }
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(m, r0 + rows_per_block);
  for (int rb = r0 + walker * SK_RU; rb < r1; rb += 8 * SK_RU) {
    float xr[SK_RU][KT], dxp[SK_RU][KT], g[SK_RU][NPT];
#pragma unroll
    for (int u = 0; u < SK_RU; ++u) {
      const int r = rb + u;
      const bool live = r < r1;
#pragma unroll
      for (int q = 0; q < KT; ++q) { xr[u][q] = (live && q < k) ? __ldg(x + (int64_t)r * ldx + q) : 0.f; dxp[u][q] = 0.f; }
#pragma unroll
      for (int j = 0; j < NPT; ++j) {
        const int c = lane + 32 * j;
        const int64_t o = (int64_t)r * n + c;
        g[u][j] = (live && c < n) ? __ldg(dy + o) : 0.f;
        if (act != HGB_ACT_NONE && live && c < n) g[u][j] *= hgb_act_grad(y ? __ldg(y + o) : 0.f, z ? __ldg(z + o) : 0.f, act, ap);
      }
    }
#pragma unroll
    for (int u = 0; u < SK_RU; ++u)
#pragma unroll
      for (int j = 0; j < NPT; ++j) {
        gw[j][KT] += g[u][j];
#pragma unroll
        for (int q = 0; q < KT; ++q) {
          gw[j][q] = fmaf(g[u][j], xr[u][q], gw[j][q]);
          dxp[u][q] = fmaf(g[u][j], wr[j][q], dxp[u][q]);
        }
      }
    if (dx) {
#pragma unroll
      for (int u = 0; u < SK_RU; ++u)
#pragma unroll
        for (int q = 0; q < KT; ++q) {
          const float sum = hgb_warp_sum(dxp[u][q]);
          if (lane == 0 && q < k && rb + u < r1) dx[(int64_t)(rb + u) * k + q] = sum;
        }
    }
  }
  // reduce the 8 row walkers -> part[blockIdx.x][n][k+1]
  float* mypart = part + (int64_t)blockIdx.x * n * (k + 1);
#pragma unroll
  for (int j = 0; j < NPT; ++j)
#pragma unroll
    for (int q = 0; q <= KT; ++q) {
      if (q < k || q == KT) {   // uniform across the block
        __syncthreads();
        red[walker * 32 + lane] = gw[j][q];
        __syncthreads();
        if (walker == 0) {
          float acc = 0.f;
#pragma unroll
          for (int w8 = 0; w8 < 8; ++w8) acc += red[w8 * 32 + lane];
          const int c = lane + 32 * j;
          if (c < n) mypart[c * (k + 1) + (q == KT ? k : q)] = acc;
        }
      }
    }
}

// out[i] = sum_b part[b][i]: 32 outputs x 8 partial-walkers per block, fixed summation order (deterministic)
__global__ void linear_smallk_reduce_kernel(const float* __restrict__ part, int nblocks, int n, int k, float* __restrict__ dw,
                                            int64_t lddw, float* __restrict__ db) {
  __shared__ float red[8][33];
  const int cnt = n * (k + 1);
  const int i = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (i < cnt) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;   // four independent load chains
    int b = threadIdx.y;
    for (; b + 24 < nblocks; b += 32) {
      a0 += part[(size_t)b * cnt + i]; a1 += part[(size_t)(b + 8) * cnt + i];
      a2 += part[(size_t)(b + 16) * cnt + i]; a3 += part[(size_t)(b + 24) * cnt + i];
    }
    for (; b < nblocks; b += 8) a0 += part[(size_t)b * cnt + i];
    acc = (a0 + a1) + (a2 + a3);
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && i < cnt) {
    float t = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][threadIdx.x];
    const int r = i / (k + 1), c = i % (k + 1);
    if (c == k) { if (db) db[r] = t; } else if (dw) dw[(int64_t)r * lddw + c] = t;
  }
}

// n <= 8 as well: one thread per row keeps the whole n x (k+1) gradient tile in registers
#define SK_NMAX 8
__global__ void __launch_bounds__(256)
linear_tiny_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                       const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, int64_t ldw, int m, int n, int k,
                       int act, float ap, int rows_per_block, float* __restrict__ dx, float* __restrict__ part) {
  __shared__ float sw[SK_NMAX * SK_KMAX];
  __shared__ float red[8];
  for (int i = threadIdx.x; i < n * k; i += blockDim.x) sw[i] = w[(int64_t)(i / k) * ldw + (i % k)];
  __syncthreads();
  float gw[SK_NMAX][SK_KMAX + 1];
#pragma unroll
  for (int j = 0; j < SK_NMAX; ++j)
#pragma unroll
    for (int q = 0; q <= SK_KMAX; ++q) gw[j][q] = 0.f;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(m, r0 + rows_per_block);
  for (int r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
    float xr[SK_KMAX], dxr[SK_KMAX];
#pragma unroll
    for (int q = 0; q < SK_KMAX; ++q) { xr[q] = q < k ? x[(int64_t)r * ldx + q] : 0.f; dxr[q] = 0.f; }
#pragma unroll
    for (int j = 0; j < SK_NMAX; ++j)
      if (j < n) {
        const int64_t o = (int64_t)r * n + j;
        float g = dy[o];
        if (act != HGB_ACT_NONE) g *= hgb_act_grad(y ? y[o] : 0.f, z ? z[o] : 0.f, act, ap);
        gw[j][SK_KMAX] += g;
#pragma unroll
        for (int q = 0; q < SK_KMAX; ++q)
          if (q < k) { gw[j][q] = fmaf(g, xr[q], gw[j][q]); dxr[q] = fmaf(g, sw[j * k + q], dxr[q]); }
      }
    if (dx) {
#pragma unroll
      for (int q = 0; q < SK_KMAX; ++q)
        if (q < k) dx[(int64_t)r * k + q] = dxr[q];
    }
  }
  float* mypart = part + (int64_t)blockIdx.x * n * (k + 1);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < SK_NMAX; ++j)
#pragma unroll
    for (int q = 0; q <= SK_KMAX; ++q)
      if (j < n && (q < k || q == SK_KMAX)) {
        const float v = hgb_warp_sum(gw[j][q]);
        __syncthreads();
        if (lane == 0) red[warp] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
          float t = 0.f;
#pragma unroll
          for (int w8 = 0; w8 < 8; ++w8) t += red[w8];
          mypart[j * (k + 1) + (q == SK_KMAX ? k : q)] = t;
        }
      }
}

static int smallk_blocks(int m, int* rows_per_block) {
  int rpb = (m + HGB_NUM_SMS * 4 - 1) / (HGB_NUM_SMS * 4);
  rpb = ((rpb + 31) / 32) * 32;      // 8 walkers x 4 rows per trip (also a multiple of the tiny kernel's needs)
  if (rpb < 32) rpb = 32;
  *rows_per_block = rpb;
  return (m + rpb - 1) / rpb;
}

extern "C" int hgb_linear_smallk_supported(int32_t n, int32_t k) { return (k >= 1 && k <= SK_KMAX && n >= 1 && n <= 32 * SK_NPT) ? 1 : 0; }

extern "C" int hgb_linear_smallk_fwd(const float* x, int64_t ldx, const float* w, int64_t ldw, const float* b, int32_t m, int32_t n,
                                     int32_t k, int32_t act, float act_param, float* y, float* z, hgb_stream_t stream) {
  HGB_REQUIRE(x && w && y && m >= 0 && hgb_linear_smallk_supported(n, k), "linear_smallk_fwd: unsupported shape n=%d k=%d", n, k);
  if (m == 0) return HGB_OK;
  const int64_t total = (int64_t)m * n;
  if (n % 4 == 0 && n >= 16 && ((uintptr_t)y % 16 == 0) && (!z || (uintptr_t)z % 16 == 0)) {
    const int cg = n / 4;                                   // <= 64 column groups
    dim3 block(cg, 256 / cg > 0 ? 256 / cg : 1);
    const int grid = hgb_grid_for(m, block.y, HGB_NUM_SMS * 8);
    cudaStream_t st = (cudaStream_t)stream;
#define SKV(KT_) linear_smallk_fwd_vec4_kernel<KT_><<<grid, block, 0, st>>>(x, ldx, w, ldw, b, m, n, k, act, act_param, y, z)
    if (k <= 1) SKV(1); else if (k <= 2) SKV(2); else if (k <= 4) SKV(4); else SKV(8);
#undef SKV
    HGB_LAUNCH_CHECK("linear_smallk_fwd");
    return HGB_OK;
  }
  linear_smallk_fwd_kernel<<<hgb_grid_for(total, 256), 256, (size_t)(n * k + n) * 4, (cudaStream_t)stream>>>(x, ldx, w, ldw, b, total, n, k,
                                                                                                       act, act_param, y, z);
  HGB_LAUNCH_CHECK("linear_smallk_fwd");
  return HGB_OK;
}

extern "C" int hgb_linear_smallk_fwd_prelu(const float* x, int64_t ldx, const float* w, int64_t ldw, const float* b, int32_t m,
                                           int32_t n, int32_t k, const float* slope, float* y, float* z, hgb_stream_t stream) {
  HGB_REQUIRE(x && w && y && z && slope && m >= 0 && hgb_linear_smallk_supported(n, k),
              "linear_smallk_fwd_prelu: bad arguments or unsupported shape n=%d k=%d", n, k);
  if (m == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (n % 4 == 0 && n >= 16 && ((uintptr_t)y % 16 == 0) && ((uintptr_t)z % 16 == 0)) {
    const int cg = n / 4;
    dim3 block(cg, 256 / cg > 0 ? 256 / cg : 1);
    const int grid = hgb_grid_for(m, block.y, HGB_NUM_SMS * 8);
#define SKV(KT_) linear_smallk_fwd_vec4_prelu_kernel<KT_><<<grid, block, 0, st>>>(x, ldx, w, ldw, b, m, n, k, y, z, slope)
    if (k <= 1) SKV(1); else if (k <= 2) SKV(2); else if (k <= 4) SKV(4); else SKV(8);
#undef SKV
  } else {
    const int64_t total = (int64_t)m * n;
    linear_smallk_fwd_prelu_kernel<<<hgb_grid_for(total, 256), 256, (size_t)(n * k + n) * 4, st>>>(x, ldx, w, ldw, b, total, n, k,
                                                                                                      y, z, slope);
  }
  HGB_LAUNCH_CHECK("linear_smallk_fwd_prelu");
  return HGB_OK;
}

extern "C" int64_t hgb_linear_smallk_bwd_workspace_bytes(int32_t m, int32_t n, int32_t k) {
  int rpb;
  return (int64_t)smallk_blocks(m, &rpb) * n * (k + 1) * 4;
}

// dy [m,n] is the gradient of the activation OUTPUT; y (or z for SiLU) lets the kernel apply act' itself.
extern "C" int hgb_linear_smallk_bwd(const float* dy, const float* y, const float* z, const float* x, int64_t ldx, const float* w,
                                     int64_t ldw, int32_t m, int32_t n, int32_t k, int32_t act, float act_param, float* dx, float* dw,
                                     int64_t lddw, float* db, void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(dy && x && w && workspace && m >= 0 && hgb_linear_smallk_supported(n, k), "linear_smallk_bwd: unsupported shape n=%d k=%d", n, k);
  HGB_REQUIRE(act != HGB_ACT_SILU || z, "linear_smallk_bwd: SiLU needs the pre-activation z");
  HGB_REQUIRE(act == HGB_ACT_SILU || act == HGB_ACT_NONE || y, "linear_smallk_bwd: needs the activation output y");
  cudaStream_t st = (cudaStream_t)stream;
  if (m == 0) {
    if (dw) cudaMemset2DAsync(dw, lddw * 4, 0, (size_t)k * 4, n, st);
    if (db) cudaMemsetAsync(db, 0, (size_t)n * 4, st);
    return HGB_OK;
  }
  int rpb;
  const int nb = smallk_blocks(m, &rpb);
  int nb_used = nb;
  if (n <= SK_NMAX) {
    // thread-per-row kernel: the per-block reduction (n (k+1) block-wide sums) dominates unless a thread owns several rows
    int rpb_t = (m + HGB_NUM_SMS * 2 - 1) / (HGB_NUM_SMS * 2);
    rpb_t = ((rpb_t + 255) / 256) * 256;
    nb_used = (m + rpb_t - 1) / rpb_t;          // <= nb: the workspace is sized for nb partials
    linear_tiny_bwd_kernel<<<nb_used, 256, 0, st>>>(dy, y, z, x, ldx, w, ldw, m, n, k, act, act_param, rpb_t, dx, (float*)workspace);
  } else {
    const int kt = k <= 1 ? 1 : (k <= 2 ? 2 : (k <= 4 ? 4 : 8));
    const int npt = n <= 32 ? 1 : (n <= 64 ? 2 : (n <= 128 ? 4 : 8));
#define SK_LAUNCH(KT_, NPT_) linear_smallk_bwd_kernel<KT_, NPT_><<<nb, dim3(32, 8), 0, st>>>(dy, y, z, x, ldx, w, ldw, m, n, k, act, act_param, rpb, dx, (float*)workspace)
#define SK_LAUNCH_N(KT_) do { if (npt == 1) SK_LAUNCH(KT_, 1); else if (npt == 2) SK_LAUNCH(KT_, 2); else if (npt == 4) SK_LAUNCH(KT_, 4); else SK_LAUNCH(KT_, 8); } while (0)
    if (kt == 1) SK_LAUNCH_N(1); else if (kt == 2) SK_LAUNCH_N(2); else if (kt == 4) SK_LAUNCH_N(4); else SK_LAUNCH_N(8);
#undef SK_LAUNCH_N
#undef SK_LAUNCH
  }
  HGB_LAUNCH_CHECK("linear_smallk_bwd");
  linear_smallk_reduce_kernel<<<(n * (k + 1) + 31) / 32, dim3(32, 8), 0, st>>>((const float*)workspace, nb_used, n, k, dw, lddw, db);
  HGB_LAUNCH_CHECK("linear_smallk_reduce");
  return HGB_OK;
}

// ---- Linear(1,1) - act - Linear(1,out<=4) on one scalar per row (the scalar_message_mlp of a width-1 PaiNN layer, quirk Q4) ----
// params8: 0 w1, 1 b1, 2 + j: w2[j], 6 + j... -> pack of 10 floats: [w1, b1, w2[0..3], b2[0..3]]; gradient pack has the same layout.
__global__ void mlp2_scalar_fwd_kernel(const float* __restrict__ x, const float* __restrict__ pk, int n, int out, int act, float ap,
                                       float* __restrict__ y) {
  __shared__ float p[10];
  if (threadIdx.x < 10) p[threadIdx.x] = pk[threadIdx.x];
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float h = hgb_act(fmaf(p[0], x[i], p[1]), act, ap);
    for (int j = 0; j < out; ++j) y[(int64_t)i * out + j] = fmaf(p[2 + j], h, p[6 + j]);
  }
}

__global__ void __launch_bounds__(256)
mlp2_scalar_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ x, const float* __restrict__ pk, int n, int out, int act,
                       float ap, float* __restrict__ gx, float* __restrict__ part) {
  __shared__ float p[10];
  __shared__ float red[8][10];
  if (threadIdx.x < 10) p[threadIdx.x] = pk[threadIdx.x];
  __syncthreads();
  float g[10];
#pragma unroll
  for (int q = 0; q < 10; ++q) g[q] = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float xi = x[i];
    const float z = fmaf(p[0], xi, p[1]);
    const float h = hgb_act(z, act, ap);
    float gh = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < out) {
        const float gj = gy[(int64_t)i * out + j];
        gh = fmaf(gj, p[2 + j], gh);
        g[2 + j] = fmaf(gj, h, g[2 + j]);
        g[6 + j] += gj;
      }
    const float gz = gh * hgb_act_grad(h, z, act, ap);
    g[0] = fmaf(gz, xi, g[0]);
    g[1] += gz;
    if (gx) gx[i] = gz * p[0];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 10; ++q) {
    const float t = hgb_warp_sum(g[q]);
    if (lane == 0) red[warp][q] = t;
  }
  __syncthreads();
  if (threadIdx.x < 10) {
    float t = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][threadIdx.x];
    part[blockIdx.x * 10 + threadIdx.x] = t;
  }
}

__global__ void mlp2_scalar_reduce_kernel(const float* __restrict__ part, int nb, float* __restrict__ gp) {
  if (threadIdx.x < 10) {
    float t = 0.f;
    for (int b = 0; b < nb; ++b) t += part[b * 10 + threadIdx.x];
    gp[threadIdx.x] = t;
  }
}

#define MLP2S_BLOCKS (HGB_NUM_SMS * 2)
extern "C" int64_t hgb_mlp2_scalar_workspace_bytes(void) { return (int64_t)MLP2S_BLOCKS * 10 * 4; }

extern "C" int hgb_mlp2_scalar_fwd(const float* x, const float* params10, int32_t n, int32_t out, int32_t act, float act_param, float* y,
                                   hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && out >= 1 && out <= 4 && x && params10 && y, "mlp2_scalar_fwd: bad arguments (1 <= out <= 4)");
  if (n == 0) return HGB_OK;
  mlp2_scalar_fwd_kernel<<<hgb_grid_for(n, 256, HGB_NUM_SMS * 4), 256, 0, (cudaStream_t)stream>>>(x, params10, n, out, act, act_param, y);
  HGB_LAUNCH_CHECK("mlp2_scalar_fwd");
  return HGB_OK;
}

extern "C" int hgb_mlp2_scalar_bwd(const float* gy, const float* x, const float* params10, int32_t n, int32_t out, int32_t act,
                                   float act_param, float* gx, float* gparams10, void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && out >= 1 && out <= 4 && gy && x && params10 && gparams10 && workspace, "mlp2_scalar_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { cudaMemsetAsync(gparams10, 0, 40, st); return HGB_OK; }
  const int nb = hgb_grid_for(n, 256, MLP2S_BLOCKS);
  mlp2_scalar_bwd_kernel<<<nb, 256, 0, st>>>(gy, x, params10, n, out, act, act_param, gx, (float*)workspace);
  HGB_LAUNCH_CHECK("mlp2_scalar_bwd");
  mlp2_scalar_reduce_kernel<<<1, 32, 0, st>>>((const float*)workspace, nb, gparams10);
  HGB_LAUNCH_CHECK("mlp2_scalar_reduce");
  return HGB_OK;
}
