// SchNet's continuous-filter convolution (hydragnn/models/SCFStack.py:267-301, CFConv with aggr "add") in one pass.
//
// For the edge e = (j -> i), i = edge_index[1] the target and j = edge_index[0] the source:
//   d_e   = |pos[i] - pos[j]|
//   a_e   = [exp(coeff (d_e - mu_k)^2), k < G | r_e]                       (GaussianSmearing, then the raw edge input r_e)
//   h_e   = A^T a_e + b1,   A = [W1[:, :G]^T ; Mt]  [G + D, NF]            (the filter network's first Linear, edge block folded)
//   W_e   = ((ssp(h_e) W2^T) + b2) * 0.5 (cos(pi d_e / cutoff) + 1)        (ssp = softplus(., threshold 20) - log 2)
//   out_i = sum_{e -> i} xl[j] * W_e
// Nothing per edge reaches memory in the forward except the optional W_e (the equivariant coordinate MLP reads it).
//
// Thread mapping: one warp per edge at a time; lane l owns the channels f = l + 32 t, t < NT = ceil(NF / 32).  A, W2, b1, b2
// and the Gaussian centres are staged in shared memory once per CTA; each warp has a small buffer for a_e and ssp(h_e).  W2 is
// stored transposed with row stride NF + 1, so both the forward (lanes vary the output channel) and the backward (lanes vary the
// input channel) read it without bank conflicts.
//
// Forward: each warp owns whole target segments, so out_i is summed in registers in CSR order.  Backward: each warp takes one
// edge of a CTA-wide tile; the per-edge factors are staged and every thread adds its own fixed entries of the parameter
// gradients, so the per-CTA partials are sums in a fixed order and the fp64 reduction over CTAs is fixed too: no atomics,
// two runs are bit-identical.
#include "hgb_common.cuh"

#define CF_MAX_G 64
#define CF_MAX_D 16
#define CF_MAX_NF 128
#define CF_FWD_WARPS 8
#define CF_BWD_MAX_WARPS 8
#define CF_BWD_MAX_BLOCKS HGB_NUM_SMS
#define CF_LOG2 0.693147182464599609375f     // PyG ShiftedSoftplus: log(2) rounded to fp32
#define CF_PI 3.14159265358979323846f

namespace {

struct CfParams {
  const float* pos;
  const int32_t* row;
  const int32_t* col;
  const float* r;
  int d;
  float coeff, cutoff;
  int g, nf, k1;           // k1 = g + d
};

__device__ __forceinline__ float cf_ssp(float x) { return (x > 20.f ? x : log1pf(expf(x))) - CF_LOG2; }
__device__ __forceinline__ float cf_ssp_grad(float x) {
  if (x > 20.f) return 1.f;
  const float z = expf(x);
  return z / (z + 1.f);
}

// Shared-memory layout: A [k1][nf] | W2t [nf][nf + 1] | b1 [nf] | b2 [nf] | mu [g] | per-warp buffers.
struct CfSmem {
  float *a, *w2t, *b1, *b2, *mu, *warp;
  __device__ CfSmem(float* s, int g, int nf, int k1) {
    a = s;
    w2t = a + k1 * nf;
    b1 = w2t + nf * (nf + 1);
    b2 = b1 + nf;
    mu = b2 + nf;
    warp = mu + g;
  }
};

__device__ __forceinline__ void cf_stage(const CfSmem& S, const CfParams& P, const float* __restrict__ a1t,
                                         const float* __restrict__ b1, const float* __restrict__ w2,
                                         const float* __restrict__ b2, const float* __restrict__ mu) {
  const int nf = P.nf;
  for (int t = threadIdx.x; t < P.k1 * nf; t += blockDim.x) S.a[t] = a1t[t];
  for (int t = threadIdx.x; t < nf * nf; t += blockDim.x) {
    const int f = t / nf, k = t % nf;                           // W2[f][k] -> W2t[k][f]
    S.w2t[k * (nf + 1) + f] = w2[t];
  }
  for (int t = threadIdx.x; t < nf; t += blockDim.x) {
    S.b1[t] = b1[t];
    S.b2[t] = b2[t];
  }
  for (int t = threadIdx.x; t < P.g; t += blockDim.x) S.mu[t] = mu[t];
}

// The filter of one edge, computed by one warp: d, the envelope C, a_e (into abuf), h and u = ssp(h) W2^T + b2 for the lane's
// channels, ssp(h) into sbuf.  The forward and the backward both call this, so the backward sees the forward's values bit for bit.
template <int NT>
__device__ __forceinline__ void cf_filter(const CfSmem& S, const CfParams& P, int64_t e, int i, int j, float* abuf, float* sbuf,
                                          float& d, float& c, float (&h)[NT], float (&u)[NT]) {
  const int lane = threadIdx.x & 31, nf = P.nf;
  const float dx = P.pos[3 * i] - P.pos[3 * j], dy = P.pos[3 * i + 1] - P.pos[3 * j + 1], dz = P.pos[3 * i + 2] - P.pos[3 * j + 2];
  d = sqrtf(dx * dx + dy * dy + dz * dz);
  c = 0.5f * (cosf(d * CF_PI / P.cutoff) + 1.f);
  for (int k = lane; k < P.g; k += 32) {
    const float t = d - S.mu[k];
    abuf[k] = expf(P.coeff * (t * t));
  }
  for (int k = lane; k < P.d; k += 32) abuf[P.g + k] = P.r[e * P.d + k];
  __syncwarp();
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int f = lane + 32 * t;
    float acc = 0.f;
    if (f < nf) {
      acc = S.b1[f];
      for (int k = 0; k < P.k1; ++k) acc = fmaf(S.a[k * nf + f], abuf[k], acc);
      sbuf[f] = cf_ssp(acc);
    }
    h[t] = acc;
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int f = lane + 32 * t;
    float acc = 0.f;
    if (f < nf) {
      acc = S.b2[f];
      for (int k = 0; k < nf; ++k) acc = fmaf(S.w2t[k * (nf + 1) + f], sbuf[k], acc);
    }
    u[t] = acc;
  }
}

template <int NT>
__global__ void __launch_bounds__(CF_FWD_WARPS * 32) cfconv_fwd_kernel(
    CfParams P, const float* __restrict__ xl, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm,
    const float* __restrict__ a1t, const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
    const float* __restrict__ mu, int n, float* __restrict__ out, float* __restrict__ w_e) {
  extern __shared__ float smem[];
  const int nf = P.nf, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  CfSmem S(smem, P.g, nf, P.k1);
  cf_stage(S, P, a1t, b1, w2, b2, mu);
  __syncthreads();
  float* abuf = S.warp + warp * (P.k1 + nf);
  float* sbuf = abuf + P.k1;
  for (int node = blockIdx.x * CF_FWD_WARPS + warp; node < n; node += gridDim.x * CF_FWD_WARPS) {
    float acc[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) acc[t] = 0.f;
    for (int p = rowptr[node]; p < rowptr[node + 1]; ++p) {
      const int64_t e = perm ? perm[p] : p;
      const int j = P.row[e];
      float d, c, h[NT], u[NT];
      cf_filter<NT>(S, P, e, node, j, abuf, sbuf, d, c, h, u);
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int f = lane + 32 * t;
        if (f < nf) {
          const float w = u[t] * c;
          acc[t] = fmaf(xl[(int64_t)j * nf + f], w, acc[t]);
          if (w_e) w_e[e * nf + f] = w;
        }
      }
      __syncwarp();                                     // abuf / sbuf are rewritten by the next edge
    }
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int f = lane + 32 * t;
      if (f < nf) out[(int64_t)node * nf + f] = acc[t];
    }
  }
}

// Per edge (g_W = g_out[i] * xl[j] + g_We[e]):
//   g_xl_e = g_out[i] * W_e                        (edge order; the host sums it over the sources)
//   g_u = g_W * C,   g_C = <g_W, u>,   g_s = W2^T g_u,   g_h = g_s * ssp'(h)
//   g_d = g_C dC/dd + sum_k g_a[k] d a_k / dd (k < G),   g_r = Mt g_h
//   parameter sums: g_A += a_e g_h^T, g_b1 += g_h, g_W2 += g_u ssp(h)^T, g_b2 += g_u
// part [gridDim.x, k1 * nf + nf + nf * nf + nf] = per-CTA [g_A | g_b1 | g_W2 | g_b2].
template <int NT>
__global__ void __launch_bounds__(CF_BWD_MAX_WARPS * 32) cfconv_bwd_kernel(
    CfParams P, const float* __restrict__ g_out, const float* __restrict__ g_we, const float* __restrict__ xl,
    const float* __restrict__ a1t, const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
    const float* __restrict__ mu, int64_t ne, float* __restrict__ g_xle, float* __restrict__ g_dist, float* __restrict__ g_r,
    float* __restrict__ part) {
  extern __shared__ float smem[];
  const int nf = P.nf, k1 = P.k1, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  CfSmem S(smem, P.g, nf, k1);
  const int wstride = k1 + 3 * nf;                         // per warp: a_e [k1] | ssp(h) [nf] | g_u [nf] | g_h [nf]
  float* acc_a = S.warp + nw * wstride;                    // [k1][nf]
  float* acc_b1 = acc_a + k1 * nf;                         // [nf]
  float* acc_w2 = acc_b1 + nf;                             // [nf][nf]
  float* acc_b2 = acc_w2 + nf * nf;                        // [nf]
  const int nacc = k1 * nf + nf + nf * nf + nf;
  cf_stage(S, P, a1t, b1, w2, b2, mu);
  for (int t = threadIdx.x; t < nacc; t += blockDim.x) acc_a[t] = 0.f;
  __syncthreads();
  float* abuf = S.warp + warp * wstride;
  float* sbuf = abuf + k1;
  float* gubuf = sbuf + nf;
  float* ghbuf = gubuf + nf;
  const float dcdd = -0.5f * CF_PI / P.cutoff;
  for (int64_t base = (int64_t)blockIdx.x * nw; base < ne; base += (int64_t)gridDim.x * nw) {
    const int64_t e = base + warp;
    if (e < ne) {
      const int i = P.col[e], j = P.row[e];
      float d, c, h[NT], u[NT], gu[NT];
      cf_filter<NT>(S, P, e, i, j, abuf, sbuf, d, c, h, u);
      float gc = 0.f;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int f = lane + 32 * t;
        gu[t] = 0.f;
        if (f < nf) {
          const float go = g_out[(int64_t)i * nf + f];
          float gw = go * xl[(int64_t)j * nf + f];
          if (g_we) gw += g_we[e * nf + f];
          if (g_xle) g_xle[e * nf + f] = go * (u[t] * c);
          gu[t] = gw * c;
          gc = fmaf(gw, u[t], gc);
          gubuf[f] = gu[t];
        }
      }
      __syncwarp();
      float gdr = 0.f;                                     // sum_f g_h[f] sum_k A[k][f] d a_k / dd
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int f = lane + 32 * t;
        if (f < nf) {
          float gs = 0.f;
          for (int k = 0; k < nf; ++k) gs = fmaf(S.w2t[f * (nf + 1) + k], gubuf[k], gs);      // (W2^T g_u)[f]
          const float gh = gs * cf_ssp_grad(h[t]);
          ghbuf[f] = gh;
          if (g_dist) {
            float q = 0.f;
            for (int k = 0; k < P.g; ++k) q = fmaf(S.a[k * nf + f], abuf[k] * (2.f * P.coeff * (d - S.mu[k])), q);
            gdr = fmaf(gh, q, gdr);
          }
        }
      }
      if (g_dist) {
        const float gcs = hgb_warp_sum(gc);
        const float gds = hgb_warp_sum(gdr);
        if (lane == 0) g_dist[e] = gcs * (dcdd * sinf(d * CF_PI / P.cutoff)) + gds;
      }
      if (g_r) {
        for (int q = 0; q < P.d; ++q) {
          float s = 0.f;
#pragma unroll
          for (int t = 0; t < NT; ++t) {
            const int f = lane + 32 * t;
            if (f < nf) s = fmaf(S.a[(P.g + q) * nf + f], ghbuf[f], s);
          }
          s = hgb_warp_sum(s);
          if (lane == 0) g_r[e * P.d + q] = s;
        }
      }
    } else {
      for (int t = lane; t < wstride; t += 32) abuf[t] = 0.f;     // an idle warp adds zeros
    }
    __syncthreads();
    if (!part) continue;                                   // parameter gradients not asked for (uniform over the CTA)
    // every thread owns fixed accumulator entries; the warps' edges are added in warp order
    for (int t = threadIdx.x; t < k1 * nf; t += blockDim.x) {
      const int k = t / nf, f = t % nf;
      float s = acc_a[t];
      for (int w = 0; w < nw; ++w) s = fmaf(S.warp[w * wstride + k], S.warp[w * wstride + k1 + 2 * nf + f], s);
      acc_a[t] = s;
    }
    for (int t = threadIdx.x; t < nf * nf; t += blockDim.x) {
      const int f = t / nf, k = t % nf;
      float s = acc_w2[t];
      for (int w = 0; w < nw; ++w) s = fmaf(S.warp[w * wstride + k1 + nf + f], S.warp[w * wstride + k1 + k], s);
      acc_w2[t] = s;
    }
    for (int t = threadIdx.x; t < nf; t += blockDim.x) {
      float s1 = acc_b1[t], s2 = acc_b2[t];
      for (int w = 0; w < nw; ++w) {
        s1 += S.warp[w * wstride + k1 + 2 * nf + t];
        s2 += S.warp[w * wstride + k1 + nf + t];
      }
      acc_b1[t] = s1;
      acc_b2[t] = s2;
    }
    __syncthreads();
  }
  if (part)
    for (int t = threadIdx.x; t < nacc; t += blockDim.x) part[(int64_t)blockIdx.x * nacc + t] = acc_a[t];
}

// out[r] = sum over the CTAs in index order (fp64) of part[b, r]
__global__ void cfconv_reduce_kernel(const float* __restrict__ part, int nblk, int rows, float* __restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += (double)part[(int64_t)b * rows + r];
    out[r] = (float)s;
  }
}

size_t cf_fwd_smem(int g, int nf, int k1) {
  return sizeof(float) * ((size_t)k1 * nf + (size_t)nf * (nf + 1) + 2 * nf + g + (size_t)CF_FWD_WARPS * (k1 + nf));
}

size_t cf_bwd_smem(int g, int nf, int k1, int nw) {
  return sizeof(float) * ((size_t)k1 * nf + (size_t)nf * (nf + 1) + 2 * nf + g + (size_t)nw * (k1 + 3 * nf) +
                          (size_t)k1 * nf + 2 * nf + (size_t)nf * nf);
}

int cf_smem_limit() {
  static int limit = -1;
  if (limit < 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) limit = 0;
  }
  return limit;
}

// the most warps per backward CTA whose shared memory fits (8, else 4, 2, 1)
int cf_bwd_warps(int g, int nf, int k1) {
  int nw = CF_BWD_MAX_WARPS;
  while (nw > 1 && cf_bwd_smem(g, nf, k1, nw) > (size_t)cf_smem_limit()) nw >>= 1;
  return nw;
}

bool cf_sizes_ok(int32_t g, int32_t nf, int32_t d) {
  return g >= 1 && g <= CF_MAX_G && nf >= 1 && nf <= CF_MAX_NF && d >= 0 && d <= CF_MAX_D;
}
}  // namespace

#define CF_DISPATCH(LAUNCH)       \
  do {                            \
    switch ((nf + 31) / 32) {     \
      case 1: LAUNCH(1); break;   \
      case 2: LAUNCH(2); break;   \
      case 3: LAUNCH(3); break;   \
      default: LAUNCH(4); break;  \
    }                             \
  } while (0)

extern "C" int hgb_cfconv_supported(int32_t g, int32_t nf, int32_t d) { return cf_sizes_ok(g, nf, d) ? 1 : 0; }

extern "C" int64_t hgb_cfconv_workspace_bytes(int32_t g, int32_t nf, int32_t d) {
  if (!cf_sizes_ok(g, nf, d)) return -1;
  const int64_t nacc = (int64_t)(g + d) * nf + nf + (int64_t)nf * nf + nf;
  return (int64_t)CF_BWD_MAX_BLOCKS * nacc * (int64_t)sizeof(float);
}

extern "C" int hgb_cfconv_fwd(const float* xl, const float* pos, const int32_t* row, const int32_t* rowptr, const int32_t* perm,
                              const float* r, int32_t d, const float* mu, float coeff, float cutoff, const float* a1t,
                              const float* b1, const float* w2, const float* b2, int32_t n, int64_t e, int32_t g, int32_t nf,
                              float* out, float* w_e, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && e >= 0 && e < INT32_MAX && cf_sizes_ok(g, nf, d),
              "cfconv_fwd: bad sizes (n %d, e %lld, g %d, nf %d, d %d; 1 <= g <= %d, 1 <= nf <= %d, 0 <= d <= %d)", n,
              (long long)e, g, nf, d, CF_MAX_G, CF_MAX_NF, CF_MAX_D);
  HGB_REQUIRE(cutoff > 0.f, "cfconv_fwd: cutoff must be positive (got %g)", (double)cutoff);
  HGB_REQUIRE(xl && pos && row && rowptr && mu && a1t && b1 && w2 && b2 && out, "cfconv_fwd: null argument");
  HGB_REQUIRE(d == 0 || r, "cfconv_fwd: d > 0 needs the raw edge input r");
  if (n == 0) return HGB_OK;
  const CfParams P{pos, row, nullptr, r, d, coeff, cutoff, g, nf, g + d};
  const size_t smem = cf_fwd_smem(g, nf, g + d);
  HGB_REQUIRE(smem <= (size_t)cf_smem_limit(), "cfconv_fwd: %zu bytes of shared memory exceed the device limit", smem);
  const int grid = hgb_grid_for(n, CF_FWD_WARPS, HGB_NUM_SMS * 2);
#define CF_FWD(NT)                                                                                                  \
  cudaFuncSetAttribute(cfconv_fwd_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
  cfconv_fwd_kernel<NT><<<grid, CF_FWD_WARPS * 32, smem, (cudaStream_t)stream>>>(P, xl, rowptr, perm, a1t, b1, w2, b2, \
                                                                                  mu, n, out, w_e)
  CF_DISPATCH(CF_FWD);
#undef CF_FWD
  HGB_LAUNCH_CHECK("cfconv_fwd");
  return HGB_OK;
}

extern "C" int hgb_cfconv_bwd(const float* g_out, const float* g_we, const float* xl, const float* pos, const int32_t* row,
                              const int32_t* col, const float* r, int32_t d, const float* mu, float coeff, float cutoff,
                              const float* a1t, const float* b1, const float* w2, const float* b2, int32_t n, int64_t e,
                              int32_t g, int32_t nf, float* g_xle, float* g_dist, float* g_r, float* g_params, void* workspace,
                              hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && e >= 0 && e < INT32_MAX && cf_sizes_ok(g, nf, d),
              "cfconv_bwd: bad sizes (n %d, e %lld, g %d, nf %d, d %d; 1 <= g <= %d, 1 <= nf <= %d, 0 <= d <= %d)", n,
              (long long)e, g, nf, d, CF_MAX_G, CF_MAX_NF, CF_MAX_D);
  HGB_REQUIRE(cutoff > 0.f, "cfconv_bwd: cutoff must be positive (got %g)", (double)cutoff);
  HGB_REQUIRE(g_out && xl && pos && row && col && mu && a1t && b1 && w2 && b2, "cfconv_bwd: null argument");
  HGB_REQUIRE(!g_params || workspace, "cfconv_bwd: g_params needs the workspace");
  HGB_REQUIRE(d == 0 || r, "cfconv_bwd: d > 0 needs the raw edge input r");
  const int k1 = g + d;
  const int rows = k1 * nf + nf + nf * nf + nf;
  if (e == 0) {
    if (g_params) cudaMemsetAsync(g_params, 0, sizeof(float) * (size_t)rows, (cudaStream_t)stream);
    HGB_LAUNCH_CHECK("cfconv_bwd");
    return HGB_OK;
  }
  const int nw = cf_bwd_warps(g, nf, k1);
  const size_t smem = cf_bwd_smem(g, nf, k1, nw);
  HGB_REQUIRE(smem <= (size_t)cf_smem_limit(), "cfconv_bwd: %zu bytes of shared memory exceed the device limit", smem);
  const CfParams P{pos, row, col, r, d, coeff, cutoff, g, nf, k1};
  const int grid = hgb_grid_for(e, nw, CF_BWD_MAX_BLOCKS);
  float* part = g_params ? static_cast<float*>(workspace) : nullptr;
#define CF_BWD(NT)                                                                                                   \
  cudaFuncSetAttribute(cfconv_bwd_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);              \
  cfconv_bwd_kernel<NT><<<grid, nw * 32, smem, (cudaStream_t)stream>>>(P, g_out, g_we, xl, a1t, b1, w2, b2, mu, e, g_xle, \
                                                                        g_dist, g_r, part)
  CF_DISPATCH(CF_BWD);
#undef CF_BWD
  HGB_LAUNCH_CHECK("cfconv_bwd");
  if (!g_params) return HGB_OK;
  cfconv_reduce_kernel<<<hgb_grid_for(rows, 256), 256, 0, (cudaStream_t)stream>>>(part, grid, rows, g_params);
  HGB_LAUNCH_CHECK("cfconv_reduce");
  return HGB_OK;
}
