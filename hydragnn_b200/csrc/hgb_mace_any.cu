// libhgb.so -- closed (any-order differentiable) primitives for the MACE force-training path and for the shapes the fused
// first-order kernels of hgb_mace.cu do not cover (correlation 3, channel counts that are not a multiple of 32).
//
// Round 1 composed these from torch.einsum; VERDICT r1 asked for hand-written primitives that are closed under differentiation,
// like GatherRows <-> SegmentSum.  Two families:
//
// (1) per-edge coupling of one tensor-product path (blocks.py:386-397, o3.TensorProduct "uvu" with per-edge weights):
//       tp_out   o[e, k, f] = w[e, f] * sum_{i, j} C[i, j, k] a[e, i, f] y[e, j]
//       tp_y     o[e, j]    = sum_f w[e, f] sum_{i, k} C[i, j, k] a[e, i, f] g[e, k, f]
//       tp_w     o[e, f]    = sum_{i, j, k} C[i, j, k] a[e, i, f] y[e, j] g[e, k, f]
//     C = real coupling tensor of the path (<= 7 x 7 x 7).  The three forms are each other's derivatives (the derivative of
//     tp_out w.r.t. a is tp_out again with C permuted), so any order of differentiation stays inside these kernels.
//
// (2) per-node, per-channel contraction steps of the symmetric contraction (symmetric_contraction.py:217-239):
//       chan_cl  o[b, c, p]    = sum_i t[b, c, p, i] x[b, i, c]        ("contract last")
//       chan_ou  o[b, c, p, i] = g[b, c, p] x[b, i, c]                 ("outer")
//       chan_rp  o[b, i, c]    = sum_p g[b, c, p] t[b, c, p, i]        ("reduce p")
//     again mutually adjoint.  The U-matrix x weight products in front of them are plain MatMuls (closed already).
//
// (3) edge-attribute mixing of the 0e paths' weight blocks (edge_dim > 0):
//       edge_mix    o[e, u]    = c * sum_v w[e, u, v] a[e, v]          a = [edge_attr, 1]
//       edge_mix_t  o[e, u, v] = c * g[e, u] a[e, v]
//     mutually adjoint and linear in w / g; the edge attributes are data.
//
// All are bandwidth-trivial elementwise-style SIMT kernels: one thread per output element (tp_y: one warp per edge).
#include "hgb_common.cuh"

namespace {

constexpr int CMAX = 7 * 7 * 7;

__global__ void tp_out_kernel(const float* __restrict__ a, const float* __restrict__ y, const float* __restrict__ w,
                              const float* __restrict__ cg, int64_t e, int f, int ni, int nj, int nk, float* __restrict__ out) {
  __shared__ float sc[CMAX];
  for (int q = threadIdx.x; q < ni * nj * nk; q += blockDim.x) sc[q] = cg[q];
  __syncthreads();
  const int64_t total = e * f;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ed = idx / f;
    const int c = (int)(idx - ed * f);
    float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < ni; ++i) {
      const float av = a[(ed * ni + i) * f + c];
      for (int j = 0; j < nj; ++j) {
        const float ay = av * y[ed * nj + j];
        const float* cr = sc + (i * nj + j) * nk;
        for (int k = 0; k < nk; ++k) acc[k] = fmaf(cr[k], ay, acc[k]);
      }
    }
    const float wv = w[ed * f + c];
    for (int k = 0; k < nk; ++k) out[(ed * nk + k) * f + c] = wv * acc[k];
  }
}

// one warp per edge, lanes over channels
__global__ void tp_y_kernel(const float* __restrict__ a, const float* __restrict__ g, const float* __restrict__ w,
                            const float* __restrict__ cg, int64_t e, int f, int ni, int nj, int nk, float* __restrict__ out) {
  __shared__ float sc[CMAX];
  for (int q = threadIdx.x; q < ni * nj * nk; q += blockDim.x) sc[q] = cg[q];
  __syncthreads();
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int64_t ed = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); ed < e; ed += (int64_t)gridDim.x * wpb) {
    float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = lane; c < f; c += 32) {
      const float wv = w[ed * f + c];
      for (int i = 0; i < ni; ++i) {
        const float av = a[(ed * ni + i) * f + c] * wv;
        for (int k = 0; k < nk; ++k) {
          const float ag = av * g[(ed * nk + k) * f + c];
          for (int j = 0; j < nj; ++j) acc[j] = fmaf(sc[(i * nj + j) * nk + k], ag, acc[j]);
        }
      }
    }
    for (int j = 0; j < nj; ++j) {
      const float s = hgb_warp_sum(acc[j]);
      if (lane == 0) out[ed * nj + j] = s;
    }
  }
}

__global__ void tp_w_kernel(const float* __restrict__ a, const float* __restrict__ y, const float* __restrict__ g,
                            const float* __restrict__ cg, int64_t e, int f, int ni, int nj, int nk, float* __restrict__ out) {
  __shared__ float sc[CMAX];
  for (int q = threadIdx.x; q < ni * nj * nk; q += blockDim.x) sc[q] = cg[q];
  __syncthreads();
  const int64_t total = e * f;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ed = idx / f;
    const int c = (int)(idx - ed * f);
    float gv[7];
    for (int k = 0; k < nk; ++k) gv[k] = g[(ed * nk + k) * f + c];
    float acc = 0.f;
    for (int i = 0; i < ni; ++i) {
      const float av = a[(ed * ni + i) * f + c];
      for (int j = 0; j < nj; ++j) {
        const float* cr = sc + (i * nj + j) * nk;
        float t = 0.f;
        for (int k = 0; k < nk; ++k) t = fmaf(cr[k], gv[k], t);
        acc = fmaf(av * y[ed * nj + j], t, acc);
      }
    }
    out[idx] = acc;
  }
}

__global__ void chan_cl_kernel(const float* __restrict__ t, const float* __restrict__ x, int64_t n, int f, int p, int ni,
                               float* __restrict__ out) {
  const int64_t total = n * f * p;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bc = idx / p;
    const int64_t b = bc / f;
    const int c = (int)(bc - b * f);
    float acc = 0.f;
    for (int i = 0; i < ni; ++i) acc = fmaf(t[idx * ni + i], x[(b * ni + i) * f + c], acc);
    out[idx] = acc;
  }
}

__global__ void chan_ou_kernel(const float* __restrict__ g, const float* __restrict__ x, int64_t n, int f, int p, int ni,
                               float* __restrict__ out) {
  const int64_t total = n * f * p * ni;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx % ni);
    const int64_t bcp = idx / ni;
    const int64_t bc = bcp / p;
    const int64_t b = bc / f;
    const int c = (int)(bc - b * f);
    out[idx] = g[bcp] * x[(b * ni + i) * f + c];
  }
}

__global__ void chan_rp_kernel(const float* __restrict__ g, const float* __restrict__ t, int64_t n, int f, int p, int ni,
                               float* __restrict__ out) {
  const int64_t total = n * ni * f;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % f);
    const int64_t bi = idx / f;
    const int i = (int)(bi % ni);
    const int64_t b = bi / ni;
    const int64_t base = (b * f + c) * p;
    float acc = 0.f;
    for (int q = 0; q < p; ++q) acc = fmaf(g[base + q], t[(base + q) * ni + i], acc);
    out[idx] = acc;
  }
}

// edge-attribute mixing of a 0e path's [F, d+1] weight block; one thread per output element
__global__ void edge_mix_kernel(const float* __restrict__ w, int64_t ld, const float* __restrict__ ea, int64_t e, int f, int d, float c,
                                float* __restrict__ out) {
  const int64_t total = e * f;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ed = idx / f;
    const int u = (int)(idx - ed * f);
    const float* q = w + ed * ld + (int64_t)u * (d + 1);
    float s = q[d];
    for (int v = 0; v < d; ++v) s = fmaf(q[v], ea[ed * d + v], s);
    out[idx] = c * s;
  }
}

__global__ void edge_mix_t_kernel(const float* __restrict__ g, int64_t ld, const float* __restrict__ ea, int64_t e, int f, int d, float c,
                                  float* __restrict__ out) {
  const int64_t total = e * f * (d + 1);
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t eu = idx / (d + 1);
    const int v = (int)(idx - eu * (d + 1));
    const int64_t ed = eu / f;
    const int u = (int)(eu - ed * f);
    const float gv = c * g[ed * ld + u];
    out[idx] = v < d ? gv * ea[ed * d + v] : gv;
  }
}

}  // namespace

extern "C" int hgb_mace_edge_mix(int32_t mode, const float* src, int64_t ld, const float* eattr, int64_t e, int32_t f, int32_t d, float c,
                                 float* out, hgb_stream_t stream) {
  HGB_REQUIRE((mode == 0 || mode == 1) && src && eattr && out && e >= 0 && f >= 1 && d >= 1 &&
                  ld >= (mode == 0 ? (int64_t)f * (d + 1) : (int64_t)f),
              "mace_edge_mix: bad arguments");
  if (e == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) edge_mix_kernel<<<hgb_grid_for(e * f, 256), 256, 0, st>>>(src, ld, eattr, e, f, d, c, out);
  else edge_mix_t_kernel<<<hgb_grid_for(e * f * (d + 1), 256), 256, 0, st>>>(src, ld, eattr, e, f, d, c, out);
  HGB_LAUNCH_CHECK("mace_edge_mix");
  return HGB_OK;
}

#define HGB_TP_CHECK(name)                                                                                               \
  HGB_REQUIRE(e >= 0 && f >= 1 && ni >= 1 && nj >= 1 && nk >= 1 && ni <= 7 && nj <= 7 && nk <= 7 && cg && out, name ": bad arguments")

// mode 0: tp_out (p0 = a [e, ni, f], p1 = y [e, nj], p2 = w [e, f])        -> out [e, nk, f]
// mode 1: tp_y   (p0 = a [e, ni, f], p1 = g [e, nk, f], p2 = w [e, f])     -> out [e, nj]
// mode 2: tp_w   (p0 = a [e, ni, f], p1 = y [e, nj], p2 = g [e, nk, f])    -> out [e, f]
extern "C" int hgb_mace_tp_path(int32_t mode, const float* p0, const float* p1, const float* p2, const float* cg, int64_t e,
                                int32_t f, int32_t ni, int32_t nj, int32_t nk, float* out, hgb_stream_t stream) {
  HGB_TP_CHECK("mace_tp_path");
  HGB_REQUIRE(mode >= 0 && mode <= 2 && p0 && p1 && p2, "mace_tp_path: bad mode / operands");
  if (e == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) tp_out_kernel<<<hgb_grid_for(e * f, 256), 256, 0, st>>>(p0, p1, p2, cg, e, f, ni, nj, nk, out);
  else if (mode == 1) tp_y_kernel<<<hgb_grid_for(e, 8), 256, 0, st>>>(p0, p1, p2, cg, e, f, ni, nj, nk, out);
  else tp_w_kernel<<<hgb_grid_for(e * f, 256), 256, 0, st>>>(p0, p1, p2, cg, e, f, ni, nj, nk, out);
  HGB_LAUNCH_CHECK("mace_tp_path");
  return HGB_OK;
}

// mode 0: chan_cl (p0 = t [n, f, p, ni], p1 = x [n, ni, f]) -> out [n, f, p]
// mode 1: chan_ou (p0 = g [n, f, p],     p1 = x [n, ni, f]) -> out [n, f, p, ni]
// mode 2: chan_rp (p0 = g [n, f, p],     p1 = t [n, f, p, ni]) -> out [n, ni, f]
extern "C" int hgb_mace_chan_contract(int32_t mode, const float* p0, const float* p1, int64_t n, int32_t f, int32_t p, int32_t ni,
                                      float* out, hgb_stream_t stream) {
  HGB_REQUIRE(mode >= 0 && mode <= 2 && p0 && p1 && out && n >= 0 && f >= 1 && p >= 1 && ni >= 1, "mace_chan_contract: bad arguments");
  if (n == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) chan_cl_kernel<<<hgb_grid_for(n * f * p, 256), 256, 0, st>>>(p0, p1, n, f, p, ni, out);
  else if (mode == 1) chan_ou_kernel<<<hgb_grid_for(n * f * p * ni, 256), 256, 0, st>>>(p0, p1, n, f, p, ni, out);
  else chan_rp_kernel<<<hgb_grid_for(n * ni * f, 256), 256, 0, st>>>(p0, p1, n, f, p, ni, out);
  HGB_LAUNCH_CHECK("mace_chan_contract");
  return HGB_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// MACE edge embedding (SURVEY K2): edge vector -> real spherical harmonics (component normalisation, e3nn axis convention:
// polar axis y; hydragnn/models/MACEStack.py:455-466 via o3.SphericalHarmonics) and Bessel basis x polynomial cutoff
// (mace_utils/modules/radial.py:18-60,110-148, blocks.py:164-177) in ONE pass per edge, with the analytic gradient
// d/d vec in the backward.  l <= 3, num_bessel <= 64 (a loop bound: nothing is sized by it).  vec = pos[col] - pos[row] + shift.
// ------------------------------------------------------------------------------------------------------------------
namespace {

#define HGB_SQ3 1.7320508075688772f
#define HGB_SQ5 2.2360679774997897f
#define HGB_SQ7 2.6457513110645906f
#define HGB_PI_F 3.14159265358979323846f

// sh[0 .. (lmax+1)^2) at unit vector (x, y, z); if GRAD, also d sh / d(x, y, z) as unconstrained polynomial gradients
template <bool GRAD>
__device__ __forceinline__ void sh_eval(int lmax, float x, float y, float z, float* sh, float (*g)[3]) {
  sh[0] = 1.f;
  if (GRAD) { g[0][0] = g[0][1] = g[0][2] = 0.f; }
  if (lmax >= 1) {
    sh[1] = HGB_SQ3 * x; sh[2] = HGB_SQ3 * y; sh[3] = HGB_SQ3 * z;
    if (GRAD) {
      g[1][0] = HGB_SQ3; g[1][1] = 0.f; g[1][2] = 0.f;
      g[2][0] = 0.f; g[2][1] = HGB_SQ3; g[2][2] = 0.f;
      g[3][0] = 0.f; g[3][1] = 0.f; g[3][2] = HGB_SQ3;
    }
  }
  if (lmax >= 2) {
    const float c = HGB_SQ5 * HGB_SQ3;
    sh[4] = c * x * z; sh[5] = c * x * y; sh[6] = HGB_SQ5 * (y * y - 0.5f * (x * x + z * z)); sh[7] = c * y * z;
    sh[8] = 0.5f * c * (z * z - x * x);
    if (GRAD) {
      g[4][0] = c * z; g[4][1] = 0.f; g[4][2] = c * x;
      g[5][0] = c * y; g[5][1] = c * x; g[5][2] = 0.f;
      g[6][0] = -HGB_SQ5 * x; g[6][1] = 2.f * HGB_SQ5 * y; g[6][2] = -HGB_SQ5 * z;
      g[7][0] = 0.f; g[7][1] = c * z; g[7][2] = c * y;
      g[8][0] = -c * x; g[8][1] = 0.f; g[8][2] = c * z;
    }
  }
  if (lmax >= 3) {
    const float c1 = HGB_SQ7 * 0.9128709291752769f * HGB_SQ3;   // sqrt(7) sqrt(5/6) sqrt(3)
    const float c2 = HGB_SQ7 * HGB_SQ5 * HGB_SQ3;               // sqrt(7) sqrt(5) sqrt(3)
    const float c3 = HGB_SQ7 * 0.6123724356957945f;             // sqrt(7) sqrt(3/8)
    const float c4 = HGB_SQ7 * 0.5f;
    const float x2 = x * x, y2 = y * y, z2 = z * z;
    sh[9] = c1 * (1.5f * x * z2 - 0.5f * x * x2);
    sh[10] = c2 * x * y * z;
    sh[11] = c3 * x * (4.f * y2 - x2 - z2);
    sh[12] = c4 * y * (2.f * y2 - 3.f * (x2 + z2));
    sh[13] = c3 * z * (4.f * y2 - x2 - z2);
    sh[14] = 0.5f * c2 * y * (z2 - x2);
    sh[15] = c1 * (0.5f * z * z2 - 1.5f * x2 * z);
    if (GRAD) {
      g[9][0] = c1 * 1.5f * (z2 - x2); g[9][1] = 0.f; g[9][2] = c1 * 3.f * x * z;
      g[10][0] = c2 * y * z; g[10][1] = c2 * x * z; g[10][2] = c2 * x * y;
      g[11][0] = c3 * (4.f * y2 - 3.f * x2 - z2); g[11][1] = c3 * 8.f * x * y; g[11][2] = -c3 * 2.f * x * z;
      g[12][0] = -c4 * 6.f * x * y; g[12][1] = c4 * (6.f * y2 - 3.f * x2 - 3.f * z2); g[12][2] = -c4 * 6.f * y * z;
      g[13][0] = -c3 * 2.f * x * z; g[13][1] = c3 * 8.f * y * z; g[13][2] = c3 * (4.f * y2 - x2 - 3.f * z2);
      g[14][0] = -c2 * x * y; g[14][1] = 0.5f * c2 * (z2 - x2); g[14][2] = c2 * y * z;
      g[15][0] = -c1 * 3.f * x * z; g[15][1] = 0.f; g[15][2] = c1 * 1.5f * (z2 - x2);
    }
  }
}

__device__ __forceinline__ void edge_vec(const float* __restrict__ pos, const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                         const float* __restrict__ shifts, int64_t i, float& vx, float& vy, float& vz) {
  const int r = row[i], c = col[i];
  vx = pos[3 * c] - pos[3 * r]; vy = pos[3 * c + 1] - pos[3 * r + 1]; vz = pos[3 * c + 2] - pos[3 * r + 2];
  if (shifts) { vx += shifts[3 * i]; vy += shifts[3 * i + 1]; vz += shifts[3 * i + 2]; }
}

// polynomial cutoff envelope and its derivative with respect to d (zero beyond r_max)
__device__ __forceinline__ void poly_cutoff(float d, float rc, float p, float& env, float& denv) {
  if (d >= rc) { env = 0.f; denv = 0.f; return; }
  const float x = d / rc;
  const float xp = powf(x, p), xm = powf(x, p - 1.f);
  const float a = (p + 1.f) * (p + 2.f) * 0.5f, b = p * (p + 2.f), c = p * (p + 1.f) * 0.5f;
  env = 1.f - a * xp + b * xp * x - c * xp * x * x;
  denv = (-a * p * xm + b * (p + 1.f) * xp - c * (p + 2.f) * xp * x) / rc;
}

// ---- distance transforms (mace_utils/modules/radial.py:151-245; blocks.py:141-177) ------------------------------------
// t = T(d, r0_e) with r0_e from the covalent radii of the edge's two elements.  radii [119] (index = atomic number Z, the
// element index z + 1) and the parameters are device buffers of the model, read at run time: a loaded state dict or an
// optimiser-free in-place change reaches a captured step.
//   Agnesi (c0 = q, c1 = p, c2 = a):  r0 = (R_u + R_v) / 2,  u = d / r0,  T = 1 / (1 + a u^q / (1 + u^(q-p)))
//   Soft   (c0 = a, c1 = b):          r0 = (R_u + R_v) / 4,  u = d / r0,  T = d + tanh(-u - a u^b) / 2 + 1 / 2
// dt_eval returns T, T' = dT/dd and (ORDER 2) T'' for one edge.  Agnesi is evaluated as f = a u^q sigma_w with the smaller
// of u^(q-p) and u^(p-q) in the denominator, so u^(q-p) never overflows: at d -> 0 T -> 1, T' -> 0, T'' -> 0, all finite.
constexpr int DT_RADII = 119;

__device__ __forceinline__ float dt_radius(const float* sr, const int64_t* __restrict__ z, int node) {
  const int64_t k = z[node];
  return sr[1 + (int)(k < 0 ? 0 : (k > DT_RADII - 2 ? DT_RADII - 2 : k))];   // element index 0..117 -> Z 1..118
}

template <int ORDER>
__device__ __forceinline__ void dt_eval(int kind, float d, float rsum, float c0, float c1, float c2, float& t, float& t1, float& t2) {
  if (kind == HGB_DT_AGNESI) {
    const float q = c0, p = c1, a = c2, r0 = 0.5f * rsum;
    const float u = d / r0;
    // sig = 1 / (1 + u^(p-q)) = u^(q-p) / (1 + u^(q-p)) and f / u^k = a u^(q-k) / (1 + u^(q-p)), k = 0, 1, 2
    float sig, f, fu1, fu2;
    if ((q - p) * logf(u) > 0.f) {               // u^(q-p) > 1 (small u): divide through by it
      const float s = powf(u, p - q);
      sig = 1.f / (1.f + s);
      f = a * powf(u, p) * sig;
      fu1 = a * powf(u, p - 1.f) * sig;
      fu2 = a * powf(u, p - 2.f) * sig;
    } else {
      const float w = powf(u, q - p), den = 1.f / (1.f + w);
      sig = w * den;
      f = a * powf(u, q) * den;
      fu1 = a * powf(u, q - 1.f) * den;
      fu2 = a * powf(u, q - 2.f) * den;
    }
    const float tt = 1.f / (1.f + f);
    const float g = q + (p - q) * sig;            // u f_u / f
    const float fd = fu1 * g / r0;                // df/dd
    t = tt;
    t1 = -tt * tt * fd;
    if (ORDER >= 2) {
      const float fdd = fu2 * (g * g - g - (p - q) * (p - q) * sig * (1.f - sig)) / (r0 * r0);
      t2 = tt * tt * (2.f * tt * fd * fd - fdd);
    }
  } else {
    const float a = c0, b = c1, r0 = 0.25f * rsum;
    const float u = d / r0;
    const float v = -u - a * powf(u, b);
    const float ev = expf(-2.f * fabsf(v));       // tanh and sech^2 from exp(-2|v|): no cancellation in 1 -/+ tanh
    const float inv1 = 1.f / (1.f + ev);
    const float th = copysignf((1.f - ev) * inv1, v);
    const float sech2 = 4.f * ev * inv1 * inv1;
    t = d + (v < 0.f ? ev * inv1 : inv1);         // d + (1 + tanh v) / 2
    if (sech2 > 0.f) {                            // else tanh is flat: T' = 1, T'' = 0 (never 0 * inf)
      const float dv = -(1.f + a * b * powf(u, b - 1.f)) / r0;
      t1 = fmaf(0.5f * sech2, dv, 1.f);
      if (ORDER >= 2) t2 = 0.5f * sech2 * (-a * b * (b - 1.f) * powf(u, b - 2.f) / (r0 * r0) - 2.f * th * dv * dv);
    } else {
      t1 = 1.f;
      if (ORDER >= 2) t2 = 0.f;
    }
  }
}

// transform operands of one launch: kind 0 = none (the original kernels), else the radii table staged in shared memory
struct DtArgs {
  int kind;
  const int64_t* z;
  const float* radii;
  const float* c0;
  const float* c1;
  const float* c2;
};

__device__ __forceinline__ void dt_stage(const DtArgs& ta, float* sr, float& c0, float& c1, float& c2) {
  for (int q = threadIdx.x; q < DT_RADII; q += blockDim.x) sr[q] = ta.radii[q];
  c0 = *ta.c0;
  c1 = *ta.c1;
  c2 = ta.kind == HGB_DT_AGNESI ? *ta.c2 : 0.f;
  __syncthreads();
}

// Bessel basis (of t = d, or of the transformed length) times the polynomial cutoff of the raw d, blocks.py:172-177
template <bool DT>
__device__ __forceinline__ void edge_embed_fwd_body(const float* __restrict__ pos, const int32_t* __restrict__ row,
                                                    const int32_t* __restrict__ col, const float* __restrict__ shifts, int64_t e,
                                                    int lmax, int nb, float rc, float p, const DtArgs& ta, float* sr,
                                                    float* __restrict__ sh, float* __restrict__ radial) {
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (DT) dt_stage(ta, sr, c0, c1, c2);
  const int ns = (lmax + 1) * (lmax + 1);
  const float pref = sqrtf(2.f / rc);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    float vx, vy, vz;
    edge_vec(pos, row, col, shifts, i, vx, vy, vz);
    const float d = sqrtf(vx * vx + vy * vy + vz * vz);
    const float inv = 1.f / fmaxf(d, 1e-12f);
    float s[16];
    sh_eval<false>(lmax, vx * inv, vy * inv, vz * inv, s, nullptr);
    for (int k = 0; k < ns; ++k) sh[i * ns + k] = s[k];
    float env, denv;
    poly_cutoff(d, rc, p, env, denv);
    float t = d, tinv = inv;
    if (DT) {
      float t1, t2;
      dt_eval<1>(ta.kind, d, dt_radius(sr, ta.z, row[i]) + dt_radius(sr, ta.z, col[i]), c0, c1, c2, t, t1, t2);
      tinv = 1.f / t;
    }
    for (int n = 0; n < nb; ++n) radial[i * nb + n] = pref * sinf((float)(n + 1) * HGB_PI_F / rc * t) * tinv * env;
  }
}

template <bool DT>
__device__ __forceinline__ void edge_embed_bwd_body(const float* __restrict__ pos, const int32_t* __restrict__ row,
                                                    const int32_t* __restrict__ col, const float* __restrict__ shifts,
                                                    const float* __restrict__ g_sh, const float* __restrict__ g_radial, int64_t e,
                                                    int lmax, int nb, float rc, float p, const DtArgs& ta, float* sr,
                                                    float* __restrict__ g_vec) {
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (DT) dt_stage(ta, sr, c0, c1, c2);
  const int ns = (lmax + 1) * (lmax + 1);
  const float pref = sqrtf(2.f / rc);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    float vx, vy, vz;
    edge_vec(pos, row, col, shifts, i, vx, vy, vz);
    const float d = sqrtf(vx * vx + vy * vy + vz * vz);
    const float inv = 1.f / fmaxf(d, 1e-12f);
    const float ux = vx * inv, uy = vy * inv, uz = vz * inv;
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (g_sh) {
      float s[16], g[16][3];
      sh_eval<true>(lmax, ux, uy, uz, s, g);
      float ax = 0.f, ay = 0.f, az = 0.f;            // d L / d u (unconstrained)
      for (int k = 1; k < ns; ++k) {
        const float w = g_sh[i * ns + k];
        ax = fmaf(w, g[k][0], ax); ay = fmaf(w, g[k][1], ay); az = fmaf(w, g[k][2], az);
      }
      const float dot = ax * ux + ay * uy + az * uz;  // u = vec / d:  d u / d vec = (I - u u^T) / d
      gx = (ax - dot * ux) * inv; gy = (ay - dot * uy) * inv; gz = (az - dot * uz) * inv;
    }
    if (g_radial) {
      float env, denv;
      poly_cutoff(d, rc, p, env, denv);
      float t = d, tinv = inv, t1 = 1.f;
      if (DT) {
        float t2;
        dt_eval<1>(ta.kind, d, dt_radius(sr, ta.z, row[i]) + dt_radius(sr, ta.z, col[i]), c0, c1, c2, t, t1, t2);
        tinv = 1.f / t;
      }
      float gd = 0.f;
      for (int n = 0; n < nb; ++n) {
        const float w = (float)(n + 1) * HGB_PI_F / rc;
        float sn, cs;
        sincosf(w * t, &sn, &cs);
        const float bes = pref * sn * tinv;
        const float dbes = pref * (w * cs * tinv - sn * tinv * tinv);
        // chain term basis'(t) T'(d) cutoff(d) (zero where the cutoff is) + basis(t) cutoff'(d)
        gd = fmaf(g_radial[i * nb + n], (DT ? dbes * t1 : dbes) * env + bes * denv, gd);
      }
      gx = fmaf(gd, ux, gx); gy = fmaf(gd, uy, gy); gz = fmaf(gd, uz, gz);
    }
    g_vec[3 * i] = gx; g_vec[3 * i + 1] = gy; g_vec[3 * i + 2] = gz;
  }
}

__global__ void mace_edge_embed_fwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                           const float* __restrict__ shifts, int64_t e, int lmax, int nb, float rc, float p,
                                           float* __restrict__ sh, float* __restrict__ radial) {
  edge_embed_fwd_body<false>(pos, row, col, shifts, e, lmax, nb, rc, p, DtArgs{}, nullptr, sh, radial);
}

__global__ void mace_edge_embed_bwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                           const float* __restrict__ shifts, const float* __restrict__ g_sh,
                                           const float* __restrict__ g_radial, int64_t e, int lmax, int nb, float rc, float p,
                                           float* __restrict__ g_vec) {
  edge_embed_bwd_body<false>(pos, row, col, shifts, g_sh, g_radial, e, lmax, nb, rc, p, DtArgs{}, nullptr, g_vec);
}

__global__ void mace_edge_embed_dt_fwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                              const float* __restrict__ shifts, int64_t e, int lmax, int nb, float rc, float p, DtArgs ta,
                                              float* __restrict__ sh, float* __restrict__ radial) {
  __shared__ float sr[DT_RADII];
  edge_embed_fwd_body<true>(pos, row, col, shifts, e, lmax, nb, rc, p, ta, sr, sh, radial);
}

__global__ void mace_edge_embed_dt_bwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                              const float* __restrict__ shifts, const float* __restrict__ g_sh,
                                              const float* __restrict__ g_radial, int64_t e, int lmax, int nb, float rc, float p, DtArgs ta,
                                              float* __restrict__ g_vec) {
  __shared__ float sr[DT_RADII];
  edge_embed_bwd_body<true>(pos, row, col, shifts, g_sh, g_radial, e, lmax, nb, rc, p, ta, sr, g_vec);
}

// out[i] = (g ? g[i] : 1) * T^(order)(d[i]) for order 0, 1, 2
__global__ void mace_dist_transform_kernel(int order, const float* __restrict__ d, const float* __restrict__ g, const int32_t* __restrict__ row,
                                           const int32_t* __restrict__ col, int64_t e, DtArgs ta, float* __restrict__ out) {
  __shared__ float sr[DT_RADII];
  float c0, c1, c2;
  dt_stage(ta, sr, c0, c1, c2);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    float t, t1, t2 = 0.f;
    dt_eval<2>(ta.kind, d[i], dt_radius(sr, ta.z, row[i]) + dt_radius(sr, ta.z, col[i]), c0, c1, c2, t, t1, t2);
    const float v = order == 0 ? t : (order == 1 ? t1 : t2);
    out[i] = g ? g[i] * v : v;
  }
}

}  // namespace

extern "C" int hgb_mace_edge_embed_fwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, int64_t e,
                                       int32_t lmax, int32_t num_bessel, float r_max, float p, float* sh, float* radial,
                                       hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && lmax >= 0 && lmax <= 3 && num_bessel >= 1 && num_bessel <= 64 && r_max > 0.f, "mace_edge_embed_fwd: bad arguments");
  if (e == 0) return HGB_OK;   // no edges: no kernel runs (the arrays may then be NULL)
  HGB_REQUIRE(pos && row && col && sh && radial, "mace_edge_embed_fwd: bad arguments");
  mace_edge_embed_fwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(pos, row, col, shifts, e, lmax, num_bessel, r_max, p, sh, radial);
  HGB_LAUNCH_CHECK("mace_edge_embed_fwd");
  return HGB_OK;
}

extern "C" int hgb_mace_edge_embed_bwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, const float* g_sh,
                                       const float* g_radial, int64_t e, int32_t lmax, int32_t num_bessel, float r_max, float p,
                                       float* g_vec, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && lmax >= 0 && lmax <= 3 && num_bessel >= 1 && num_bessel <= 64 && r_max > 0.f, "mace_edge_embed_bwd: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(pos && row && col && g_vec, "mace_edge_embed_bwd: bad arguments");
  mace_edge_embed_bwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(pos, row, col, shifts, g_sh, g_radial, e, lmax, num_bessel,
                                                                                    r_max, p, g_vec);
  HGB_LAUNCH_CHECK("mace_edge_embed_bwd");
  return HGB_OK;
}

static bool dt_args_ok(int32_t kind, const int64_t* z, const float* radii, const float* c0, const float* c1, const float* c2) {
  return (kind == HGB_DT_AGNESI || kind == HGB_DT_SOFT) && z && radii && c0 && c1 && (kind != HGB_DT_AGNESI || c2);
}

extern "C" int hgb_mace_edge_embed_dt_fwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, const int64_t* z,
                                          int64_t e, int32_t lmax, int32_t num_bessel, float r_max, float p, int32_t kind,
                                          const float* radii, const float* c0, const float* c1, const float* c2, float* sh, float* radial,
                                          hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && lmax >= 0 && lmax <= 3 && num_bessel >= 1 && num_bessel <= 64 && r_max > 0.f &&
                  (kind == HGB_DT_AGNESI || kind == HGB_DT_SOFT),
              "mace_edge_embed_dt_fwd: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(pos && row && col && sh && radial && dt_args_ok(kind, z, radii, c0, c1, c2), "mace_edge_embed_dt_fwd: bad arguments");
  mace_edge_embed_dt_fwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(pos, row, col, shifts, e, lmax, num_bessel, r_max, p,
                                                                                       DtArgs{kind, z, radii, c0, c1, c2}, sh, radial);
  HGB_LAUNCH_CHECK("mace_edge_embed_dt_fwd");
  return HGB_OK;
}

extern "C" int hgb_mace_edge_embed_dt_bwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, const int64_t* z,
                                          const float* g_sh, const float* g_radial, int64_t e, int32_t lmax, int32_t num_bessel, float r_max,
                                          float p, int32_t kind, const float* radii, const float* c0, const float* c1, const float* c2,
                                          float* g_vec, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && lmax >= 0 && lmax <= 3 && num_bessel >= 1 && num_bessel <= 64 && r_max > 0.f &&
                  (kind == HGB_DT_AGNESI || kind == HGB_DT_SOFT),
              "mace_edge_embed_dt_bwd: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(pos && row && col && g_vec && dt_args_ok(kind, z, radii, c0, c1, c2), "mace_edge_embed_dt_bwd: bad arguments");
  mace_edge_embed_dt_bwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(pos, row, col, shifts, g_sh, g_radial, e, lmax,
                                                                                       num_bessel, r_max, p, DtArgs{kind, z, radii, c0, c1, c2},
                                                                                       g_vec);
  HGB_LAUNCH_CHECK("mace_edge_embed_dt_bwd");
  return HGB_OK;
}

extern "C" int hgb_mace_dist_transform(int32_t order, int32_t kind, const float* d, const float* g, const int32_t* row, const int32_t* col,
                                       const int64_t* z, const float* radii, const float* c0, const float* c1, const float* c2, int64_t e,
                                       float* out, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && order >= 0 && order <= 2 && (kind == HGB_DT_AGNESI || kind == HGB_DT_SOFT), "mace_dist_transform: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(d && row && col && out && dt_args_ok(kind, z, radii, c0, c1, c2), "mace_dist_transform: bad arguments");
  mace_dist_transform_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(order, d, g, row, col, e, DtArgs{kind, z, radii, c0, c1, c2},
                                                                                    out);
  HGB_LAUNCH_CHECK("mace_dist_transform");
  return HGB_OK;
}
