// libhgb.so -- per-edge geometry and PaiNN's radial embedding, forward and first-order backward.
// One thread per edge; every array is touched once (HBM-bound, trivially small next to the gathers).
#include "hgb_common.cuh"

__global__ void edge_geom_fwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ row,
                                     const int32_t* __restrict__ col, const float* __restrict__ shifts, int64_t e,
                                     float eps, float* __restrict__ vec, float* __restrict__ len, float* __restrict__ unit) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = row[i], c = col[i];
    float vx = pos[3 * c] - pos[3 * r], vy = pos[3 * c + 1] - pos[3 * r + 1], vz = pos[3 * c + 2] - pos[3 * r + 2];
    if (shifts) { vx += shifts[3 * i]; vy += shifts[3 * i + 1]; vz += shifts[3 * i + 2]; }
    const float l = sqrtf(vx * vx + vy * vy + vz * vz);
    if (vec) { vec[3 * i] = vx; vec[3 * i + 1] = vy; vec[3 * i + 2] = vz; }
    if (len) len[i] = l;
    if (unit) {
      const float inv = 1.f / (l + eps);
      unit[3 * i] = vx * inv; unit[3 * i + 1] = vy * inv; unit[3 * i + 2] = vz * inv;
    }
  }
}

extern "C" int hgb_edge_geom_fwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, int64_t e,
                                 float eps, float* vec, float* len, float* unit, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0, "edge_geom_fwd: bad arguments");
  if (e == 0) return HGB_OK;   // no edges: no kernel runs (the arrays may then be NULL)
  HGB_REQUIRE(pos && row && col, "edge_geom_fwd: bad arguments");
  edge_geom_fwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(pos, row, col, shifts, e, eps, vec, len, unit);
  HGB_LAUNCH_CHECK("edge_geom_fwd");
  return HGB_OK;
}

// unit_k = vec_k / L, L = len + eps:  d unit_k / d vec_m = delta_km / L - vec_k vec_m / (L^2 len)
__global__ void edge_geom_bwd_kernel(const float* __restrict__ vec, const float* __restrict__ len, float eps,
                                     const float* __restrict__ g_vec_in, const float* __restrict__ g_len,
                                     const float* __restrict__ g_unit, int64_t e, float* __restrict__ g_vec) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    const float vx = vec[3 * i], vy = vec[3 * i + 1], vz = vec[3 * i + 2];
    const float l = len[i];
    const float il = l > 0.f ? 1.f / l : 0.f;  // subgradient 0 at the origin, as torch.linalg.norm does
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (g_vec_in) { gx = g_vec_in[3 * i]; gy = g_vec_in[3 * i + 1]; gz = g_vec_in[3 * i + 2]; }
    float radial = g_len ? g_len[i] * il : 0.f;  // coefficient of vec
    if (g_unit) {
      const float ux = g_unit[3 * i], uy = g_unit[3 * i + 1], uz = g_unit[3 * i + 2];
      const float iL = 1.f / (l + eps);
      gx += ux * iL; gy += uy * iL; gz += uz * iL;
      radial -= (ux * vx + uy * vy + uz * vz) * iL * iL * il;
    }
    g_vec[3 * i] = gx + radial * vx; g_vec[3 * i + 1] = gy + radial * vy; g_vec[3 * i + 2] = gz + radial * vz;
  }
}

extern "C" int hgb_edge_geom_bwd(const float* vec, const float* len, float eps, const float* g_vec_in, const float* g_len,
                                 const float* g_unit, int64_t e, float* g_vec, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0, "edge_geom_bwd: bad arguments");
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(vec && len && g_vec, "edge_geom_bwd: bad arguments");
  edge_geom_bwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(vec, len, eps, g_vec_in, g_len, g_unit, e, g_vec);
  HGB_LAUNCH_CHECK("edge_geom_bwd");
  return HGB_OK;
}

// ---- PaiNN radial embedding --------------------------------------------------------------------
#define HGB_PI 3.14159265358979323846f

// epack [e,12] = { sin(n pi d / rc)/d * fcut for n = 1..r (zero padded to 8), fcut, unit/d (x, y, z) }
__global__ void painn_edge_embed_fwd_kernel(const float* __restrict__ unit, const float* __restrict__ len, int64_t e, int r,
                                            float cutoff, float* __restrict__ epack) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = len[i];
    const float id = 1.f / d;
    const float cut = d < cutoff ? 0.5f * (cosf(HGB_PI * d / cutoff) + 1.f) : 0.f;
    float o[12];
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = q < r ? sinf(d * (float)(q + 1) * HGB_PI / cutoff) * id * cut : 0.f;
    o[8] = cut;
    o[9] = unit[3 * i] * id; o[10] = unit[3 * i + 1] * id; o[11] = unit[3 * i + 2] * id;
    float4* op = reinterpret_cast<float4*>(epack + i * 12);
    op[0] = make_float4(o[0], o[1], o[2], o[3]); op[1] = make_float4(o[4], o[5], o[6], o[7]); op[2] = make_float4(o[8], o[9], o[10], o[11]);
  }
}

extern "C" int hgb_painn_edge_embed_fwd(const float* unit, const float* len, int64_t e, int32_t r, float cutoff, float* epack,
                                        hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && r > 0 && r <= 8, "painn_edge_embed_fwd: bad arguments (0 < num_radial <= 8, got %d)", r);
  if (e == 0) return HGB_OK;   // no edges: no kernel runs (the arrays may then be NULL)
  HGB_REQUIRE(unit && len && epack && (uintptr_t)epack % 16 == 0, "painn_edge_embed_fwd: null pointer or epack not 16-byte aligned");
  painn_edge_embed_fwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(unit, len, e, r, cutoff, epack);
  HGB_LAUNCH_CHECK("painn_edge_embed_fwd");
  return HGB_OK;
}

__global__ void painn_edge_embed_bwd_kernel(const float* __restrict__ unit, const float* __restrict__ len,
                                            const float* __restrict__ g_epack, int64_t e, int r, float cutoff,
                                            float* __restrict__ g_unit, float* __restrict__ g_len) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = len[i];
    const float id = 1.f / d;
    const float* g = g_epack + i * 12;
    const float gx = g[9], gy = g[10], gz = g[11];
    g_unit[3 * i] = gx * id; g_unit[3 * i + 1] = gy * id; g_unit[3 * i + 2] = gz * id;
    float gl = -(gx * unit[3 * i] + gy * unit[3 * i + 1] + gz * unit[3 * i + 2]) * id * id;
    const bool in = d < cutoff;
    const float w = HGB_PI / cutoff;
    const float cut = in ? 0.5f * (cosf(w * d) + 1.f) : 0.f;
    const float dcut = in ? -0.5f * w * sinf(w * d) : 0.f;
    gl += g[8] * dcut;
    for (int q = 0; q < r; ++q) {
      const float a = (float)(q + 1) * w;
      float sn, cs;
      sincosf(a * d, &sn, &cs);
      const float sinc = sn * id;
      const float dsinc = (a * cs - sinc) * id;
      gl += g[q] * (dsinc * cut + sinc * dcut);
    }
    g_len[i] = gl;
  }
}

extern "C" int hgb_painn_edge_embed_bwd(const float* unit, const float* len, const float* g_epack, int64_t e, int32_t r, float cutoff,
                                        float* g_unit, float* g_len, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && r > 0 && r <= 8, "painn_edge_embed_bwd: bad arguments (0 < num_radial <= 8, got %d)", r);
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(unit && len && g_epack && g_unit && g_len, "painn_edge_embed_bwd: null pointer");
  painn_edge_embed_bwd_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(unit, len, g_epack, e, r, cutoff, g_unit, g_len);
  HGB_LAUNCH_CHECK("painn_edge_embed_bwd");
  return HGB_OK;
}
