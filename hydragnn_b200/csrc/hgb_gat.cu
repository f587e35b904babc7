// GATv2Conv fused (hydragnn/models/GATStack.py:175-205; torch_geometric 2.6.1 GATv2Conv with add_self_loops=True,
// fill_value="mean", share_weights=False, residual=False).  One pass over the by-target CSR with an online (flash-style) softmax
// per head: no [E, H*C] tensor (x_i + x_j, lin_edge(a), leaky_relu, the messages) is ever written.
//
// For the edge j -> i (i the target) with attribute a_e:  z = x_r[i] + x_l[j] + mt^T a_e,  s_h = sum_c leaky_relu(z_hc) att_hc,
// alpha = softmax_i(s) over the in-edges of i plus its self-loop, out[i] = sum alpha keep / (1 - p) x_l[j] (concat: [n, H*C];
// mean: averaged over the heads), + bias.  Input edges with src == dst are skipped (remove_self_loops); every node then gets
// one self-loop whose attribute is the mean of its remaining in-edges' attributes (0 without any), processed last.
//
// Thread mapping: a group of G lanes owns one target (G the power of two >= the number of VEC-wide channel vectors, at most
// 32); lane sub owns the vectors t G + sub, t < NV.  The head scores are group sums through a fixed xor tree, so every lane
// holds every head's score and the online max / sum of each head.  A lane's channel set is fixed and it walks the edges in
// CSR order (ascending edge id), so the result is the same function of the input on every run: no atomics.
//
// Dropout on alpha (after normalisation, as PyG applies it): keep(seed, edge id, head) is one Philox4x32-10 draw, the
// self-loop of node i has edge id e + i, so the mask does not depend on CSR order.  The seed is read on the device.
#include "hgb_common.cuh"

#define GAT_MAX_H 8
#define GAT_MAX_HC 512
#define GAT_MAX_D 16
#define GAT_BWD_MAX_BLOCKS (HGB_NUM_SMS * 4)
#define GAT_SMEM_LIMIT (200 * 1024)

// ---- Philox4x32-10 keep mask ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 gat_philox(uint4 x, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * x.x, hi0 = __umulhi(0xD2511F53u, x.x);
    const uint32_t lo1 = 0xCD9E8D57u * x.z, hi1 = __umulhi(0xCD9E8D57u, x.z);
    x = make_uint4(hi1 ^ x.y ^ k.x, lo1, hi0 ^ x.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return x;
}

// the four 32-bit draws for heads 4 q .. 4 q + 3 of edge id eid
__device__ __forceinline__ uint4 gat_draw4(uint64_t seed, int64_t eid, int q) {
  return gat_philox(make_uint4((uint32_t)eid, (uint32_t)((uint64_t)eid >> 32), (uint32_t)q, 0x47415476u),
                    make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}

// keep factor 1 / (1 - p) where the uniform draw (the top 24 bits) is >= p, else 0
__device__ __forceinline__ float gat_keep1(uint32_t w, float p, float inv) {
  return ((float)(w >> 8) * (1.0f / 16777216.0f)) >= p ? inv : 0.f;
}

__device__ __forceinline__ void gat_keep(uint64_t seed, int64_t eid, int heads, float p, float (&kf)[GAT_MAX_H]) {
  if (p <= 0.f) {
#pragma unroll
    for (int h = 0; h < GAT_MAX_H; ++h) kf[h] = 1.f;
    return;
  }
  const float inv = 1.f / (1.f - p);
  const uint4 a = gat_draw4(seed, eid, 0);
  kf[0] = gat_keep1(a.x, p, inv), kf[1] = gat_keep1(a.y, p, inv), kf[2] = gat_keep1(a.z, p, inv), kf[3] = gat_keep1(a.w, p, inv);
  kf[4] = kf[5] = kf[6] = kf[7] = inv;
  if (heads > 4) {
    const uint4 b = gat_draw4(seed, eid, 1);
    kf[4] = gat_keep1(b.x, p, inv), kf[5] = gat_keep1(b.y, p, inv), kf[6] = gat_keep1(b.z, p, inv), kf[7] = gat_keep1(b.w, p, inv);
  }
}

// ---- per-lane channel slots ---------------------------------------------------------------------------------------------
template <int VEC>
__device__ __forceinline__ void gat_ld(const float* __restrict__ p, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
  } else {
    v[0] = __ldg(p);
  }
}

template <int VEC>
__device__ __forceinline__ void gat_st(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else p[0] = v[0];
}

// the value of a per-head register array at a runtime head (a select chain: no local memory)
__device__ __forceinline__ float gat_pick(const float (&a)[GAT_MAX_H], int h) {
  float r = a[0];
#pragma unroll
  for (int k = 1; k < GAT_MAX_H; ++k) r = (h == k) ? a[k] : r;
  return r;
}

// sum over the G lanes of a group (xor tree: every lane of the group gets the same bits)
__device__ __forceinline__ float gat_group_sum(float v, int G) {
  for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int VEC, int NV>
struct GatSlots {
  int ch[NV];   // first channel of the slot (clamped to 0 where the lane has none)
  int hs[NV];   // head of the slot; GAT_MAX_H where the lane has none
  __device__ __forceinline__ GatSlots(int sub, int G, int hc, int c) {
#pragma unroll
    for (int t = 0; t < NV; ++t) {
      const int k = (t * G + sub) * VEC;
      ch[t] = k < hc ? k : 0;
      hs[t] = k < hc ? k / c : GAT_MAX_H;
    }
  }
};

// per-head group sums of per-slot values
template <int VEC, int NV>
__device__ __forceinline__ void gat_head_sums(const GatSlots<VEC, NV>& S, const float (&v)[NV][VEC], int heads, int G,
                                              float (&out)[GAT_MAX_H]) {
#pragma unroll
  for (int h = 0; h < GAT_MAX_H; ++h) {
    out[h] = 0.f;
    if (h < heads) {
      float p = 0.f;
#pragma unroll
      for (int t = 0; t < NV; ++t)
        if (S.hs[t] == h) {
#pragma unroll
          for (int u = 0; u < VEC; ++u) p += v[t][u];
        }
      out[h] = gat_group_sum(p, G);
    }
  }
}

// z = (x_r[i] + x_l[j]) + mt^T a with a = arow[k] / adiv (a row of eattr over 1, or for the self-loop the attribute sum of
// the target's in-edges over their count, as PyG's scatter mean divides), and the per-slot score terms leaky_relu(z) att.  Forward and both backward passes call
// it, so the backward sees the forward's z bit for bit.
template <int VEC, int NV>
__device__ __forceinline__ void gat_z(const GatSlots<VEC, NV>& S, const float (&xr)[NV][VEC], const float (&xl)[NV][VEC],
                                      const float* smt, const float* satt, int hc, int d, const float* arow, float adiv,
                                      float slope, float (&z)[NV][VEC], float (&sv)[NV][VEC]) {
  float ea[NV][VEC];
#pragma unroll
  for (int t = 0; t < NV; ++t)
#pragma unroll
    for (int u = 0; u < VEC; ++u) ea[t][u] = 0.f;
  for (int k = 0; k < d; ++k) {
    const float a = arow[k] / adiv;
#pragma unroll
    for (int t = 0; t < NV; ++t)
#pragma unroll
      for (int u = 0; u < VEC; ++u) ea[t][u] = fmaf(smt[k * hc + S.ch[t] + u], a, ea[t][u]);
  }
#pragma unroll
  for (int t = 0; t < NV; ++t)
#pragma unroll
    for (int u = 0; u < VEC; ++u) {
      z[t][u] = (xr[t][u] + xl[t][u]) + ea[t][u];
      const float lr = z[t][u] > 0.f ? z[t][u] : z[t][u] * slope;
      sv[t][u] = S.hs[t] < GAT_MAX_H ? lr * satt[S.ch[t] + u] : 0.f;
    }
}

template <int VEC, int NV>
__device__ __forceinline__ void gat_ld_row(const GatSlots<VEC, NV>& S, const float* __restrict__ row, float (&v)[NV][VEC]) {
#pragma unroll
  for (int t = 0; t < NV; ++t) gat_ld<VEC>(row + S.ch[t], v[t]);
}

__device__ __forceinline__ void gat_stage(float* sm, const float* __restrict__ mt, const float* __restrict__ att, int hc, int d) {
  const int nm = d * hc;
  for (int t = threadIdx.x; t < nm + hc; t += blockDim.x) sm[t] = t < nm ? __ldg(mt + t) : __ldg(att + t - nm);
}

// ---- forward --------------------------------------------------------------------------------------------------------------
// shared: mt [d, hc], att [hc], per group the attribute sum of its target's in-edges [GAT_MAX_D] and in mean mode a [hc] row
// for the head average.  A group's shared entries are written by its lane 0 and read after a __syncwarp (the row and edge
// loops are warp-uniform).
template <int VEC, int NV>
__global__ void __launch_bounds__(256, 1) gat_fwd_kernel(
    const float* __restrict__ xlr, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm,
    const int32_t* __restrict__ src, const float* __restrict__ eattr, int d, const float* __restrict__ mt,
    const float* __restrict__ att, const float* __restrict__ bias, int n, int e, int heads, int c, int concat, float slope,
    float p, const int64_t* __restrict__ seed_ptr, int gl2, float* __restrict__ out, float* __restrict__ lse) {
  extern __shared__ float gat_sm[];
  const int hc = heads * c;
  const float* smt = gat_sm;
  const float* satt = gat_sm + d * hc;
  gat_stage(gat_sm, mt, att, hc, d);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int G = 1 << gl2, sub = lane & (G - 1), gpw = 32 >> gl2;
  const int grp = warp * gpw + (lane >> gl2);
  float* sattr = gat_sm + (d + 1) * hc + grp * GAT_MAX_D;
  float* srow = gat_sm + (d + 1) * hc + nwarps * gpw * GAT_MAX_D + grp * hc;
  const uint64_t seed = (p > 0.f) ? (uint64_t)*seed_ptr : 0ull;
  const GatSlots<VEC, NV> S(sub, G, hc, c);
  const int64_t ld = 2 * (int64_t)hc;
  for (int first = (blockIdx.x * nwarps + warp) * gpw; first < n; first += gridDim.x * nwarps * gpw) {
    const int row = first + (lane >> gl2);
    const bool rv = row < n;
    const int rr = rv ? row : 0;
    const int lo = rowptr[rr], len = rv ? rowptr[rr + 1] - lo : 0;
    const int maxlen = (int)__reduce_max_sync(0xffffffffu, (unsigned)(len + 1));
    float xr[NV][VEC], acc[NV][VEC], m[GAT_MAX_H], l[GAT_MAX_H];
    gat_ld_row(S, xlr + rr * ld + hc, xr);
#pragma unroll
    for (int t = 0; t < NV; ++t)
#pragma unroll
      for (int u = 0; u < VEC; ++u) acc[t][u] = 0.f;
#pragma unroll
    for (int h = 0; h < GAT_MAX_H; ++h) m[h] = -INFINITY, l[h] = 0.f;
    __syncwarp();
    if (sub == 0)
      for (int k = 0; k < d; ++k) sattr[k] = 0.f;
    int cnt = 0;
    for (int it = 0; it < maxlen; ++it) {
      __syncwarp();
      const bool loop = it == len;
      const int q = lo + it;
      const int j = loop ? rr : (it < len ? src[q] : rr);
      const int eid = (it < len) ? (perm ? perm[q] : q) : 0;
      const bool ev = rv && it <= len && (loop || j != row);
      const float* arow = (it < len) ? eattr + (int64_t)eid * d : sattr;
      const float adiv = (loop && cnt > 0) ? (float)cnt : 1.f;
      float xl[NV][VEC], z[NV][VEC], sv[NV][VEC], s[GAT_MAX_H];
      gat_ld_row(S, xlr + j * ld, xl);
      gat_z<VEC, NV>(S, xr, xl, smt, satt, hc, d, arow, adiv, slope, z, sv);
      gat_head_sums<VEC, NV>(S, sv, heads, G, s);
      if (ev && !loop) {
        ++cnt;
        if (sub == 0)
          for (int k = 0; k < d; ++k) sattr[k] += __ldg(arow + k);
      }
      if (ev) {
        float kf[GAT_MAX_H], sc[GAT_MAX_H], wk[GAT_MAX_H];
        gat_keep(seed, loop ? (int64_t)e + row : (int64_t)eid, heads, p, kf);
#pragma unroll
        for (int h = 0; h < GAT_MAX_H; ++h) {
          const float mn = fmaxf(m[h], s[h]);
          sc[h] = expf(m[h] - mn);
          const float w = expf(s[h] - mn);
          l[h] = l[h] * sc[h] + w;
          m[h] = mn;
          wk[h] = w * kf[h];
        }
#pragma unroll
        for (int t = 0; t < NV; ++t) {
          const float a = gat_pick(sc, S.hs[t]), b = gat_pick(wk, S.hs[t]);
#pragma unroll
          for (int u = 0; u < VEC; ++u) acc[t][u] = fmaf(b, xl[t][u], acc[t][u] * a);
        }
      }
    }
    // normalise; lse = m + log(l) per head for the backward
    if (rv && sub < heads) {
      float v = 0.f;
#pragma unroll
      for (int h = 0; h < GAT_MAX_H; ++h)
        if (h == sub) v = m[h] + logf(l[h]);
      lse[(int64_t)row * heads + sub] = v;
    }
    float inv[GAT_MAX_H];
#pragma unroll
    for (int h = 0; h < GAT_MAX_H; ++h) inv[h] = 1.f / l[h];
    if (concat) {
      if (rv) {
#pragma unroll
        for (int t = 0; t < NV; ++t)
          if (S.hs[t] < GAT_MAX_H) {
            const float a = gat_pick(inv, S.hs[t]);
            float o[VEC];
#pragma unroll
            for (int u = 0; u < VEC; ++u) o[u] = acc[t][u] * a + __ldg(bias + S.ch[t] + u);
            gat_st<VEC>(out + (int64_t)row * hc + S.ch[t], o);
          }
      }
    } else {
#pragma unroll
      for (int t = 0; t < NV; ++t)
        if (S.hs[t] < GAT_MAX_H) {
          const float a = gat_pick(inv, S.hs[t]);
#pragma unroll
          for (int u = 0; u < VEC; ++u) srow[S.ch[t] + u] = acc[t][u] * a;
        }
      __syncwarp();
      if (rv) {
        const float rh = 1.f / (float)heads;
        for (int cc = sub; cc < c; cc += G) {
          float v = 0.f;
          for (int h = 0; h < heads; ++h) v += srow[h * c + cc];
          out[(int64_t)row * c + cc] = v * rh + __ldg(bias + cc);
        }
      }
    }
  }
}

// ---- backward pass A, by target -----------------------------------------------------------------------------------------
// Per target and head: D_h = sum_e alpha k (g_h . x_l[j]) (walk 1, which also sums the self-loop attribute), then per edge
// (walk 2, self-loop first) g_s = alpha (k (g_h . x_l[j]) - D_h), g_z = g_s att leaky_relu'(z): g_xr[i] = sum g_z; g_s and
// alpha k go to the workspace [e + n, H] for pass B, the self-loop attribute to mean_ws [n, d]; g_eattr = mt g_z (+ the edge's
// share g_loop / count of its target's self-loop mean); g_att += g_s leaky_relu(z) and g_mt += a g_z in the group's shared
// slice, summed over the CTA's groups in order into part [gridDim.x, 1 + d, hc].
template <int VEC, int NV>
__global__ void __launch_bounds__(256, 1) gat_bwd_a_kernel(
    const float* __restrict__ g_out, const float* __restrict__ xlr, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ src, const float* __restrict__ eattr, int d,
    const float* __restrict__ mt, const float* __restrict__ att, const float* __restrict__ lse, int n, int e, int heads, int c,
    int concat, float slope, float p, const int64_t* __restrict__ seed_ptr, int gl2, float* __restrict__ g_xlr,
    float* __restrict__ g_eattr, float* __restrict__ gs_ws, float* __restrict__ ak_ws, float* __restrict__ mean_ws,
    float* __restrict__ part) {
  extern __shared__ float gat_sm[];
  const int hc = heads * c;
  const float* smt = gat_sm;
  const float* satt = gat_sm + d * hc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int G = 1 << gl2, sub = lane & (G - 1), gpw = 32 >> gl2;
  const int ngrp = nwarps * gpw, grp = warp * gpw + (lane >> gl2);
  const int slice = (d + 1) * hc;
  float* sattr = gat_sm + (d + 1) * hc + grp * 2 * GAT_MAX_D;
  float* sgl = sattr + GAT_MAX_D;
  float* sacc = gat_sm + (d + 1) * hc + ngrp * 2 * GAT_MAX_D;
  gat_stage(gat_sm, mt, att, hc, d);
  if (part)
    for (int t = threadIdx.x; t < ngrp * slice; t += blockDim.x) sacc[t] = 0.f;
  __syncthreads();
  float* gacc = sacc + grp * slice;
  const uint64_t seed = (p > 0.f) ? (uint64_t)*seed_ptr : 0ull;
  const GatSlots<VEC, NV> S(sub, G, hc, c);
  const int64_t ld = 2 * (int64_t)hc;
  const float rh = concat ? 1.f : 1.f / (float)heads;
  for (int first = (blockIdx.x * nwarps + warp) * gpw; first < n; first += gridDim.x * nwarps * gpw) {
    const int row = first + (lane >> gl2);
    const bool rv = row < n;
    const int rr = rv ? row : 0;
    const int lo = rowptr[rr], len = rv ? rowptr[rr + 1] - lo : 0;
    const int maxlen = (int)__reduce_max_sync(0xffffffffu, (unsigned)(len + 1));
    float xr[NV][VEC], go[NV][VEC], lsev[GAT_MAX_H], Dh[GAT_MAX_H];
    gat_ld_row(S, xlr + rr * ld + hc, xr);
#pragma unroll
    for (int t = 0; t < NV; ++t) {
      if (concat) gat_ld<VEC>(g_out + (int64_t)rr * hc + S.ch[t], go[t]);
      else gat_ld<VEC>(g_out + (int64_t)rr * c + (S.ch[t] % c), go[t]);
#pragma unroll
      for (int u = 0; u < VEC; ++u) go[t][u] = rv ? go[t][u] * rh : 0.f;
    }
#pragma unroll
    for (int h = 0; h < GAT_MAX_H; ++h) {
      lsev[h] = (h < heads) ? __ldg(lse + (int64_t)rr * heads + h) : 0.f;
      Dh[h] = 0.f;
    }
    __syncwarp();
    if (sub == 0)
      for (int k = 0; k < d; ++k) sattr[k] = 0.f;
    int cnt = 0;
    // walk 1: D_h and the self-loop attribute (the self-loop last, as in the forward)
    for (int it = 0; it < maxlen; ++it) {
      __syncwarp();
      const bool loop = it == len;
      const int q = lo + it;
      const int j = loop ? rr : (it < len ? src[q] : rr);
      const int eid = (it < len) ? (perm ? perm[q] : q) : 0;
      const bool ev = rv && it <= len && (loop || j != row);
      const float* arow = (it < len) ? eattr + (int64_t)eid * d : sattr;
      const float adiv = (loop && cnt > 0) ? (float)cnt : 1.f;
      float xl[NV][VEC], z[NV][VEC], sv[NV][VEC], dv[NV][VEC], s[GAT_MAX_H], dot[GAT_MAX_H];
      gat_ld_row(S, xlr + j * ld, xl);
      gat_z<VEC, NV>(S, xr, xl, smt, satt, hc, d, arow, adiv, slope, z, sv);
#pragma unroll
      for (int t = 0; t < NV; ++t)
#pragma unroll
        for (int u = 0; u < VEC; ++u) dv[t][u] = go[t][u] * xl[t][u];
      gat_head_sums<VEC, NV>(S, sv, heads, G, s);
      gat_head_sums<VEC, NV>(S, dv, heads, G, dot);
      if (ev && !loop) {
        ++cnt;
        if (sub == 0)
          for (int k = 0; k < d; ++k) sattr[k] += __ldg(arow + k);
      }
      if (ev) {
        float kf[GAT_MAX_H];
        gat_keep(seed, loop ? (int64_t)e + row : (int64_t)eid, heads, p, kf);
#pragma unroll
        for (int h = 0; h < GAT_MAX_H; ++h)
          if (h < heads) Dh[h] = fmaf(expf(s[h] - lsev[h]) * kf[h], dot[h], Dh[h]);
      }
    }
    const float mdiv = cnt > 0 ? (float)cnt : 1.f;
    __syncwarp();
    if (rv && sub == 0)
      for (int k = 0; k < d; ++k) mean_ws[(int64_t)row * d + k] = sattr[k] / mdiv;
    // walk 2: the self-loop first, then the in-edges in CSR order
    float gxr[NV][VEC];
#pragma unroll
    for (int t = 0; t < NV; ++t)
#pragma unroll
      for (int u = 0; u < VEC; ++u) gxr[t][u] = 0.f;
    for (int it = 0; it < maxlen; ++it) {
      __syncwarp();
      const bool loop = it == 0;
      const int q = lo + it - 1;
      const bool in = !loop && it <= len;
      const int j = loop ? rr : (in ? src[q] : rr);
      const int eid = in ? (perm ? perm[q] : q) : 0;
      const bool ev = rv && (loop || (in && j != row));
      const float* arow = in ? eattr + (int64_t)eid * d : sattr;
      const float adiv = loop ? mdiv : 1.f;
      float xl[NV][VEC], z[NV][VEC], sv[NV][VEC], dv[NV][VEC], s[GAT_MAX_H], dot[GAT_MAX_H], gsh[GAT_MAX_H];
      gat_ld_row(S, xlr + j * ld, xl);
      gat_z<VEC, NV>(S, xr, xl, smt, satt, hc, d, arow, adiv, slope, z, sv);
#pragma unroll
      for (int t = 0; t < NV; ++t)
#pragma unroll
        for (int u = 0; u < VEC; ++u) dv[t][u] = go[t][u] * xl[t][u];
      gat_head_sums<VEC, NV>(S, sv, heads, G, s);
      gat_head_sums<VEC, NV>(S, dv, heads, G, dot);
      float kf[GAT_MAX_H];
      gat_keep(seed, loop ? (int64_t)e + rr : (int64_t)eid, heads, p, kf);
      const int64_t slot = loop ? (int64_t)e + rr : (int64_t)eid;
#pragma unroll
      for (int h = 0; h < GAT_MAX_H; ++h) {
        const float a = expf(s[h] - lsev[h]);
        gsh[h] = ev ? a * (kf[h] * dot[h] - Dh[h]) : 0.f;
        if (ev && h < heads && sub == 0) {
          gs_ws[slot * heads + h] = gsh[h];
          ak_ws[slot * heads + h] = a * kf[h];
        }
      }
      float gz[NV][VEC];
#pragma unroll
      for (int t = 0; t < NV; ++t) {
        const float g = gat_pick(gsh, S.hs[t]);
#pragma unroll
        for (int u = 0; u < VEC; ++u) {
          const float lr = z[t][u] > 0.f ? z[t][u] : z[t][u] * slope;
          gz[t][u] = S.hs[t] < GAT_MAX_H ? g * satt[S.ch[t] + u] * (z[t][u] > 0.f ? 1.f : slope) : 0.f;
          gxr[t][u] += gz[t][u];
          if (part && ev && S.hs[t] < GAT_MAX_H) gacc[S.ch[t] + u] = fmaf(g, lr, gacc[S.ch[t] + u]);
        }
      }
      if (part && ev) {
        for (int k = 0; k < d; ++k) {
          const float a = arow[k] / adiv;
          float* gk = gacc + (k + 1) * hc;
#pragma unroll
          for (int t = 0; t < NV; ++t)
            if (S.hs[t] < GAT_MAX_H) {
#pragma unroll
              for (int u = 0; u < VEC; ++u) gk[S.ch[t] + u] = fmaf(a, gz[t][u], gk[S.ch[t] + u]);
            }
        }
      }
      if (g_eattr) {
        const float rc = 1.f / mdiv;
        for (int k = 0; k < d; ++k) {
          float v = 0.f;
#pragma unroll
          for (int t = 0; t < NV; ++t)
#pragma unroll
            for (int u = 0; u < VEC; ++u) v = fmaf(smt[k * hc + S.ch[t] + u], gz[t][u], v);
          v = gat_group_sum(v, G);
          if (loop) {
            if (sub == 0) sgl[k] = v;
          } else if (in && rv && sub == 0) {
            g_eattr[(int64_t)eid * d + k] = ev ? v + sgl[k] * rc : 0.f;
          }
        }
      }
    }
    if (rv) {
#pragma unroll
      for (int t = 0; t < NV; ++t)
        if (S.hs[t] < GAT_MAX_H) gat_st<VEC>(g_xlr + (int64_t)row * ld + hc + S.ch[t], gxr[t]);
    }
  }
  if (!part) return;
  __syncthreads();
  for (int r = threadIdx.x; r < slice; r += blockDim.x) {
    float s = 0.f;
    for (int g = 0; g < ngrp; ++g) s += sacc[g * slice + r];
    part[(int64_t)blockIdx.x * slice + r] = s;
  }
}

// ---- backward pass B, by source -------------------------------------------------------------------------------------------
// g_xl[j] = sum over the out-edges e = (j -> i) of alpha k g_h[i] + g_z, and the self-loop of j last.  alpha k and g_s come
// from pass A's workspace; z is recomputed through gat_z (the self-loop's attribute from pass A's mean).
template <int VEC, int NV>
__global__ void __launch_bounds__(256, 1) gat_bwd_b_kernel(
    const float* __restrict__ g_out, const float* __restrict__ xlr, const int32_t* __restrict__ rowptr,
    const int32_t* __restrict__ perm, const int32_t* __restrict__ dst, const float* __restrict__ eattr, int d,
    const float* __restrict__ mt, const float* __restrict__ att, int n, int e, int heads, int c, int concat, float slope,
    int gl2, const float* __restrict__ gs_ws, const float* __restrict__ ak_ws, const float* __restrict__ mean_ws,
    float* __restrict__ g_xlr) {
  extern __shared__ float gat_sm[];
  const int hc = heads * c;
  const float* smt = gat_sm;
  const float* satt = gat_sm + d * hc;
  gat_stage(gat_sm, mt, att, hc, d);
  __syncthreads();
  const int G = 1 << gl2, sub = threadIdx.x & (G - 1), gpb = blockDim.x >> gl2;
  const GatSlots<VEC, NV> S(sub, G, hc, c);
  const int64_t ld = 2 * (int64_t)hc;
  const float rh = concat ? 1.f : 1.f / (float)heads;
  for (int row = blockIdx.x * gpb + (threadIdx.x >> gl2); row < n; row += gridDim.x * gpb) {
    const int lo = rowptr[row], hi = rowptr[row + 1];
    float xl[NV][VEC], acc[NV][VEC];
    gat_ld_row(S, xlr + row * ld, xl);
#pragma unroll
    for (int t = 0; t < NV; ++t)
#pragma unroll
      for (int u = 0; u < VEC; ++u) acc[t][u] = 0.f;
    for (int q = lo; q <= hi; ++q) {
      const bool loop = q == hi;
      const int i = loop ? row : dst[q];
      if (!loop && i == row) continue;                 // an input self-loop: removed before the softmax
      const int64_t slot = loop ? (int64_t)e + row : (int64_t)(perm ? perm[q] : q);
      const float* arow = loop ? mean_ws + (int64_t)row * d : eattr + slot * d;
      float xr[NV][VEC], go[NV][VEC], z[NV][VEC], sv[NV][VEC];
      gat_ld_row(S, xlr + i * ld + hc, xr);
#pragma unroll
      for (int t = 0; t < NV; ++t) {
        if (concat) gat_ld<VEC>(g_out + (int64_t)i * hc + S.ch[t], go[t]);
        else gat_ld<VEC>(g_out + (int64_t)i * c + (S.ch[t] % c), go[t]);
      }
      gat_z<VEC, NV>(S, xr, xl, smt, satt, hc, d, arow, 1.f, slope, z, sv);
#pragma unroll
      for (int t = 0; t < NV; ++t) {
        if (S.hs[t] >= GAT_MAX_H) continue;
        const float a = __ldg(ak_ws + slot * heads + S.hs[t]) * rh, g = __ldg(gs_ws + slot * heads + S.hs[t]);
#pragma unroll
        for (int u = 0; u < VEC; ++u)
          acc[t][u] += fmaf(a, go[t][u], g * satt[S.ch[t] + u] * (z[t][u] > 0.f ? 1.f : slope));
      }
    }
#pragma unroll
    for (int t = 0; t < NV; ++t)
      if (S.hs[t] < GAT_MAX_H) gat_st<VEC>(g_xlr + (int64_t)row * ld + S.ch[t], acc[t]);
  }
}

// out[r] = sum over the CTAs in index order (fp64) of part[b, r]
__global__ void gat_reduce_kernel(const float* __restrict__ part, int nblk, int rows, float* __restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += (double)part[(int64_t)b * rows + r];
    out[r] = (float)s;
  }
}

__global__ void gat_keep_kernel(int64_t slots, int heads, float p, const int64_t* __restrict__ seed_ptr,
                                uint8_t* __restrict__ keep) {
  const uint64_t seed = (uint64_t)*seed_ptr;
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < slots; s += (int64_t)gridDim.x * blockDim.x) {
    float kf[GAT_MAX_H];
    gat_keep(seed, s, heads, p, kf);
    for (int h = 0; h < heads; ++h) keep[s * heads + h] = kf[h] != 0.f ? 1 : 0;
  }
}

namespace {
struct GatLaunch {
  int vec, nv, gl2;
};

// VEC 4 where every head's channels are whole float4s and the row pointers allow it; nv rounded up to an instantiated count
// (a lane holds at most 16 channels of each operand: above that the backward would spill)
GatLaunch gat_launch(int heads, int c, bool aligned) {
  GatLaunch L;
  const int hc = heads * c;
  L.vec = (c % 4 == 0 && aligned) ? 4 : 1;
  const int nvec = hc / L.vec;
  L.gl2 = 0;
  while ((1 << L.gl2) < nvec && L.gl2 < 5) ++L.gl2;
  const int need = (nvec + (1 << L.gl2) - 1) >> L.gl2;
  if (L.vec == 4) L.nv = need;
  else L.nv = need <= 2 ? need : (need <= 4 ? 4 : (need <= 8 ? 8 : 16));
  return L;
}

bool gat_aligned(std::initializer_list<const void*> ps) {
  for (const void* q : ps)
    if ((uintptr_t)q % 16) return false;
  return true;
}

// warps per CTA of pass A: the per-group parameter slices must fit in shared memory
int gat_bwd_warps(int hc, int d, int gl2, bool grads) {
  for (int w = 8; w > 1; w >>= 1) {
    const size_t groups = (size_t)w * (32 >> gl2);
    const size_t fl = (size_t)(d + 1) * hc + groups * 2 * GAT_MAX_D + (grads ? groups * (d + 1) * hc : 0);
    if (fl * 4 <= GAT_SMEM_LIMIT) return w;
  }
  return 1;
}
}  // namespace

#define GAT_DISPATCH(LAUNCH)                    \
  do {                                          \
    if (L.vec == 4) {                           \
      switch (L.nv) {                           \
        case 1: LAUNCH(4, 1); break;            \
        case 2: LAUNCH(4, 2); break;            \
        case 3: LAUNCH(4, 3); break;            \
        default: LAUNCH(4, 4); break;           \
      }                                         \
    } else {                                    \
      switch (L.nv) {                           \
        case 1: LAUNCH(1, 1); break;            \
        case 2: LAUNCH(1, 2); break;            \
        case 4: LAUNCH(1, 4); break;            \
        default: LAUNCH(1, 8); break;           \
      }                                         \
    }                                           \
  } while (0)

// heads c <= 512 when every head's channels are whole float4s (4 float4 slots per lane), else <= 256 (8 scalar slots)
static bool gat_shape_ok(int heads, int c, int d) {
  return heads >= 1 && heads <= GAT_MAX_H && c >= 1 && heads * c <= (c % 4 == 0 ? GAT_MAX_HC : GAT_MAX_HC / 2) && d >= 0 &&
         d <= GAT_MAX_D;
}

extern "C" int hgb_gat_supported(int32_t heads, int32_t c, int32_t d) { return gat_shape_ok(heads, c, d); }

extern "C" int64_t hgb_gat_workspace_bytes(int32_t n, int32_t e, int32_t heads, int32_t c, int32_t d) {
  if (n < 0 || e < 0 || !hgb_gat_supported(heads, c, d)) return -1;
  const int64_t hc = (int64_t)heads * c;
  return 4 * (2 * ((int64_t)e + n) * heads + (int64_t)n * d + (int64_t)GAT_BWD_MAX_BLOCKS * (d + 1) * hc);
}

#define GAT_CHECK_ARGS(name)                                                                                                   \
  HGB_REQUIRE(n >= 0 && e >= 0 && hgb_gat_supported(heads, c, d),                                                           \
              name ": bad sizes (n %d, e %d, heads %d, c %d, d %d; 1 <= heads <= %d, 1 <= c, heads c <= %d (%d when c %% 4 "  \
              "!= 0), 0 <= d <= %d)", n, e, heads, c, d, GAT_MAX_H, GAT_MAX_HC, GAT_MAX_HC / 2, GAT_MAX_D);                 \
  HGB_REQUIRE(p >= 0.f && p < 1.f, name ": dropout probability %g outside [0, 1)", (double)p);                               \
  HGB_REQUIRE(p == 0.f || seed, name ": dropout needs the seed");                                                            \
  HGB_REQUIRE(n == 0 || (xlr && rowptr && att), name ": null argument");                                                     \
  HGB_REQUIRE(e == 0 || src, name ": null argument");                                                                        \
  HGB_REQUIRE(d == 0 || (mt && (e == 0 || eattr)), name ": d > 0 needs the edge attributes and mt")

extern "C" int hgb_gat_fwd(const float* xlr, const int32_t* rowptr, const int32_t* perm, const int32_t* src, const float* eattr,
                           int32_t d, const float* mt, const float* att, const float* bias, int32_t n, int32_t e, int32_t heads,
                           int32_t c, int32_t concat, float negative_slope, float p, const int64_t* seed, float* out, float* lse,
                           hgb_stream_t stream) {
  GAT_CHECK_ARGS("gat_fwd");
  HGB_REQUIRE(n == 0 || (bias && out && lse), "gat_fwd: null argument");
  const int hc = heads * c;
  const GatLaunch L = gat_launch(heads, c, gat_aligned({xlr, out}));
  HGB_REQUIRE(L.vec == 4 || hc <= GAT_MAX_HC / 2, "gat_fwd: heads c = %d > %d needs 16-byte aligned xlr and out", hc,
              GAT_MAX_HC / 2);
  if (n == 0) return HGB_OK;
  const int gpw = 32 >> L.gl2;
  const size_t smem = 4 * ((size_t)(d + 1) * hc + (size_t)8 * gpw * (GAT_MAX_D + (concat ? 0 : hc)));
  const int grid = hgb_grid_for(n, 8 * gpw);
#define GAT_FWD(V, NV)                                                                                                         \
  do {                                                                                                                         \
    cudaFuncSetAttribute(gat_fwd_kernel<V, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                      \
    gat_fwd_kernel<V, NV><<<grid, 256, smem, (cudaStream_t)stream>>>(xlr, rowptr, perm, src, eattr, d, mt, att, bias, n, e,    \
                                                                    heads, c, concat, negative_slope, p, seed, L.gl2, out,   \
                                                                    lse);                                                    \
  } while (0)
  GAT_DISPATCH(GAT_FWD);
#undef GAT_FWD
  HGB_LAUNCH_CHECK("gat_fwd");
  return HGB_OK;
}

extern "C" int hgb_gat_dropout_keep(int32_t n, int32_t e, int32_t heads, float p, const int64_t* seed, void* keep,
                                    hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && e >= 0 && heads >= 1 && heads <= GAT_MAX_H, "gat_dropout_keep: bad sizes (n %d, e %d, heads %d)", n, e,
              heads);
  HGB_REQUIRE(p >= 0.f && p < 1.f, "gat_dropout_keep: dropout probability %g outside [0, 1)", (double)p);
  HGB_REQUIRE(seed && keep, "gat_dropout_keep: null argument");
  const int64_t slots = (int64_t)e + n;
  if (slots == 0) return HGB_OK;
  gat_keep_kernel<<<hgb_grid_for(slots, 256), 256, 0, (cudaStream_t)stream>>>(slots, heads, p, seed, static_cast<uint8_t*>(keep));
  HGB_LAUNCH_CHECK("gat_dropout_keep");
  return HGB_OK;
}

extern "C" int hgb_gat_bwd(const float* g_out, const float* xlr, const int32_t* rowptr, const int32_t* perm, const int32_t* src,
                           const int32_t* row_rowptr, const int32_t* row_perm, const int32_t* row_dst, const float* eattr,
                           int32_t d, const float* mt, const float* att, const float* lse, int32_t n, int32_t e, int32_t heads,
                           int32_t c, int32_t concat, float negative_slope, float p, const int64_t* seed, float* g_xlr,
                           float* g_eattr, float* g_params, void* workspace, hgb_stream_t stream) {
  GAT_CHECK_ARGS("gat_bwd");
  HGB_REQUIRE(n == 0 || (g_out && lse && g_xlr && row_rowptr && workspace), "gat_bwd: null argument");
  HGB_REQUIRE(e == 0 || row_dst, "gat_bwd: null argument");
  HGB_REQUIRE(!g_eattr || d > 0, "gat_bwd: g_eattr needs d > 0");
  const int hc = heads * c;
  const int rows = (d + 1) * hc;
  const GatLaunch L = gat_launch(heads, c, gat_aligned({xlr, g_out, g_xlr}));
  HGB_REQUIRE(L.vec == 4 || hc <= GAT_MAX_HC / 2, "gat_bwd: heads c = %d > %d needs 16-byte aligned xlr, g_out and g_xlr", hc,
              GAT_MAX_HC / 2);
  if (n == 0) {                              // no nodes: no edges either, every gradient is empty or zero
    if (g_params) cudaMemsetAsync(g_params, 0, sizeof(float) * (size_t)rows, (cudaStream_t)stream);
    return cudaPeekAtLastError() == cudaSuccess ? HGB_OK : HGB_ECUDA;
  }
  const bool grads = g_params != nullptr;
  float* gs_ws = static_cast<float*>(workspace);
  float* ak_ws = gs_ws + ((int64_t)e + n) * heads;
  float* mean_ws = ak_ws + ((int64_t)e + n) * heads;
  float* part = grads ? mean_ws + (int64_t)n * d : nullptr;
  const int gpw = 32 >> L.gl2;
  const int warps = gat_bwd_warps(hc, d, L.gl2, grads);
  const size_t smem_a =
      4 * ((size_t)(d + 1) * hc + (size_t)warps * gpw * 2 * GAT_MAX_D + (grads ? (size_t)warps * gpw * (d + 1) * hc : 0));
  const int grid_a = hgb_grid_for(n, warps * gpw, GAT_BWD_MAX_BLOCKS);
#define GAT_BWD_A(V, NV)                                                                                                       \
  do {                                                                                                                         \
    cudaFuncSetAttribute(gat_bwd_a_kernel<V, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_a);                  \
    gat_bwd_a_kernel<V, NV><<<grid_a, warps * 32, smem_a, (cudaStream_t)stream>>>(                                            \
        g_out, xlr, rowptr, perm, src, eattr, d, mt, att, lse, n, e, heads, c, concat, negative_slope, p, seed, L.gl2, g_xlr,  \
        g_eattr, gs_ws, ak_ws, mean_ws, part);                                                                                \
  } while (0)
  GAT_DISPATCH(GAT_BWD_A);
#undef GAT_BWD_A
  HGB_LAUNCH_CHECK("gat_bwd_a");
  const size_t smem_b = 4 * (size_t)(d + 1) * hc;
  const int grid_b = hgb_grid_for(n, 256 >> L.gl2);
#define GAT_BWD_B(V, NV)                                                                                                       \
  do {                                                                                                                         \
    cudaFuncSetAttribute(gat_bwd_b_kernel<V, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_b);                  \
    gat_bwd_b_kernel<V, NV><<<grid_b, 256, smem_b, (cudaStream_t)stream>>>(g_out, xlr, row_rowptr, row_perm, row_dst, eattr,  \
                                                                          d, mt, att, n, e, heads, c, concat, negative_slope, \
                                                                          L.gl2, gs_ws, ak_ws, mean_ws, g_xlr);               \
  } while (0)
  GAT_DISPATCH(GAT_BWD_B);
#undef GAT_BWD_B
  HGB_LAUNCH_CHECK("gat_bwd_b");
  if (grads) {
    gat_reduce_kernel<<<hgb_grid_for(rows, 256), 256, 0, (cudaStream_t)stream>>>(part, grid_a, rows, g_params);
    HGB_LAUNCH_CHECK("gat_reduce");
  }
  return HGB_OK;
}
