// libhgb.so -- MACE hot path (hydragnn/utils/model/mace_utils/modules/blocks.py:369-402 and symmetric_contraction.py):
//   * tensor-product paths fused with the segmented scatter: per receiver node, a warp walks the node's CSR segment and
//     accumulates   sum_edges  c * C[m1 m2 m3] * Y[e, m2] * w[e, path, ch] * up[sender, m1, ch]   in registers; the message
//     tensor mji [E, F (L+1)^2] of the reference (blocks.py:390-392) never exists.  No atomics: summation order = CSR order.
//   * symmetric contraction (correlation 2) per (node, channel), weights selected by the node's element.
// Features are channel-last: [N, spherical index, F].  The straight-line coupling code is generated (hgb_mace_gen.cuh).
#include "hgb_common.cuh"
#include "hgb_mace_gen.cuh"

#define MWPB 4   // warps per block


// ---- per-warp asynchronous staging of one edge's operands (path weights, sender rows, harmonics) ------------------------------
__device__ __forceinline__ void mace_cp16(void* smem, const void* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void mace_cp4(void* smem, const void* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void mace_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void mace_cp_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

template <class T, int CPL>
struct MaceStage {
  static constexpr int CH = 32 * CPL;                                   // channels handled per pass
  static constexpr int FLOATS = (T::NPATH + T::S_IN) * CH + 16;         // w rows | up rows | harmonics (padded)
  // buffer layout (floats): [0, NPATH*CH) path weights, [NPATH*CH, (NPATH+S_IN)*CH) sender rows, then S_SH harmonics
  __device__ __forceinline__ static void issue(float* buf, const float* __restrict__ up, const float* __restrict__ sh,
                                               const float* __restrict__ tpw, int64_t e, int j, int f, int c0, int sh_ld, int lane) {
    constexpr int Q = CH / 4;                                           // 16-byte pieces per row
    const float* wsrc = tpw + e * T::NPATH * f + c0;
#pragma unroll
    for (int idx = lane; idx < T::NPATH * Q; idx += 32) mace_cp16(buf + idx * 4, wsrc + (int64_t)(idx / Q) * f + (idx % Q) * 4);
    const float* usrc = up + (int64_t)j * T::S_IN * f + c0;
    float* ub = buf + T::NPATH * CH;
#pragma unroll
    for (int idx = lane; idx < T::S_IN * Q; idx += 32) mace_cp16(ub + idx * 4, usrc + (int64_t)(idx / Q) * f + (idx % Q) * 4);
    if (lane < T::S_SH) mace_cp4(buf + (T::NPATH + T::S_IN) * CH + lane, sh + e * sh_ld + lane);
  }
  __device__ __forceinline__ static void read(const float* buf, int lane, float (&y)[T::S_SH], float (&u)[T::S_IN][CPL],
                                              float (&w)[T::NPATH][CPL]) {
#pragma unroll
    for (int k = 0; k < T::NPATH; ++k)
#pragma unroll
      for (int t = 0; t < CPL; ++t) w[k][t] = buf[k * CH + lane * CPL + t];
#pragma unroll
    for (int s = 0; s < T::S_IN; ++s)
#pragma unroll
      for (int t = 0; t < CPL; ++t) u[s][t] = buf[(T::NPATH + s) * CH + lane * CPL + t];
#pragma unroll
    for (int s = 0; s < T::S_SH; ++s) y[s] = buf[(T::NPATH + T::S_IN) * CH + s];
  }
};

// Edge-attribute variant (MACEStack.py:198-203, blocks.py:314-326): the edge irreps are (D+1)x0e + 1x1o + ..., so each of the
// P0 = LIN + 1 paths whose edge irrep is the 0e entry has a [F, D+1] weight block (u-major, v fastest) in the reference's
// tpw row; every other path keeps its F weights.  The effective per-channel weight of a 0e path is
//   w[u] = (1 / sqrt(D+1)) * sum_v tpw[e, k, u, v] * a[e, v],   a = [edge_attr, 1]
// (the 1/sqrt(D+1) is the fan-in part of that path's constant sqrt((2 l3 + 1) / (D+1)); T keeps sqrt(2 l3 + 1)).  It is mixed
// here while the staged row is read into registers, so no mixed [E, P F] copy of tpw exists.
// Path order is that of e3.tp_paths: generation order (l1 outer, l2 inner) stably sorted by l3.
__host__ __device__ constexpr int mace_path_l2(int lin, int lsh, int k) {
  int idx = 0;
  for (int l3 = 0; l3 <= lsh; ++l3)
    for (int l1 = 0; l1 <= lin; ++l1)
      for (int l2 = 0; l2 <= lsh; ++l2)
        if (l3 >= (l1 > l2 ? l1 - l2 : l2 - l1) && l3 <= l1 + l2 && (l1 + l2 + l3) % 2 == 0) {
          if (idx == k) return l2;
          ++idx;
        }
  return -1;
}

// Largest edge_dim of the fused kernels: the worst stage, (LIN, LSH) = (2, 2) at 64 channels per pass, takes
// 4 warps x 2 buffers x ((11 + 3 D + 9) x 64 + 32) floats = 140 KB of shared memory at D = 16, under the 227 KB opt-in limit.
#define MACE_TP_MAX_D 16

template <int LIN, int LSH, int CPL>
struct MaceStageEdge {
  using T = MaceTP<LIN, LSH>;
  static constexpr int CH = 32 * CPL;
  static constexpr int P0 = LIN + 1;
  __host__ __device__ static constexpr bool is0e(int k) { return mace_path_l2(LIN, LSH, k) == 0; }
  __host__ __device__ static constexpr int n0_before(int k) {
    int c = 0;
    for (int q = 0; q < k; ++q) c += is0e(q) ? 1 : 0;
    return c;
  }
  // buffer layout (floats): path k's weights at (k + d n0_before(k)) CH, (1 + d is0e(k)) CH of them; then S_IN sender rows,
  // 16 harmonics (padded), 16 edge attributes (d <= MACE_TP_MAX_D)
  __host__ __device__ static constexpr int floats(int d) { return (T::NPATH + d * P0 + T::S_IN) * CH + 32; }
  __device__ __forceinline__ static void issue(float* buf, const float* __restrict__ up, const float* __restrict__ sh,
                                               const float* __restrict__ tpw, const float* __restrict__ eattr, int64_t e, int j,
                                               int f, int c0, int sh_ld, int d, int lane) {
    constexpr int Q = CH / 4;
    const float* wrow = tpw + e * (int64_t)(T::NPATH + d * P0) * f;
#pragma unroll
    for (int k = 0; k < T::NPATH; ++k) {
      const int wid = is0e(k) ? d + 1 : 1;
      const float* src = wrow + (int64_t)(k + d * n0_before(k)) * f + c0 * wid;
      float* dst = buf + (k + d * n0_before(k)) * CH;
      for (int idx = lane; idx < Q * wid; idx += 32) mace_cp16(dst + idx * 4, src + idx * 4);
    }
    const float* usrc = up + (int64_t)j * T::S_IN * f + c0;
    float* ub = buf + (T::NPATH + d * P0) * CH;
#pragma unroll
    for (int idx = lane; idx < T::S_IN * Q; idx += 32) mace_cp16(ub + idx * 4, usrc + (int64_t)(idx / Q) * f + (idx % Q) * 4);
    float* hb = ub + T::S_IN * CH;
    if (lane < T::S_SH) mace_cp4(hb + lane, sh + e * sh_ld + lane);
    if (lane < d) mace_cp4(hb + 16 + lane, eattr + e * d + lane);
  }
  __device__ __forceinline__ static void read(const float* buf, int lane, int d, float cmix, float (&y)[T::S_SH],
                                              float (&u)[T::S_IN][CPL], float (&w)[T::NPATH][CPL]) {
    const float* ub = buf + (T::NPATH + d * P0) * CH;
    const float* ab = ub + T::S_IN * CH + 16;
#pragma unroll
    for (int k = 0; k < T::NPATH; ++k) {
      const float* wb = buf + (k + d * n0_before(k)) * CH;
#pragma unroll
      for (int t = 0; t < CPL; ++t) {
        if (is0e(k)) {
          const float* q = wb + (lane * CPL + t) * (d + 1);
          float s = q[d];
          for (int v = 0; v < d; ++v) s = fmaf(q[v], ab[v], s);
          w[k][t] = s * cmix;
        } else {
          w[k][t] = wb[lane * CPL + t];
        }
      }
    }
#pragma unroll
    for (int s = 0; s < T::S_IN; ++s)
#pragma unroll
      for (int t = 0; t < CPL; ++t) u[s][t] = ub[s * CH + lane * CPL + t];
#pragma unroll
    for (int s = 0; s < T::S_SH; ++s) y[s] = ub[T::S_IN * CH + s];
  }
};

// float offset of accumulator row r of node i inside the packed output (segments per output degree)
template <class T>
__device__ __forceinline__ int64_t mace_row_offset(int r, int i, int n, int f) {
  int l3 = 0;
#pragma unroll
  for (int l = 1; l <= T::LOUT; ++l)
    if (r >= T::acc_base(l)) l3 = l;
  const int rows = T::n_paths(l3) * (2 * l3 + 1);
  return (int64_t)n * f * T::acc_base(l3) + ((int64_t)i * rows + (r - T::acc_base(l3))) * f;
}

// EDGE: tpw rows carry the [F, D+1] blocks of the 0e paths (MaceStageEdge); eattr [E, d], cmix = 1 / sqrt(d + 1)
template <int LIN, int LSH, int CPL, bool EDGE>
__global__ void __launch_bounds__(MWPB * 32)
mace_tp_scatter_fwd_kernel(const float* __restrict__ up, const float* __restrict__ sh, const float* __restrict__ tpw,
                           const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm, const int32_t* __restrict__ snd, int n,
                           int f, int sh_ld, float* __restrict__ out, const float* __restrict__ eattr, int d, float cmix) {
  using T = MaceTP<LIN, LSH>;
  using ST = MaceStage<T, CPL>;
  using SE = MaceStageEdge<LIN, LSH, CPL>;
  extern __shared__ __align__(16) float mace_smem[];
  const int stage = EDGE ? SE::floats(d) : ST::FLOATS;
  float* sbuf = mace_smem + (threadIdx.x >> 5) * 2 * stage;            // this warp's two edge buffers
  const int lane = threadIdx.x & 31;
  const int ncb = f / (32 * CPL);
  for (int i = blockIdx.x * MWPB + (threadIdx.x >> 5); i < n; i += gridDim.x * MWPB) {
    const int lo = rowptr[i], hi = rowptr[i + 1];
    for (int cb = 0; cb < ncb; ++cb) {
      const int c = (cb * 32 + lane) * CPL;
      float acc[T::NACC][CPL];
#pragma unroll
      for (int r = 0; r < T::NACC; ++r)
#pragma unroll
        for (int t = 0; t < CPL; ++t) acc[r][t] = 0.f;
      if (lo < hi) {
        if constexpr (EDGE) SE::issue(sbuf, up, sh, tpw, eattr, perm[lo], snd[lo], f, cb * ST::CH, sh_ld, d, lane);
        else ST::issue(sbuf, up, sh, tpw, perm[lo], snd[lo], f, cb * ST::CH, sh_ld, lane);
      }
      mace_cp_commit();
      int cur = 0;
      for (int p = lo; p < hi; ++p) {
        mace_cp_wait();
        __syncwarp();
        if (p + 1 < hi) {
          if constexpr (EDGE) SE::issue(sbuf + (cur ^ 1) * stage, up, sh, tpw, eattr, perm[p + 1], snd[p + 1], f, cb * ST::CH, sh_ld, d, lane);
          else ST::issue(sbuf + (cur ^ 1) * stage, up, sh, tpw, perm[p + 1], snd[p + 1], f, cb * ST::CH, sh_ld, lane);
        }
        mace_cp_commit();
        float y[T::S_SH], u[T::S_IN][CPL], w[T::NPATH][CPL];
        if constexpr (EDGE) SE::read(sbuf + cur * stage, lane, d, cmix, y, u, w);
        else ST::read(sbuf + cur * stage, lane, y, u, w);
        T::template fwd<CPL>(y, u, w, acc);
        cur ^= 1;
      }
      __syncwarp();
#pragma unroll
      for (int r = 0; r < T::NACC; ++r)
#pragma unroll
        for (int t = 0; t < CPL; ++t) out[mace_row_offset<T>(r, i, n, f) + c + t] = acc[r][t];
    }
  }
}

// backward, edge-major in the same CSR order: per edge the gradient of the path weights, of the sender features (one
// row per edge; the caller reduces them per sender with the segmented sum) and optionally of the harmonics.
// EDGE: g_tpw in the same layout as tpw; a 0e path's block gets g_tpw[e, k, u, v] = cmix * gw[k][u] * a[e, v]
template <int LIN, int LSH, int CPL, bool NEED_Y, bool EDGE>
__global__ void __launch_bounds__(MWPB * 32)
mace_tp_scatter_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ up, const float* __restrict__ sh,
                           const float* __restrict__ tpw, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ perm,
                           const int32_t* __restrict__ snd, int n, int f, int sh_ld, float* __restrict__ g_tpw,
                           float* __restrict__ g_up_edge, float* __restrict__ g_sh, int multi_cb, const float* __restrict__ eattr, int d,
                           float cmix) {
  using T = MaceTP<LIN, LSH>;
  using ST = MaceStage<T, CPL>;
  using SE = MaceStageEdge<LIN, LSH, CPL>;
  extern __shared__ __align__(16) float mace_smem[];
  const int stage = EDGE ? SE::floats(d) : ST::FLOATS;
  float* sbuf = mace_smem + (threadIdx.x >> 5) * 2 * stage;
  const int lane = threadIdx.x & 31;
  const int ncb = f / (32 * CPL);
  for (int i = blockIdx.x * MWPB + (threadIdx.x >> 5); i < n; i += gridDim.x * MWPB) {
    const int lo = rowptr[i], hi = rowptr[i + 1];
    if (lo == hi) continue;
    for (int cb = 0; cb < ncb; ++cb) {
      const int c = (cb * 32 + lane) * CPL;
      float g[T::NACC][CPL];
#pragma unroll
      for (int r = 0; r < T::NACC; ++r)
#pragma unroll
        for (int t = 0; t < CPL; ++t) g[r][t] = __ldg(gout + mace_row_offset<T>(r, i, n, f) + c + t);
      if constexpr (EDGE) SE::issue(sbuf, up, sh, tpw, eattr, perm[lo], snd[lo], f, cb * ST::CH, sh_ld, d, lane);
      else ST::issue(sbuf, up, sh, tpw, perm[lo], snd[lo], f, cb * ST::CH, sh_ld, lane);
      mace_cp_commit();
      int cur = 0;
      for (int p = lo; p < hi; ++p) {
        const int e = perm[p];
        mace_cp_wait();
        __syncwarp();
        if (p + 1 < hi) {
          if constexpr (EDGE) SE::issue(sbuf + (cur ^ 1) * stage, up, sh, tpw, eattr, perm[p + 1], snd[p + 1], f, cb * ST::CH, sh_ld, d, lane);
          else ST::issue(sbuf + (cur ^ 1) * stage, up, sh, tpw, perm[p + 1], snd[p + 1], f, cb * ST::CH, sh_ld, lane);
        }
        mace_cp_commit();
        float y[T::S_SH], u[T::S_IN][CPL], w[T::NPATH][CPL], gw[T::NPATH][CPL], gy[T::S_SH], gu[T::S_IN][CPL];
        if constexpr (EDGE) SE::read(sbuf + cur * stage, lane, d, cmix, y, u, w);
        else ST::read(sbuf + cur * stage, lane, y, u, w);
        cur ^= 1;
#pragma unroll
        for (int s = 0; s < T::S_SH; ++s) gy[s] = 0.f;
#pragma unroll
        for (int s = 0; s < T::S_IN; ++s)
#pragma unroll
          for (int t = 0; t < CPL; ++t) gu[s][t] = 0.f;
        T::template bwd_edge<CPL, NEED_Y>(y, u, w, g, gw, gy);
        T::template bwd_up<CPL>(y, w, g, gu);
        if constexpr (EDGE) {
          const float* ab = sbuf + (cur ^ 1) * stage + (T::NPATH + d * SE::P0 + T::S_IN) * ST::CH + 16;
          float* grow = g_tpw + (int64_t)e * (T::NPATH + d * SE::P0) * f;
#pragma unroll
          for (int k = 0; k < T::NPATH; ++k) {
            float* gk = grow + (int64_t)(k + d * SE::n0_before(k)) * f;
#pragma unroll
            for (int t = 0; t < CPL; ++t) {
              if (SE::is0e(k)) {
                const float gm = cmix * gw[k][t];
                float* q = gk + (int64_t)(c + t) * (d + 1);
                for (int v = 0; v < d; ++v) q[v] = gm * ab[v];
                q[d] = gm;
              } else {
                gk[c + t] = gw[k][t];
              }
            }
          }
        } else {
#pragma unroll
          for (int k = 0; k < T::NPATH; ++k)
#pragma unroll
            for (int t = 0; t < CPL; ++t) g_tpw[((int64_t)e * T::NPATH + k) * f + c + t] = gw[k][t];
        }
#pragma unroll
        for (int s = 0; s < T::S_IN; ++s)
#pragma unroll
          for (int t = 0; t < CPL; ++t) g_up_edge[((int64_t)e * T::S_IN + s) * f + c + t] = gu[s][t];
        if (NEED_Y) {
#pragma unroll
          for (int s = 0; s < T::S_SH; ++s) {
            const float v = hgb_warp_sum(gy[s]);
            if (lane == 0) {
              if (multi_cb) atomicAdd(g_sh + (int64_t)e * sh_ld + s, v);
              else g_sh[(int64_t)e * sh_ld + s] = v;
            }
          }
        }
      }
      __syncwarp();
    }
  }
}

static bool mace_tp_supported(int lin, int lsh) { return lin >= 0 && lin <= 2 && lsh >= 1 && lsh <= 3 && lin <= lsh; }

#define MACE_TP_DISPATCH(LIN_, LSH_, ...)                                    \
  do {                                                                        \
    const int key__ = (LIN_) * 4 + (LSH_);                                    \
    switch (key__) {                                                          \
      case 0 * 4 + 1: { constexpr int LIN = 0, LSH = 1; __VA_ARGS__; } break;        \
      case 0 * 4 + 2: { constexpr int LIN = 0, LSH = 2; __VA_ARGS__; } break;        \
      case 0 * 4 + 3: { constexpr int LIN = 0, LSH = 3; __VA_ARGS__; } break;        \
      case 1 * 4 + 1: { constexpr int LIN = 1, LSH = 1; __VA_ARGS__; } break;        \
      case 1 * 4 + 2: { constexpr int LIN = 1, LSH = 2; __VA_ARGS__; } break;        \
      case 1 * 4 + 3: { constexpr int LIN = 1, LSH = 3; __VA_ARGS__; } break;        \
      case 2 * 4 + 2: { constexpr int LIN = 2, LSH = 2; __VA_ARGS__; } break;        \
      case 2 * 4 + 3: { constexpr int LIN = 2, LSH = 3; __VA_ARGS__; } break;        \
      default: break;                                                         \
    }                                                                         \
  } while (0)

extern "C" int hgb_mace_tp_num_acc(int32_t lin, int32_t lsh) {
  int out = -1;
  if (mace_tp_supported(lin, lsh)) MACE_TP_DISPATCH(lin, lsh, out = MaceTP<LIN, LSH>::NACC);
  return out;
}

// the edge variants' stage passes the 48 KB dynamic shared-memory default for larger d (up to 140 KB, see MACE_TP_MAX_D)
template <class K>
static void mace_smem_optin(K kernel, int bytes) {
  if (bytes > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

extern "C" int hgb_mace_tp_scatter_fwd(const float* up, const float* sh, const float* tpw, const int32_t* rowptr, const int32_t* perm,
                                       const int32_t* snd, int32_t n, int32_t f, int32_t lin, int32_t lsh, int32_t sh_ld,
                                       const float* eattr, int32_t d, float* out, hgb_stream_t stream) {
  HGB_REQUIRE(mace_tp_supported(lin, lsh), "mace_tp_scatter: unsupported degrees lmax_in=%d lmax_sh=%d", lin, lsh);
  HGB_REQUIRE(n >= 0 && f > 0 && f % 32 == 0 && sh_ld >= (lsh + 1) * (lsh + 1), "mace_tp_scatter: need channels %% 32 == 0 (got %d)", f);
  HGB_REQUIRE(up && sh && tpw && rowptr && perm && snd && out, "mace_tp_scatter_fwd: null pointer");
  HGB_REQUIRE(d >= 0 && d <= MACE_TP_MAX_D && (d == 0 || eattr), "mace_tp_scatter_fwd: edge_dim %d (max %d) or null edge_attr", d,
              MACE_TP_MAX_D);
  if (n == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = hgb_grid_for(n, MWPB, HGB_NUM_SMS * 16);
  const float cmix = (float)(1.0 / sqrt((double)d + 1.0));
  MACE_TP_DISPATCH(lin, lsh, {
    const bool two = f % 64 == 0 && MaceTP<LIN, LSH>::NACC <= 40;
    if (d > 0) {
      if (two) {
        const int bytes = MWPB * 2 * MaceStageEdge<LIN, LSH, 2>::floats(d) * 4;
        mace_smem_optin(mace_tp_scatter_fwd_kernel<LIN, LSH, 2, true>, bytes);
        mace_tp_scatter_fwd_kernel<LIN, LSH, 2, true><<<grid, MWPB * 32, bytes, st>>>(up, sh, tpw, rowptr, perm, snd, n, f, sh_ld, out, eattr, d, cmix);
      } else {
        const int bytes = MWPB * 2 * MaceStageEdge<LIN, LSH, 1>::floats(d) * 4;
        mace_smem_optin(mace_tp_scatter_fwd_kernel<LIN, LSH, 1, true>, bytes);
        mace_tp_scatter_fwd_kernel<LIN, LSH, 1, true><<<grid, MWPB * 32, bytes, st>>>(up, sh, tpw, rowptr, perm, snd, n, f, sh_ld, out, eattr, d, cmix);
      }
    } else if (two)
      mace_tp_scatter_fwd_kernel<LIN, LSH, 2, false><<<grid, MWPB * 32, MWPB * 2 * MaceStage<MaceTP<LIN, LSH>, 2>::FLOATS * 4, st>>>(up, sh, tpw, rowptr, perm, snd, n, f, sh_ld, out, nullptr, 0, 1.f);
    else
      mace_tp_scatter_fwd_kernel<LIN, LSH, 1, false><<<grid, MWPB * 32, MWPB * 2 * MaceStage<MaceTP<LIN, LSH>, 1>::FLOATS * 4, st>>>(up, sh, tpw, rowptr, perm, snd, n, f, sh_ld, out, nullptr, 0, 1.f);
  });
  HGB_LAUNCH_CHECK("mace_tp_scatter_fwd");
  return HGB_OK;
}

extern "C" int hgb_mace_tp_scatter_bwd(const float* g_out, const float* up, const float* sh, const float* tpw, const int32_t* rowptr,
                                       const int32_t* perm, const int32_t* snd, int32_t n, int32_t f, int32_t lin, int32_t lsh,
                                       int32_t sh_ld, const float* eattr, int32_t d, float* g_tpw, float* g_up_edge, float* g_sh,
                                       hgb_stream_t stream) {
  HGB_REQUIRE(mace_tp_supported(lin, lsh), "mace_tp_scatter: unsupported degrees lmax_in=%d lmax_sh=%d", lin, lsh);
  HGB_REQUIRE(n >= 0 && f > 0 && f % 32 == 0 && sh_ld >= (lsh + 1) * (lsh + 1), "mace_tp_scatter: need channels %% 32 == 0 (got %d)", f);
  HGB_REQUIRE(g_out && up && sh && tpw && rowptr && perm && snd && g_tpw && g_up_edge, "mace_tp_scatter_bwd: null pointer");
  HGB_REQUIRE(d >= 0 && d <= MACE_TP_MAX_D && (d == 0 || eattr), "mace_tp_scatter_bwd: edge_dim %d (max %d) or null edge_attr", d,
              MACE_TP_MAX_D);
  if (n == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = hgb_grid_for(n, MWPB, HGB_NUM_SMS * 16);
  const float cmix = (float)(1.0 / sqrt((double)d + 1.0));
#define LAUNCH_B(C, Y) mace_tp_scatter_bwd_kernel<LIN, LSH, C, Y, false><<<grid, MWPB * 32, MWPB * 2 * MaceStage<MaceTP<LIN, LSH>, C>::FLOATS * 4, st>>>(g_out, up, sh, tpw, rowptr, perm, snd, n, f, sh_ld, g_tpw, g_up_edge, g_sh, ncb > 1, nullptr, 0, 1.f)
#define LAUNCH_BE(C, Y)                                                                                                                      \
  do {                                                                                                                                       \
    const int bytes = MWPB * 2 * MaceStageEdge<LIN, LSH, C>::floats(d) * 4;                                                                  \
    mace_smem_optin(mace_tp_scatter_bwd_kernel<LIN, LSH, C, Y, true>, bytes);                                                               \
    mace_tp_scatter_bwd_kernel<LIN, LSH, C, Y, true><<<grid, MWPB * 32, bytes, st>>>(g_out, up, sh, tpw, rowptr, perm, snd, n, f, sh_ld,   \
                                                                                     g_tpw, g_up_edge, g_sh, ncb > 1, eattr, d, cmix);      \
  } while (0)
  MACE_TP_DISPATCH(lin, lsh, {
    const bool two = f % 64 == 0 && MaceTP<LIN, LSH>::NACC <= 24;
    const int ncb = f / (32 * (two ? 2 : 1));
    if (d > 0) {
      if (two) { if (g_sh) LAUNCH_BE(2, true); else LAUNCH_BE(2, false); }
      else { if (g_sh) LAUNCH_BE(1, true); else LAUNCH_BE(1, false); }
    } else if (two) { if (g_sh) LAUNCH_B(2, true); else LAUNCH_B(2, false); }
    else { if (g_sh) LAUNCH_B(1, true); else LAUNCH_B(1, false); }
  });
#undef LAUNCH_B
#undef LAUNCH_BE
  HGB_LAUNCH_CHECK("mace_tp_scatter_bwd");
  return HGB_OK;
}

// ---- symmetric contraction, correlation 2 ----------------------------------------------------------------------------
template <int LIN, int LOUT>
__global__ void mace_symcontract_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wall, const int32_t* __restrict__ z,
                                            int64_t total, int f, float* __restrict__ out) {
  using T = MaceSC<LIN, LOUT>;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / f;
    const int c = (int)(idx - i * f);
    float xv[T::S], wt[T::KTOT], o[T::NOUT];
#pragma unroll
    for (int s = 0; s < T::S; ++s) xv[s] = __ldg(x + (i * T::S + s) * f + c);
    const int64_t zi = z[i];
#pragma unroll
    for (int k = 0; k < T::KTOT; ++k) wt[k] = __ldg(wall + (zi * T::KTOT + k) * f + c);
    T::fwd(xv, wt, o);
#pragma unroll
    for (int m = 0; m < T::NOUT; ++m) out[(i * T::NOUT + m) * f + c] = o[m];
  }
}

template <int LIN, int LOUT>
__global__ void mace_symcontract_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ x, const float* __restrict__ wall,
                                            const int32_t* __restrict__ z, int64_t total, int f, float* __restrict__ gx,
                                            float* __restrict__ gw_node) {
  using T = MaceSC<LIN, LOUT>;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / f;
    const int c = (int)(idx - i * f);
    float xv[T::S], wt[T::KTOT], go[T::NOUT], gxv[T::S], gwt[T::KTOT];
#pragma unroll
    for (int s = 0; s < T::S; ++s) xv[s] = __ldg(x + (i * T::S + s) * f + c);
    const int64_t zi = z[i];
#pragma unroll
    for (int k = 0; k < T::KTOT; ++k) wt[k] = __ldg(wall + (zi * T::KTOT + k) * f + c);
#pragma unroll
    for (int m = 0; m < T::NOUT; ++m) go[m] = __ldg(gout + (i * T::NOUT + m) * f + c);
    T::bwd(xv, wt, go, gxv, gwt);
#pragma unroll
    for (int s = 0; s < T::S; ++s) gx[(i * T::S + s) * f + c] = gxv[s];
#pragma unroll
    for (int k = 0; k < T::KTOT; ++k) gw_node[(i * T::KTOT + k) * f + c] = gwt[k];
  }
}

static bool mace_sc_supported(int lin, int lout) { return lin >= 1 && lin <= 3 && lout >= 0 && lout <= 2 && lout <= lin; }

#define MACE_SC_DISPATCH(LIN_, LOUT_, ...)                                    \
  do {                                                                         \
    switch ((LIN_) * 4 + (LOUT_)) {                                            \
      case 1 * 4 + 0: { constexpr int LIN = 1, LOUT = 0; __VA_ARGS__; } break;        \
      case 1 * 4 + 1: { constexpr int LIN = 1, LOUT = 1; __VA_ARGS__; } break;        \
      case 2 * 4 + 0: { constexpr int LIN = 2, LOUT = 0; __VA_ARGS__; } break;        \
      case 2 * 4 + 1: { constexpr int LIN = 2, LOUT = 1; __VA_ARGS__; } break;        \
      case 2 * 4 + 2: { constexpr int LIN = 2, LOUT = 2; __VA_ARGS__; } break;        \
      case 3 * 4 + 0: { constexpr int LIN = 3, LOUT = 0; __VA_ARGS__; } break;        \
      case 3 * 4 + 1: { constexpr int LIN = 3, LOUT = 1; __VA_ARGS__; } break;        \
      case 3 * 4 + 2: { constexpr int LIN = 3, LOUT = 2; __VA_ARGS__; } break;        \
      default: break;                                                          \
    }                                                                          \
  } while (0)

extern "C" int hgb_mace_symcontract_num_weights(int32_t lin, int32_t lout) {
  int out = -1;
  if (mace_sc_supported(lin, lout)) MACE_SC_DISPATCH(lin, lout, out = MaceSC<LIN, LOUT>::KTOT);
  return out;
}

extern "C" int hgb_mace_symcontract_fwd(const float* x, const float* wall, const int32_t* z, int32_t n, int32_t f, int32_t lin,
                                        int32_t lout, float* out, hgb_stream_t stream) {
  HGB_REQUIRE(mace_sc_supported(lin, lout), "mace_symcontract: unsupported degrees lmax_in=%d lmax_out=%d", lin, lout);
  HGB_REQUIRE(n >= 0 && f > 0 && x && wall && z && out, "mace_symcontract_fwd: bad arguments");
  if (n == 0) return HGB_OK;
  const int64_t total = (int64_t)n * f;
  MACE_SC_DISPATCH(lin, lout, (mace_symcontract_fwd_kernel<LIN, LOUT><<<hgb_grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>(x, wall, z, total, f, out)));
  HGB_LAUNCH_CHECK("mace_symcontract_fwd");
  return HGB_OK;
}

extern "C" int hgb_mace_symcontract_bwd(const float* g_out, const float* x, const float* wall, const int32_t* z, int32_t n, int32_t f,
                                        int32_t lin, int32_t lout, float* gx, float* gw_node, hgb_stream_t stream) {
  HGB_REQUIRE(mace_sc_supported(lin, lout), "mace_symcontract: unsupported degrees lmax_in=%d lmax_out=%d", lin, lout);
  HGB_REQUIRE(n >= 0 && f > 0 && g_out && x && wall && z && gx && gw_node, "mace_symcontract_bwd: bad arguments");
  if (n == 0) return HGB_OK;
  const int64_t total = (int64_t)n * f;
  MACE_SC_DISPATCH(lin, lout, (mace_symcontract_bwd_kernel<LIN, LOUT><<<hgb_grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>(g_out, x, wall, z, total, f, gx, gw_node)));
  HGB_LAUNCH_CHECK("mace_symcontract_bwd");
  return HGB_OK;
}
