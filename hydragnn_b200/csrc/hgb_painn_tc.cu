// libhgb.so -- the PaiNN update block (PAINNStack.py:298-328) at F = 64 on the tensor cores (TF32 mode), without the [3n, 2F]
// U/V product in HBM.  sm_90a only.
//
// The block reads uv = update_U(v) and vv = update_V(v) only through per-node reductions over the three spatial rows (|vv|,
// sum_d uv.vv) and through per-row products.  So every kernel here recomputes [uv | vv] for its tile from v instead of reading it
// back: v [n, 3, 64] is loaded through a 3-D tensor map (dims {64, 3, n}, box {32, 1, 64}, 128-byte swizzle), a 64-node tile
// arrives as three 64 x 64 A operands, one per spatial component d, and row r is node r in all three.  The wgmma accumulator layout
// is the same for the three d-GEMMs, so uv_d[r, c] and vv_d[r, c] of every d land in the same thread (uv at fragment index j, vv at
// j + 32): the reductions over d are register arithmetic.  At K = 64 the recomputation costs the tensor cores far less than the
// 24 bytes per element that storing and re-reading [uv | vv] cost HBM.
//
// Each product is the one the unfused path (PainnUpdateFn) runs on tc_linear_kernel -- m64n128k8 over K = 64 in kb-major order,
// accumulators from zero, the bias added afterwards; the dgrad m64n64k8 over K = 128, a zero bias, then the addend -- and each
// elementwise formula is written as in the painn_update_* kernels (hgb_painn.cu), so the results are the same bits.
//
// One kernel template, four steps of the block (ld: row strides; na = 2 (last) or 3):
//   UPD_FWD   mlp_in [n, 128] = [|vv|, s] (and inner [n, 64] for a last layer)
//   UPD_POST  (not last) s_out = s + a_sv * inner + a_ss;  v_out_d = v_d + a_vv * uv_d (v_d is read from the A stage itself)
//   UPD_BWD_A (not last) ga [n, 192] = [sum_d gv_out_d uv_d, gs_out * inner, gs_out]
//   (a last layer's s_out and ga need inner only: two elementwise kernels read the stored one)
//   UPD_BWD   gs = gs_out + g_mlp_in[:, 64:];  [guv_d | gvv_d] as painn_update_bwd forms them -> g_uv [3n, 128] (the U/V weight
//             gradient's operand) and, staged in shared memory as the A operand of the dgrad against [U; V]^T (K = 128) in the same
//             CTA, gv_d = [guv_d | gvv_d] [U; V] (+ gv_out_d)
// Persistent and warp-specialised like tc_linear_kernel: warp 4 issues the TMA loads of every (tile, d) item into a ring of stages
// ahead of the consumer warpgroup (warps 0-3), so the loads of the next items overlap the current one's math.  One consumer per CTA
// keeps the whole register file of a thread available to it (the BWD step holds 64 accumulators and 128 per-node values); where
// shared memory allows, two CTAs share an SM and overlap each other's epilogues.
#include "hgb_tc.cuh"

namespace {

enum { UPD_FWD, UPD_POST, UPD_BWD_A, UPD_BWD };

constexpr int UF = 64;                               // feature width
constexpr int UPD_TILE = 64;                         // nodes per tile = one wgmma M
constexpr uint32_t UPD_STAGE = UPD_TILE * UF * 4;    // one (tile, d) item: two [64 x 32] boxes, 16 KB
constexpr uint32_t UPD_B = 2 * UF * UF * 4;          // [U; V] K-major [128 x 64], 32 KB; its transpose [64 x 128] likewise
constexpr uint32_t UPD_G = UPD_TILE * 2 * UF * 4;    // one [guv | gvv] tile, K-major [64 x 128], 32 KB
constexpr int UPD_THREADS = 160;
constexpr int upd_stages(int mode) { return mode == UPD_BWD ? 5 : 4; }   // A stages in the ring: more than one tile's three items

struct UpdParams {
  int n;
  const float* wuv;       // [128, 64] = [U; V]
  const float* buv;       // [128]
  const float* s;         // FWD, POST
  const float* a;         // POST, BWD: update_mlp output [n, 64 na]
  const float* gs_out;    // BWD_A, BWD
  const float* gv_out;    // BWD_A, BWD (not last) [n, 3, 64]
  const float* g_mlp_in;  // BWD [n, 128]
  const float* mlp_in;    // BWD: |vv| in columns 0..63
  float* mlp_in_out;      // FWD
  float* inner_out;       // FWD (optional): inner = sum_d uv_d vv_d, for the elementwise post / ga of a last layer
  float* s_out;           // POST
  float* v_out;           // POST (not last)
  float* ga;              // BWD_A
  float* g_uv;            // BWD [3n, 128]
  float* gs;              // BWD
  float* gv;              // BWD [n, 3, 64]
};

// Shared memory (bytes): 1 KB alignment + [U; V] 32 KB (+ its transpose 32 KB, BWD) + stages x 16 KB + (BWD) 32 KB [guv | gvv] staging
// + 2 x stages barriers + 512 B bias.  BWD: 1,024 + 65,536 + 81,920 + 32,768 + 80 + 512 = 181,840 (one CTA per SM); the other modes:
// 1,024 + 32,768 + 65,536 + 64 + 512 = 99,904, two CTAs per SM where the registers allow it (<= 204 per thread).  Registers (ptxas,
// no spills): the d-GEMM accumulators are 64 per thread; BWD keeps g a_sv, gn / |vv|, a_vv and gv_out_d (32 each) beside them
// (255 registers, 222 when last); POST and BWD_A (not last) keep inner and a_vv or sum_d gv_out_d uv_d (233 / 214); FWD keeps inner,
// vv_0 and vv_1 (204: one CTA per SM; a bound of two spills).  The d loop is not unrolled: unrolled, ptxas spills.
constexpr size_t upd_smem(int mode) {
  return 1024 + (mode == UPD_BWD ? 2 : 1) * (size_t)UPD_B + upd_stages(mode) * (size_t)UPD_STAGE + (mode == UPD_BWD ? (size_t)UPD_G : 0) +
         2 * upd_stages(mode) * 8 + 2 * UF * 4;
}

// The 32 values of a [64 x 64] tile that this thread's accumulator fragment covers: x[4i + 2h + e] = X(row + 8h, 8i + 2(lane % 4) + e),
// p already offset by the column 2 (lane % 4); ld = stride between consecutive nodes.  Nodes >= n read as 0 and are not written.
__device__ __forceinline__ void frag_ld(float* x, const float* p, int64_t ld, int node, int n) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool in = node + 8 * h < n;
    const float* r = p + (int64_t)(node + 8 * h) * ld;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 t = in ? __ldg(reinterpret_cast<const float2*>(r + 8 * i)) : make_float2(0.f, 0.f);
      x[4 * i + 2 * h] = t.x;
      x[4 * i + 2 * h + 1] = t.y;
    }
  }
}
__device__ __forceinline__ void frag_st(float* p, int64_t ld, int node, int n, const float* x) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (node + 8 * h < n) {
      float* r = p + (int64_t)(node + 8 * h) * ld;
#pragma unroll
      for (int i = 0; i < 8; ++i) *reinterpret_cast<float2*>(r + 8 * i) = make_float2(x[4 * i + 2 * h], x[4 * i + 2 * h + 1]);
    }
}

// L2 prefetch of rows [row0, row0 + rows) of a row-major fp32 matrix with row stride ld, columns [col0, col0 + cols): one bulk
// request when the rows are whole, else one per row (the columns a kernel does not read are not fetched)
__device__ __forceinline__ void prefetch_rows_l2(const float* base, int64_t ld, int row0, int rows, int col0, int cols) {
  if (cols == ld) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + (int64_t)row0 * ld), "r"((uint32_t)(rows * ld * 4)) : "memory");
    return;
  }
  for (int r = 0; r < rows; ++r)
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + (int64_t)(row0 + r) * ld + col0), "r"((uint32_t)(cols * 4))
                 : "memory");
}

}  // namespace

// (outside the anonymous namespace so that profiles name it)
template <int MODE, bool LAST>
__global__ void __launch_bounds__(UPD_THREADS, 1) painn_update_tc_kernel(const __grid_constant__ CUtensorMap tmap_v, const UpdParams p) {
  constexpr int NA = LAST ? 2 : 3;
  constexpr bool BWD = MODE == UPD_BWD;
  constexpr int S = upd_stages(MODE);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;                                    // B(r, c) = wuv[r, c]: the U/V forward product
  uint8_t* sBd = sB + UPD_B;                             // BWD: B(r, c) = wuv[c, r]: the dgrad
  uint8_t* sA = sBd + (BWD ? UPD_B : 0);                 // S stages
  uint8_t* sG = sA + S * UPD_STAGE;                      // BWD: the [guv | gvv] tile, A operand of the dgrad
  uint64_t* full = reinterpret_cast<uint64_t*>(sG + (BWD ? UPD_G : 0));
  uint64_t* empty = full + S;
  float* sbias = reinterpret_cast<float*>(empty + S);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = (p.n + UPD_TILE - 1) / UPD_TILE;
  for (int i = threadIdx.x; i < 2 * UF; i += blockDim.x) sbias[i] = __ldg(p.buv + i);
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ===== TMA producer: the items (tile, d) of this CTA's tiles, in order =====
    if (lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        // the tile's per-node operands go to L2 now, S items before the consumer reads them with plain loads
        const int row0 = t * UPD_TILE, rows = min(UPD_TILE, p.n - row0);
        if (MODE == UPD_FWD || MODE == UPD_POST) prefetch_rows_l2(p.s, UF, row0, rows, 0, UF);
        if (MODE == UPD_POST) prefetch_rows_l2(p.a, NA * UF, row0, rows, 0, NA * UF);
        if (MODE == UPD_BWD_A || BWD) prefetch_rows_l2(p.gs_out, UF, row0, rows, 0, UF);
        if ((MODE == UPD_BWD_A || BWD) && !LAST) prefetch_rows_l2(p.gv_out, 3 * UF, row0, rows, 0, 3 * UF);
        if (BWD) {
          prefetch_rows_l2(p.g_mlp_in, 2 * UF, row0, rows, 0, 2 * UF);
          prefetch_rows_l2(p.mlp_in, 2 * UF, row0, rows, 0, UF);                       // |vv|
          prefetch_rows_l2(p.a, NA * UF, row0, rows, 0, (NA - 1) * UF);                // (a_vv,) a_sv
        }
        for (int d = 0; d < 3; ++d, ++it) {
          const int s = it % S;
          mbar_wait(empty + s, ((it / S) & 1) ^ 1);
          mbar_expect_tx(full + s, UPD_STAGE);
          tma_load_3d(sA + (size_t)s * UPD_STAGE, &tmap_v, full + s, 0, d, t * UPD_TILE);
          tma_load_3d(sA + (size_t)s * UPD_STAGE + UPD_STAGE / 2, &tmap_v, full + s, 32, d, t * UPD_TILE);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroup: stage the weights K-major (generic-proxy stores made visible to the async proxy) =====
  for (int i = threadIdx.x; i < 2 * UF * UF; i += 128) {
    const float w = __ldg(p.wuv + i);
    const int r = i / UF, c = i % UF;
    *reinterpret_cast<float*>(sB + kmajor_sw128_off(r, c, 2 * UF)) = w;
    if (BWD) *reinterpret_cast<float*>(sBd + kmajor_sw128_off(c, r, UF)) = w;
  }
  fence_proxy_async();
  named_bar_sync(1, 128);

  const int wq = warp;
  const int rsub = wq * 16 + (lane >> 2);                // this thread's tile rows: rsub and rsub + 8
  const int c2 = 2 * (lane & 3);                         // and columns 8 i + c2 (+ 1)
  const uint32_t sA_addr = smem_u32(sA), sB_addr = smem_u32(sB), sBd_addr = smem_u32(sBd);
  const uint32_t sG_addr = smem_u32(sG);

  float acc[64];
  uint32_t it = 0;                                       // items consumed so far
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int node = t * UPD_TILE + rsub;
    // per-node values kept over the three d of the tile (their meaning depends on the mode)
    float x0[32], x1[32], x2[32];
    if (MODE == UPD_FWD) {                               // mlp_in[:, 64:] = s
      frag_ld(x0, p.s + c2, UF, node, p.n);
      frag_st(p.mlp_in_out + UF + c2, 2 * UF, node, p.n, x0);
    }
    if ((MODE == UPD_POST || MODE == UPD_BWD) && !LAST) frag_ld(x2, p.a + c2, NA * UF, node, p.n);   // a_vv
    if (BWD) {                                           // x0 = g a_sv, x1 = gn / |vv| (0 at |vv| = 0), x2 = a_vv
      float g[32], q[32];
      frag_ld(g, p.gs_out + c2, UF, node, p.n);
      frag_ld(q, p.g_mlp_in + UF + c2, 2 * UF, node, p.n);
#pragma unroll
      for (int j = 0; j < 32; ++j) q[j] = g[j] + q[j];
      frag_st(p.gs + c2, UF, node, p.n, q);
      frag_ld(x0, p.a + (NA - 2) * UF + c2, NA * UF, node, p.n);
#pragma unroll
      for (int j = 0; j < 32; ++j) x0[j] = g[j] * x0[j];
      frag_ld(x1, p.mlp_in + c2, 2 * UF, node, p.n);
      frag_ld(q, p.g_mlp_in + c2, 2 * UF, node, p.n);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float nrm = x1[j];
        x1[j] = nrm > 0.f ? q[j] / nrm : 0.f;            // d|vv|/dvv = vv/|vv| (0 at the origin, as torch)
      }
    }
#pragma unroll 1
    for (int d = 0; d < 3; ++d, ++it) {
      const int s = it % S;
      float gvo[32];                                     // gv_out_d (BWD_A, BWD when not last)
      if ((MODE == UPD_BWD_A || BWD) && !LAST) frag_ld(gvo, p.gv_out + d * UF + c2, 3 * UF, node, p.n);
      mbar_wait(full + s, (it / S) & 1);
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.f;
      fence_regs<64>(acc);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4)
          wgmma_tf32<4>(acc, make_desc(sA_addr + s * UPD_STAGE + kb * (UPD_STAGE / 2) + k4 * 32),
                        make_desc(sB_addr + kb * (2 * UF) * 128 + k4 * 32));
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<64>(acc);
      const bool keep_stage = MODE == UPD_POST && !LAST;   // v_d is read from the stage below
      if (!keep_stage) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + s);
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {                     // uv = acc[j], vv = acc[32 + j]
        const int col = 8 * (j >> 2) + c2 + (j & 1);
        acc[j] = acc[j] + sbias[col];
        acc[32 + j] = acc[32 + j] + sbias[UF + col];
      }

      if (MODE == UPD_FWD) {
        if (p.inner_out) {                               // x0 = inner, as painn_update_post_fwd accumulates it; stored before x0 takes |vv|
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            if (d == 0) x0[j] = 0.f;
            x0[j] += acc[j] * acc[32 + j];
          }
          if (d == 2) frag_st(p.inner_out + c2, UF, node, p.n, x0);
        }
        if (d == 0) {
#pragma unroll
          for (int j = 0; j < 32; ++j) x1[j] = acc[32 + j];
        } else if (d == 1) {
#pragma unroll
          for (int j = 0; j < 32; ++j) x2[j] = acc[32 + j];
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float a = x1[j], b = x2[j], dd = acc[32 + j];
            x0[j] = sqrtf(a * a + b * b + dd * dd);
          }
          frag_st(p.mlp_in_out + c2, 2 * UF, node, p.n, x0);
        }
      }
      if (MODE == UPD_POST || MODE == UPD_BWD_A) {       // x0 = inner (x1 = sum_d gv_out_d uv_d)
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (d == 0) x0[j] = 0.f;
          const float u = acc[j];
          x0[j] += u * acc[32 + j];
          if (MODE == UPD_BWD_A && !LAST) {
            if (d == 0) x1[j] = 0.f;
            x1[j] += gvo[j] * u;
          }
        }
      }
      if (MODE == UPD_POST && !LAST) {
        float vo[32];
        const uint8_t* st = sA + (size_t)s * UPD_STAGE;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int r = rsub + 8 * ((j >> 1) & 1), col = 8 * (j >> 2) + c2 + (j & 1);
          vo[j] = *reinterpret_cast<const float*>(st + kmajor_sw128_off(r, col, UPD_TILE)) + x2[j] * acc[j];
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + s);
        frag_st(p.v_out + d * UF + c2, 3 * UF, node, p.n, vo);
      }
      if (BWD) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float u = acc[j], w = acc[32 + j];
          const float g_vo = LAST ? 0.f : gvo[j], a_vv = LAST ? 0.f : x2[j];
          // painn_update_bwd_kernel's guv and gvv, contracted the same explicit way
          acc[j] = fmaf(x0[j], w, g_vo * a_vv);
          acc[32 + j] = fmaf(x0[j], u, x1[j] * w);
        }
        frag_st(p.g_uv + d * 2 * UF + c2, 3 * 2 * UF, node, p.n, acc);
        frag_st(p.g_uv + d * 2 * UF + UF + c2, 3 * 2 * UF, node, p.n, acc + 32);
        named_bar_sync(1, 128);                     // the previous dgrad of this warpgroup has read sG
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const int r = rsub + 8 * ((j >> 1) & 1), col = 8 * (j >> 2) + c2;
          *reinterpret_cast<float2*>(sG + kmajor_sw128_off(r, col, UPD_TILE)) = make_float2(acc[j], acc[j + 1]);
          *reinterpret_cast<float2*>(sG + kmajor_sw128_off(r, UF + col, UPD_TILE)) = make_float2(acc[32 + j], acc[33 + j]);
        }
        fence_proxy_async();
        named_bar_sync(1, 128);                     // the whole [guv | gvv] tile is in shared memory
        float dg[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) dg[j] = 0.f;
        fence_regs<32>(dg);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < 4; ++kb)
#pragma unroll
          for (int k4 = 0; k4 < 4; ++k4)
            wgmma_tf32<2>(dg, make_desc(sG_addr + kb * (UPD_G / 4) + k4 * 32), make_desc(sBd_addr + kb * UF * 128 + k4 * 32));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs<32>(dg);
#pragma unroll
        for (int j = 0; j < 32; ++j) {                   // the dgrad epilogue: zero bias, then the direct path as addend
          float y = dg[j] + 0.f;
          if (!LAST) y += gvo[j];
          dg[j] = y;
        }
        frag_st(p.gv + d * UF + c2, 3 * UF, node, p.n, dg);
      }
    }
    if (MODE == UPD_POST) {                              // s_out = s + a_sv inner + a_ss
      float sv[32], ss[32];
      frag_ld(x1, p.s + c2, UF, node, p.n);
      frag_ld(sv, p.a + (NA - 2) * UF + c2, NA * UF, node, p.n);
      frag_ld(ss, p.a + (NA - 1) * UF + c2, NA * UF, node, p.n);
#pragma unroll
      for (int j = 0; j < 32; ++j) x1[j] = x1[j] + sv[j] * x0[j] + ss[j];
      frag_st(p.s_out + c2, UF, node, p.n, x1);
    }
    if (MODE == UPD_BWD_A) {                             // ga = [gdot (not last), g inner, g]
      float g[32];
      frag_ld(g, p.gs_out + c2, UF, node, p.n);
      if (!LAST) frag_st(p.ga + c2, NA * UF, node, p.n, x1);
#pragma unroll
      for (int j = 0; j < 32; ++j) x0[j] = g[j] * x0[j];
      frag_st(p.ga + (NA - 2) * UF + c2, NA * UF, node, p.n, x0);
      frag_st(p.ga + (NA - 1) * UF + c2, NA * UF, node, p.n, g);
    }
  }
}

// A last layer's post and ga need no [uv | vv]: only inner, which UPD_FWD stored.  Same formulas as painn_update_post_fwd /
// painn_update_post_bwd_a with na = 2.
__global__ void painn_update_tc_post_last_kernel(const float* __restrict__ s, const float* __restrict__ a, const float* __restrict__ inner,
                                                 int64_t nf, float* __restrict__ s_out) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nf; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / UF;
    const int c = (int)(t % UF);
    const float a_sv = a[i * 2 * UF + c], a_ss = a[i * 2 * UF + UF + c];
    s_out[t] = s[t] + a_sv * inner[t] + a_ss;
  }
}
__global__ void painn_update_tc_bwd_a_last_kernel(const float* __restrict__ gs_out, const float* __restrict__ inner, int64_t nf,
                                                  float* __restrict__ ga) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nf; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / UF;
    const int c = (int)(t % UF);
    const float g = gs_out[t];
    ga[i * 2 * UF + c] = g * inner[t];
    ga[i * 2 * UF + UF + c] = g;
  }
}

namespace {

template <int MODE, bool LAST>
int launch_update(const float* v, const UpdParams& p, hgb_stream_t stream, const char* name) {
  CUtensorMap tm;                                        // v [n, 3, 64] as dims {64, 3, n}: one box = 64 nodes x 32 features of one d
  const cuuint64_t dims[3] = {(cuuint64_t)UF, 3, (cuuint64_t)p.n};
  const cuuint64_t strides[2] = {(cuuint64_t)UF * 4, (cuuint64_t)3 * UF * 4};
  const cuuint32_t box[3] = {32, 1, (cuuint32_t)UPD_TILE};
  int rc = encode_tmap(&tm, v, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  constexpr size_t smem = upd_smem(MODE);
  static_assert(smem <= SMEM_MAX, "painn_update_tc: shared memory budget");
  static int per_sm = 0;                                 // resident CTAs per SM: the persistent grid is one wave
  if (!per_sm) {
    cudaFuncSetAttribute(painn_update_tc_kernel<MODE, LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, painn_update_tc_kernel<MODE, LAST>, UPD_THREADS, smem) != cudaSuccess ||
        per_sm < 1)
      per_sm = 1;
  }
  const int ntiles = (p.n + UPD_TILE - 1) / UPD_TILE;
  const int grid = ntiles < per_sm * HGB_NUM_SMS ? ntiles : per_sm * HGB_NUM_SMS;
  painn_update_tc_kernel<MODE, LAST><<<grid, UPD_THREADS, smem, (cudaStream_t)stream>>>(tm, p);
  HGB_LAUNCH_CHECK(name);
  return HGB_OK;
}

bool al16(const void* q) { return ((uintptr_t)q & 15) == 0; }

UpdParams upd_params(int n, const float* wuv, const float* buv) {
  UpdParams p = {};
  p.n = n;
  p.wuv = wuv;
  p.buv = buv;
  return p;
}

}  // namespace

extern "C" int hgb_painn_update_tc_fwd(const float* v, const float* s, const float* wuv, const float* buv, int32_t n, float* mlp_in,
                                       float* inner, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && v && s && wuv && buv && mlp_in, "painn_update_tc_fwd: bad arguments");
  HGB_REQUIRE(al16(v) && al16(s) && al16(mlp_in) && al16(inner), "painn_update_tc_fwd: operands must be 16-byte aligned");
  if (n == 0) return HGB_OK;
  UpdParams p = upd_params(n, wuv, buv);
  p.s = s;
  p.mlp_in_out = mlp_in;
  p.inner_out = inner;
  return launch_update<UPD_FWD, true>(v, p, stream, "painn_update_tc_fwd");
}

extern "C" int hgb_painn_update_tc_post(const float* v, const float* s, const float* a, const float* inner, const float* wuv,
                                        const float* buv, int32_t n, int32_t last, float* s_out, float* v_out, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && v && s && a && wuv && buv && s_out && (last ? inner != nullptr : v_out != nullptr), "painn_update_tc_post: bad arguments");
  HGB_REQUIRE(al16(v) && al16(s) && al16(a) && al16(s_out) && (last || al16(v_out)), "painn_update_tc_post: operands must be 16-byte aligned");
  if (n == 0) return HGB_OK;
  if (last) {
    const int64_t nf = (int64_t)n * UF;
    painn_update_tc_post_last_kernel<<<hgb_grid_for(nf, 256), 256, 0, (cudaStream_t)stream>>>(s, a, inner, nf, s_out);
    HGB_LAUNCH_CHECK("painn_update_tc_post_last");
    return HGB_OK;
  }
  UpdParams p = upd_params(n, wuv, buv);
  p.s = s;
  p.a = a;
  p.s_out = s_out;
  p.v_out = v_out;
  return launch_update<UPD_POST, false>(v, p, stream, "painn_update_tc_post");
}

extern "C" int hgb_painn_update_tc_bwd_a(const float* v, const float* gs_out, const float* gv_out, const float* inner, const float* wuv,
                                         const float* buv, int32_t n, int32_t last, float* ga, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && v && gs_out && wuv && buv && ga && (last ? inner != nullptr : gv_out != nullptr), "painn_update_tc_bwd_a: bad arguments");
  HGB_REQUIRE(al16(v) && al16(gs_out) && al16(ga) && (last || al16(gv_out)), "painn_update_tc_bwd_a: operands must be 16-byte aligned");
  if (n == 0) return HGB_OK;
  if (last) {
    const int64_t nf = (int64_t)n * UF;
    painn_update_tc_bwd_a_last_kernel<<<hgb_grid_for(nf, 256), 256, 0, (cudaStream_t)stream>>>(gs_out, inner, nf, ga);
    HGB_LAUNCH_CHECK("painn_update_tc_bwd_a_last");
    return HGB_OK;
  }
  UpdParams p = upd_params(n, wuv, buv);
  p.gs_out = gs_out;
  p.gv_out = gv_out;
  p.ga = ga;
  return launch_update<UPD_BWD_A, false>(v, p, stream, "painn_update_tc_bwd_a");
}

extern "C" int hgb_painn_update_tc_bwd(const float* v, const float* gs_out, const float* gv_out, const float* g_mlp_in, const float* a,
                                       const float* mlp_in, const float* wuv, const float* buv, int32_t n, int32_t last, float* g_uv,
                                       float* gs, float* gv, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && v && gs_out && g_mlp_in && a && mlp_in && wuv && buv && g_uv && gs && gv && (last || gv_out),
              "painn_update_tc_bwd: bad arguments");
  HGB_REQUIRE(al16(v) && al16(gs_out) && al16(g_mlp_in) && al16(a) && al16(mlp_in) && al16(g_uv) && al16(gs) && al16(gv) &&
                  (last || al16(gv_out)),
              "painn_update_tc_bwd: operands must be 16-byte aligned");
  if (n == 0) return HGB_OK;
  UpdParams p = upd_params(n, wuv, buv);
  p.gs_out = gs_out;
  p.gv_out = gv_out;
  p.g_mlp_in = g_mlp_in;
  p.a = a;
  p.mlp_in = mlp_in;
  p.g_uv = g_uv;
  p.gs = gs;
  p.gv = gv;
  return last ? launch_update<UPD_BWD, true>(v, p, stream, "painn_update_tc_bwd") : launch_update<UPD_BWD, false>(v, p, stream, "painn_update_tc_bwd");
}
