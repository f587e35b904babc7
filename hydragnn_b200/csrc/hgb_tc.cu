// libhgb.so -- tensor-core (wgmma / TMA / mbarrier) dense layers for the large-M, small-N/K GEMMs of the
// node/edge MLPs.  sm_90a only.
//
// Why TF32: activations live in HBM as fp32 (parameters are fp32 in every reference precision mode,
// hydragnn/train/train_validate_test.py:43-49).  wgmma .tf32 consumes fp32 bit patterns straight from shared
// memory, so the activation tiles go HBM -> smem by TMA with no conversion pass, and the result (10-bit mantissa
// products, fp32 accumulation in registers) is strictly more accurate than the bf16 autocast the reference runs
// under precision="bf16".  These GEMMs are memory-bound (AI ~ 12-24 FLOP/B), so TF32's half-rate is irrelevant.
//
// Kernels:
//   tc_linear_kernel  : Y[M,NO] = act(A[M,KR] . B^T + bias)   B = W (NO x KR, forward) or W^T (dgrad)
//                       persistent, warp-specialised: warp 0 = TMA producer, warps 1-3 = splitters (fp32-accurate mode),
//                       warpgroups 1 and 2 = consumers.  The weight operand is staged once per CTA (K-major, 128-byte
//                       swizzle); 64-row A tiles stream through mbarrier rings; the two consumer warpgroups take
//                       alternate tiles (ping-pong), each from its OWN ring, so the epilogue of one overlaps the wgmma of
//                       the other and every barrier is waited on phase by phase by the one warpgroup that consumes it.
//   tc_wgrad_kernel   : dW[NO,KO] (+ db[NO]) = dZ[M,NO]^T . X[M,KO], reduction over M split across CTAs, per-CTA partials +
//                       deterministic final reduce.  TF32 wgmma wants both operands K-major (M contiguous), the tensors are
//                       row-major: the TMA lands row slabs and the consumer warpgroups transpose them into a K-major buffer
//                       (splitting into TF32 hi / lo in fp32-accurate mode) while the previous buffer is on the tensor cores.
//                       The bias gradient rides along as 16 extra "ones" rows of the B operand.
#include <cuda.h>

#include "hgb_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ---- wgmma (warpgroup MMA: 4 warps, A and B from shared memory, D in registers) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// warpgroup register reallocation: the producer warpgroup hands registers to the accumulator-holding consumers
template <int R>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers

// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// D[64 x 32] += A[64 x 8] . B[32 x 8]^T, tf32 in, fp32 accumulate.  Fragment: d[4i + 2h + e] = D(16 w + lane/4 + 8h, 8i + 2(lane%4) + e)
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(ad), "l"(bd), "r"(1));
}
// D[64 x 16] += A[64 x 8] . B[16 x 8]^T
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(ad), "l"(bd), "r"(1));
}

// shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle: rows of 32 fp32 (128 B), 8-row groups 1024 B
// apart (SBO); the k-step of 8 tf32 inside the swizzle atom is a 32-byte advance of the start address.  The operand base must be
// 1024-byte aligned (the swizzle phase is taken from the address bits).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;                 // leading byte offset: unused by swizzled K-major operands
  d |= (uint64_t)(1024 >> 4) << 32;       // stride byte offset
  d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
  return d;
}

// byte offset of element (r, c) of a K-major SWIZZLE_128B operand stored as column blocks of 32 fp32:
// block cb = c/32 is a [rows x 128 B] slab; 8-row groups are 1024 B apart; 16-B chunks are XOR-swizzled by r%8
__device__ __forceinline__ uint32_t kmajor_sw128_off(int r, int c, int rows) {
  const int cb = c >> 5, cc = (c & 31) >> 2, j = c & 3;
  return (uint32_t)cb * rows * 128 + (uint32_t)(r >> 3) * 1024 + (uint32_t)(r & 7) * 128 + (uint32_t)((cc ^ (r & 7)) << 4) + j * 4;
}

// round to TF32 (10 mantissa bits), nearest, ties away from zero -- what cvt.rna.tf32.f32 does, as two full-rate integer
// instructions (the splitters run this on every operand element)
__device__ __forceinline__ float tf32_rna(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

__device__ __forceinline__ void split_f4(const float4 v, float4& h, float4& l) {
  h.x = tf32_rna(v.x); h.y = tf32_rna(v.y); h.z = tf32_rna(v.z); h.w = tf32_rna(v.w);
  l.x = tf32_rna(v.x - h.x); l.y = tf32_rna(v.y - h.y); l.z = tf32_rna(v.z - h.z); l.w = tf32_rna(v.w - h.w);
}

struct LinParams {
  int m, kr, no;        // rows, reduction length, output columns
  const float* w;       // weight matrix [n_w, k_w], row stride ldw
  int64_t ldw;
  int trans_b;          // 0: B(r, c) = w[r, c] (forward: no = n_w, kr = k_w); 1: B(r, c) = w[c, r] (dgrad: no = k_w, kr = n_w)
  const float* bias;
  int act;
  float act_param;
  float* y;
  float* z;
  const float* addend;  // optional [m, no] (row stride ldy): y = act(a.B^T + bias) + addend  (gradient accumulation without an extra pass)
  int64_t ldy;          // row stride of y / z / addend (>= no: column chunks of a wider matrix)
  const float* gsrc;    // optional [m, no] (row stride ldy): the result is multiplied by act'(gsrc), i.e. this GEMM is the dgrad of a
  int gact;             //   layer whose INPUT was act(.): gsrc = saved pre-activation (SiLU) or activation output (others)
  int z_deriv;          // forward with a SiLU and z != NULL: z receives silu'(pre-activation) instead of the pre-activation
  int stages;           // in total: two rings (one per consumer warpgroup) of stages / 2 each
  int split;            // 1: fp32-accurate mode -- every operand is split into a TF32 hi / lo pair and each k-step runs the three
                        //    products lo*hi + hi*lo + hi*hi (3xTF32); warps 1..3 split the A stages in shared memory
};

constexpr int TILE_M = 64;                       // rows per tile = one wgmma M
constexpr uint32_t A_STAGE = TILE_M * 128;       // one pipeline stage = one [64 x 32 fp32] k-block (8 KB)
constexpr int LIN_THREADS = 384;

// the epilogue of two adjacent outputs (row, col), (row, col + 1)
__device__ __forceinline__ void lin_epilogue2(const LinParams& p, const float* sbias, int row, int col, float v0, float v1) {
  if (row >= p.m) return;
  const int64_t o = (int64_t)row * p.ldy + col;
  v0 += sbias[col];
  v1 += sbias[col + 1];
  if (p.z && !(p.z_deriv && p.act == HGB_ACT_SILU)) *reinterpret_cast<float2*>(p.z + o) = make_float2(v0, v1);
  switch (p.act) {
    case HGB_ACT_NONE: break;
    case HGB_ACT_RELU: v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); break;
    case HGB_ACT_SILU:
      if (p.z && p.z_deriv) {   // z receives silu'(pre) = s + y (1 - s): the backward then needs one multiply per element
        const float s0 = __fdividef(1.f, 1.f + __expf(-v0)), s1 = __fdividef(1.f, 1.f + __expf(-v1));
        v0 *= s0;
        v1 *= s1;
        *reinterpret_cast<float2*>(p.z + o) = make_float2(fmaf(v0, 1.f - s0, s0), fmaf(v1, 1.f - s1, s1));
      } else {
        v0 = __fdividef(v0, 1.f + __expf(-v0));
        v1 = __fdividef(v1, 1.f + __expf(-v1));
      }
      break;
    case HGB_ACT_TANH: v0 = tanhf(v0); v1 = tanhf(v1); break;
    default: v0 = hgb_act(v0, p.act, p.act_param); v1 = hgb_act(v1, p.act, p.act_param);
  }
  if (p.addend) {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p.addend + o));
    v0 += a.x;
    v1 += a.y;
  }
  if (p.gsrc) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(p.gsrc + o));
    if (p.gact == HGB_ACT_DERIV) {          // gsrc already holds act'(.)
      v0 *= g.x;
      v1 *= g.y;
    } else {
      v0 *= hgb_act_grad(g.x, g.x, p.gact, p.act_param);
      v1 *= hgb_act_grad(g.y, g.y, p.gact, p.act_param);
    }
  }
  *reinterpret_cast<float2*>(p.y + o) = make_float2(v0, v1);
}

template <int NC, bool SPLIT>   // NO = 32 * NC output columns; SPLIT: the fp32-accurate mode
__global__ void __launch_bounds__(LIN_THREADS, 1) tc_linear_kernel(const __grid_constant__ CUtensorMap tmap_a, const LinParams p) {
  constexpr int NO = NC * 32;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int KB = p.kr >> 5;
  const uint32_t b_pad = ((uint32_t)KB * NO * 128 + 1023) & ~1023u;
  uint8_t* sB = smem;
  uint8_t* sBlo = sB + b_pad;                                 // split mode only
  uint8_t* sA = sB + (SPLIT ? 2 : 1) * (size_t)b_pad;
  const int S = p.stages;
  const int SR = S >> 1;                                      // stages per ring: stage (r * SR + slot) belongs to ring r
  uint8_t* sAlo = sA + (size_t)S * A_STAGE;                   // split mode only
  uint64_t* full = reinterpret_cast<uint64_t*>(sA + (size_t)(SPLIT ? 2 : 1) * S * A_STAGE);
  uint64_t* empty = full + S;
  uint64_t* full2 = empty + S;                                // split mode: "stage s is split" (3 splitter warps arrive)
  float* sbias = reinterpret_cast<float*>(full2 + S);         // [NO]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = (p.m + TILE_M - 1) / TILE_M;
  for (int i = threadIdx.x; i < NO; i += blockDim.x) sbias[i] = p.bias ? __ldg(p.bias + i) : 0.f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 4); mbar_init(full2 + s, 3); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_dec<PRODUCER_REGS>();
    if (warp == 0) {
    // ===== TMA producer: the A k-blocks of this CTA's tiles, in order; local tile li goes to ring li & 1 (its consumer's) =====
    if (lane == 0) {
      uint32_t li = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++li)
        for (int kb = 0; kb < KB; ++kb) {
          const uint32_t n = (li >> 1) * KB + kb;             // item index within the ring
          const int s = (li & 1) * SR + n % SR;
          mbar_wait(empty + s, ((n / SR) & 1) ^ 1);
          mbar_expect_tx(full + s, A_STAGE);
          tma_load_2d(sA + (size_t)s * A_STAGE, &tmap_a, full + s, kb * 32, t * TILE_M);
        }
    }
    } else {
    // ===== splitters (split mode only): as soon as the TMA has landed stage s, rewrite it in place as the TF32 "hi" part and put the
    // "lo" remainder at the same (swizzled) offsets of the twin buffer, then release the stage to its consumer =====
    if (SPLIT) {
      const int tl = threadIdx.x - 32;
      uint32_t li = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++li)
        for (int kb = 0; kb < KB; ++kb) {                     // every item of both rings, in the producer's order
          const uint32_t n = (li >> 1) * KB + kb;
          const int s = (li & 1) * SR + n % SR;
          mbar_wait(full + s, (n / SR) & 1);
          float4* pa = reinterpret_cast<float4*>(sA + (size_t)s * A_STAGE);
          float4* pl = reinterpret_cast<float4*>(sAlo + (size_t)s * A_STAGE);
          for (int idx = tl; idx < (int)(A_STAGE / 16); idx += 96) {
            float4 h, l;
            split_f4(pa[idx], h, l);
            pa[idx] = h;
            pl[idx] = l;
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(full2 + s);
        }
    }
    }
  } else {
    regs_inc<CONSUMER_REGS>();
    // ===== consumer warpgroups: stage the weight operand into its K-major SWIZZLE_128B layout (generic-proxy stores made visible to the
    // async proxy), then run wgmma + epilogue on alternate tiles =====
    {
      const int total = NO * p.kr;
      constexpr int SU = 8;   // independent loads in flight per thread: the staging is latency-, not bandwidth-limited
      for (int base = threadIdx.x - 128; base < total; base += 256 * SU) {
        float val[SU];
        uint32_t off[SU];
#pragma unroll
        for (int u = 0; u < SU; ++u) {
          const int i = base + u * 256;
          val[u] = 0.f;
          off[u] = 0xffffffffu;
          if (i < total) {
            if (!p.trans_b) {
              const int r = i / p.kr, c = i - r * p.kr;
              off[u] = kmajor_sw128_off(r, c, NO);
              val[u] = __ldg(p.w + (int64_t)r * p.ldw + c);
            } else {
              const int c = i / NO, r = i - c * NO;  // r fastest: w[c, r] is contiguous in r
              off[u] = kmajor_sw128_off(r, c, NO);
              val[u] = __ldg(p.w + (int64_t)c * p.ldw + r);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < SU; ++u)
          if (off[u] != 0xffffffffu) {
            if (SPLIT) {
              const float hi = tf32_rna(val[u]);
              *reinterpret_cast<float*>(sB + off[u]) = hi;
              *reinterpret_cast<float*>(sBlo + off[u]) = tf32_rna(val[u] - hi);
            } else {
              *reinterpret_cast<float*>(sB + off[u]) = val[u];
            }
          }
      }
      fence_proxy_async();
    }
    named_bar_sync(1, 256);
    const int cw = (warp - 4) >> 2;     // consumer warpgroup: takes local tiles cw, cw + 2, ... from ring cw, every item in order
    const int wq = warp & 3;            // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of the tile
    const uint32_t sA_addr = smem_u32(sA), sAlo_addr = smem_u32(sAlo), sB_addr = smem_u32(sB), sBlo_addr = smem_u32(sBlo);
    float acc[NC][16];
    int li = cw;
    for (int t = blockIdx.x + cw * gridDim.x; t < ntiles; t += 2 * gridDim.x, li += 2) {
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[c][j] = 0.f;
      const uint32_t n0 = (uint32_t)(li >> 1) * KB;             // first item of this tile within ring cw
      for (int kb = 0; kb < KB; ++kb) {
        const uint32_t n = n0 + kb;
        const int s = cw * SR + n % SR;
        mbar_wait(SPLIT ? full2 + s : full + s, (n / SR) & 1);
        fence_regs<NC * 16>(&acc[0][0]);
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const uint64_t ad = make_desc(sA_addr + s * A_STAGE + k4 * 32);
          const uint64_t adl = make_desc(sAlo_addr + s * A_STAGE + k4 * 32);
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const uint32_t boff = (uint32_t)kb * NO * 128 + c * 4096 + k4 * 32;
            const uint64_t bd = make_desc(sB_addr + boff);
            if (SPLIT) {        // small terms first: lo*hi + hi*lo + hi*hi
              wgmma_n32(acc[c], adl, bd);
              wgmma_n32(acc[c], ad, make_desc(sBlo_addr + boff));
            }
            wgmma_n32(acc[c], ad, bd);
          }
        }
        wgmma_commit();
        fence_regs<NC * 16>(&acc[0][0]);
        if (kb > 0) {                   // the MMAs of the previous k-block have read their stage: release it
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(empty + cw * SR + (n - 1) % SR);
        }
      }
      wgmma_wait<0>();
      fence_regs<NC * 16>(&acc[0][0]);
      if (lane == 0) mbar_arrive(empty + cw * SR + (n0 + KB - 1) % SR);
      // ===== epilogue straight from the accumulator registers =====
      const int r0 = t * TILE_M + wq * 16 + (lane >> 2);
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int col = c * 32 + i * 8 + 2 * (lane & 3);
          lin_epilogue2(p, sbias, r0, col, acc[c][4 * i], acc[c][4 * i + 1]);
          lin_epilogue2(p, sbias, r0 + 8, col, acc[c][4 * i + 2], acc[c][4 * i + 3]);
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// weight gradient: dW[NO, KO] (+ db[NO]) = sum_m dZ[m, NO]^T X[m, KO]
// ------------------------------------------------------------------------------------------------
struct WgParams {
  int m, no, ko;
  int chunks_per_cta;   // number of 32-row chunks each CTA reduces
  int stages;           // TMA ring of raw row slabs
  int tbufs;            // K-major (transposed) operand buffers: 2 = transposition of chunk c+1 overlaps the MMAs of chunk c
  int split;            // 1: fp32-accurate mode -- both operands are split into TF32 hi / lo twins and every k-step runs lo*hi + hi*lo + hi*hi
  int flush;            // > 0: the register accumulators are added into the partial every `flush` chunks and restarted, so each chain
                        //   of tensor-core additions stays short (the fp32-accurate mode)
  float* part;          // [gridDim.x, no, ko + 1]
};

constexpr int WG_ROWS = 32;                      // rows of dZ / X per chunk = one 128-byte K-major row of the transposed operands
constexpr int WG_NA = 128;                       // rows of dW per CTA (two consumer warpgroups x 64)
constexpr int WG_THREADS = 384;                  // 2 consumer warpgroups + 1 producer warpgroup (one warp issues the TMA)

template <int Q, bool SPLIT>    // KO = 32 * Q; SPLIT: the fp32-accurate mode
__global__ void __launch_bounds__(WG_THREADS, 1) tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dz,
                                                                 const __grid_constant__ CUtensorMap tmap_x, const WgParams p) {
  constexpr int KO = 32 * Q, NB = KO + 16;
  constexpr uint32_t SLAB = WG_ROWS * 128;       // one [32 rows x 32 fp32] TMA box
  constexpr uint32_t HI_BYTES = (uint32_t)(WG_NA + NB) * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int n0 = blockIdx.y * WG_NA;
  const int nrows = min(WG_NA, p.no - n0);
  const int nsl = nrows >> 5;
  const uint32_t raw_bytes = (uint32_t)(nsl + Q) * SLAB;
  const uint32_t tb_bytes = HI_BYTES * (SPLIT ? 2 : 1);
  const int S = p.stages, T = p.tbufs;
  uint8_t* tbuf = smem;                                   // T x [A hi (128 rows) | B hi (NB rows) | A lo | B lo]
  uint8_t* raw = smem + (size_t)T * tb_bytes;             // S x [nsl dZ slabs | Q X slabs], row-major as loaded
  uint64_t* full = reinterpret_cast<uint64_t*>(raw + (size_t)S * raw_bytes);
  uint64_t* empty = full + S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int total_chunks = (p.m + WG_ROWS - 1) / WG_ROWS;
  const int c_beg = blockIdx.x * p.chunks_per_cta;
  const int nchunks = max(0, min(total_chunks, c_beg + p.chunks_per_cta) - c_beg);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 8); }
    fence_barrier_init();
  }
  // transposed buffers: A rows >= nrows stay zero, B rows KO.. are the ones rows (lo twins: zero); everything else is rewritten per chunk
  for (int i = threadIdx.x; i < (int)(T * tb_bytes / 4); i += blockDim.x) {
    const uint32_t o = (uint32_t)i * 4 % tb_bytes;
    const bool lo = o >= HI_BYTES;
    const int row = (int)((lo ? o - HI_BYTES : o) / 128);
    reinterpret_cast<float*>(tbuf)[i] = (!lo && row >= WG_NA + KO) ? 1.f : 0.f;
  }
  fence_proxy_async();
  __syncthreads();

  if (warp >= 8) {
    // ===== TMA producer: this CTA's dZ columns n0.. and all of X, 32 rows per chunk =====
    regs_dec<PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      for (int c = 0; c < nchunks; ++c) {
        const int s = c % S;
        mbar_wait(empty + s, ((c / S) & 1) ^ 1);
        mbar_expect_tx(full + s, raw_bytes);
        uint8_t* st = raw + (size_t)s * raw_bytes;
        const int row0 = (c_beg + c) * WG_ROWS;
        for (int j = 0; j < nsl; ++j) tma_load_2d(st + (size_t)j * SLAB, &tmap_dz, full + s, n0 + j * 32, row0);
        for (int j = 0; j < Q; ++j) tma_load_2d(st + (size_t)(nsl + j) * SLAB, &tmap_x, full + s, j * 32, row0);
      }
    }
    return;
  }

  // ===== consumer warpgroups (threads 0..255): transpose, then wgmma; warpgroup wg owns dW rows n0 + 64 wg .. +63 =====
  regs_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const bool mma_on = wg * 64 < nrows;
  const int rows_t = nsl * 32 + KO;                       // operand rows to transpose per chunk
  float acc[Q][16], accb[8];
#pragma unroll
  for (int c = 0; c < Q; ++c)
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[c][j] = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) accb[j] = 0.f;
  bool first = true;
  float* part = p.part + (size_t)blockIdx.x * p.no * (p.ko + 1);

  auto flush = [&]() {   // partial (+)= accumulators; accumulators restart at zero
    if (mma_on) {
      const int rb = n0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rb + 8 * h;
        if (row < n0 + nrows) {
          float* pr = part + (size_t)row * (KO + 1);
#pragma unroll
          for (int c = 0; c < Q; ++c)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int col = c * 32 + i * 8 + 2 * (lane & 3) + e;
                const float v = acc[c][4 * i + 2 * h + e];
                pr[col] = first ? v : pr[col] + v;
              }
          if ((lane & 3) == 0) pr[KO] = first ? accb[2 * h] : pr[KO] + accb[2 * h];   // ones column KO: the bias gradient
        }
      }
    }
    first = false;
#pragma unroll
    for (int c = 0; c < Q; ++c)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[c][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) accb[j] = 0.f;
  };

  for (int c = 0; c < nchunks; ++c) {
    const int s = c % S;
    uint8_t* tb = tbuf + (size_t)(c % T) * tb_bytes;
    const uint8_t* st = raw + (size_t)s * raw_bytes;
    mbar_wait(full + s, (c / S) & 1);
    // transpose: operand row r (A: dZ column n0 + r; B: X column r - nrows) gets the 32 values of this chunk as one K-major 128-byte
    // row; each item is 4 consecutive m of one row (four conflict-free column reads, one swizzled 16-byte store)
    for (int it = threadIdx.x; it < rows_t * 8; it += 256) {
      const int r = it % rows_t, m4 = it / rows_t;
      const int slab = r < nrows ? r >> 5 : nsl + ((r - nrows) >> 5);
      const float* src = reinterpret_cast<const float*>(st + (size_t)slab * SLAB) + (r & 31) + m4 * 4 * 32;
      const float4 v = make_float4(src[0], src[32], src[64], src[96]);
      const int orow = r < nrows ? r : WG_NA + (r - nrows);
      const uint32_t off = (uint32_t)orow * 128 + ((m4 ^ (orow & 7)) << 4);
      if (SPLIT) {
        float4 h, l;
        split_f4(v, h, l);
        *reinterpret_cast<float4*>(tb + off) = h;
        *reinterpret_cast<float4*>(tb + HI_BYTES + off) = l;
      } else {
        *reinterpret_cast<float4*>(tb + off) = v;
      }
    }
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + s);               // the raw slabs are no longer needed
    named_bar_sync(1, 256);                              // the transposed chunk is complete
    if (mma_on) {
      const uint32_t ta = smem_u32(tb);
      fence_regs<Q * 16>(&acc[0][0]);
      fence_regs<8>(accb);
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint32_t aoff = (uint32_t)(wg * 64) * 128 + k4 * 32;
        const uint64_t ad = make_desc(ta + aoff), adl = make_desc(ta + HI_BYTES + aoff);
#pragma unroll
        for (int j = 0; j < Q; ++j) {
          const uint32_t boff = (uint32_t)WG_NA * 128 + (uint32_t)j * 4096 + k4 * 32;
          const uint64_t bd = make_desc(ta + boff);
          if (SPLIT) {                                   // small terms first: lo*hi + hi*lo + hi*hi
            wgmma_n32(acc[j], adl, bd);
            wgmma_n32(acc[j], ad, make_desc(ta + HI_BYTES + boff));
          }
          wgmma_n32(acc[j], ad, bd);
        }
        const uint64_t bones = make_desc(ta + (uint32_t)(WG_NA + KO) * 128 + k4 * 32);   // the 16 ones rows (lo(1) = 0: no hi*lo term)
        if (SPLIT) wgmma_n16(accb, adl, bones);
        wgmma_n16(accb, ad, bones);
      }
      wgmma_commit();
      fence_regs<Q * 16>(&acc[0][0]);
      fence_regs<8>(accb);
    }
    // the buffer transposed next must no longer be read by either warpgroup's MMAs
    if (T == 2) wgmma_wait<1>(); else wgmma_wait<0>();
    if (p.flush && (c + 1) % p.flush == 0 && c + 1 < nchunks) {
      wgmma_wait<0>();
      fence_regs<Q * 16>(&acc[0][0]);
      fence_regs<8>(accb);
      flush();
    }
    named_bar_sync(2, 256);
  }
  wgmma_wait<0>();
  fence_regs<Q * 16>(&acc[0][0]);
  fence_regs<8>(accb);
  flush();                                                // (a CTA without chunks writes zeros)
}

// 32 outputs x 8 partial-walkers per block; fixed summation order
__global__ void tc_wgrad_reduce_kernel(const float* __restrict__ part, int nparts, int no, int ko, float* __restrict__ dw,
                                       int64_t lddw, float* __restrict__ db, int accumulate) {
  __shared__ float red[8][33];
  const int w = ko + 1;
  const int cnt = no * w;
  const int i = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (i < cnt) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;   // four independent load chains
    int b = threadIdx.y;
    for (; b + 24 < nparts; b += 32) {
      a0 += part[(size_t)b * cnt + i]; a1 += part[(size_t)(b + 8) * cnt + i];
      a2 += part[(size_t)(b + 16) * cnt + i]; a3 += part[(size_t)(b + 24) * cnt + i];
    }
    for (; b < nparts; b += 8) a0 += part[(size_t)b * cnt + i];
    acc = (a0 + a1) + (a2 + a3);
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && i < cnt) {
    float t = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][threadIdx.x];
    const int r = i / w, c = i % w;
    if (c == ko) {
      if (db) db[r] = accumulate ? db[r] + t : t;
    } else {
      float* o = dw + (int64_t)r * lddw + c;
      *o = accumulate ? *o + t : t;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 2-D fp32 row-major tensor [rows, cols] with row stride ld (elements); box = [box_rows x 32 cols]
int make_tmap(CUtensorMap* tm, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, CUtensorMapSwizzle swz) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { hgb_set_error("tc: cuTensorMapEncodeTiled is not available from the driver"); return HGB_ECUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { hgb_set_error("tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return HGB_ECUDA; }
  return HGB_OK;
}

bool shape_ok(int kr, int no) { return kr >= 32 && kr <= 256 && kr % 32 == 0 && no >= 32 && no <= 256 && no % 32 == 0; }

constexpr size_t SMEM_MAX = 227 * 1024;          // opt-in dynamic shared memory per block

template <int NC, bool SPLIT>
void launch_linear_t(int grid, size_t smem, cudaStream_t st, const CUtensorMap& tm, const LinParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(tc_linear_kernel<NC, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
    attr_set = true;
  }
  tc_linear_kernel<NC, SPLIT><<<grid, LIN_THREADS, smem, st>>>(tm, p);
}
template <int NC>
void launch_linear(int grid, size_t smem, cudaStream_t st, const CUtensorMap& tm, const LinParams& p) {
  if (p.split) launch_linear_t<NC, true>(grid, smem, st, tm, p); else launch_linear_t<NC, false>(grid, smem, st, tm, p);
}

template <int Q, bool SPLIT>
void launch_wgrad_t(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& tdz, const CUtensorMap& tx, const WgParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(tc_wgrad_kernel<Q, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
    attr_set = true;
  }
  tc_wgrad_kernel<Q, SPLIT><<<grid, WG_THREADS, smem, st>>>(tdz, tx, p);
}
template <int Q>
void launch_wgrad(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& tdz, const CUtensorMap& tx, const WgParams& p) {
  if (p.split) launch_wgrad_t<Q, true>(grid, smem, st, tdz, tx, p); else launch_wgrad_t<Q, false>(grid, smem, st, tdz, tx, p);
}

}  // namespace

// wide operands are cut into <= 256-column / <= 256-deep pieces (see hgb_tc_linear below)
static bool wide_ok(int kr, int no) { return kr >= 32 && kr <= 1024 && kr % 32 == 0 && no >= 32 && no <= 1024 && no % 32 == 0; }

extern "C" int hgb_tc_linear_supported(int32_t m, int32_t n_out, int32_t k_red) { return (m >= 128 && wide_ok(k_red, n_out)) ? 1 : 0; }

// one (<= 256) x (<= 256) piece: y[m, no] = act(a[m, kr] . B^T + bias) + addend, y / z / addend with row stride ldy
static int tc_linear_piece(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t trans_b, const float* bias, int32_t m,
                           int32_t n_out, int32_t k_red, int32_t act, float act_param, float* y, float* z, const float* addend,
                           const float* gsrc, int32_t gact, int64_t ldy, int32_t exact, hgb_stream_t stream) {
  HGB_REQUIRE(a && w && y && m >= 128 && shape_ok(k_red, n_out), "tc_linear: unsupported shape m=%d n=%d k=%d", m, n_out, k_red);
  HGB_REQUIRE(lda % 4 == 0 && ldy % 4 == 0 && ((uintptr_t)a % 16 == 0) && ((uintptr_t)y % 16 == 0) && (!z || (uintptr_t)z % 16 == 0),
              "tc_linear: operands must be 16-byte aligned with a row stride that is a multiple of 4");
  CUtensorMap tm;
  int rc = make_tmap(&tm, a, m, k_red, lda, TILE_M, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  LinParams p;
  p.m = m; p.kr = k_red; p.no = n_out; p.w = w; p.ldw = ldw; p.trans_b = trans_b; p.bias = bias; p.act = act; p.act_param = act_param;
  p.y = y; p.z = z; p.addend = addend; p.ldy = ldy; p.gsrc = gsrc; p.gact = gact; p.z_deriv = (!gsrc && gact == HGB_ACT_DERIV) ? 1 : 0;
  const int KB = k_red / 32;
  const int dup = exact ? 2 : 1;                   // split mode keeps a hi and a lo copy of the weights and of every A stage
  const size_t b_bytes = ((size_t)KB * n_out * 128 + 1023) & ~(size_t)1023;
  const size_t fixed = 1024 + dup * b_bytes + (size_t)n_out * 4 + 64;
  int stages = fixed < SMEM_MAX ? (int)((SMEM_MAX - fixed) / (dup * A_STAGE + 3 * 8)) : 0;
  if (stages > 8) stages = 8;
  stages &= ~1;                                    // two equal rings, one per consumer warpgroup
  HGB_REQUIRE(stages >= 4, "tc_linear: weight operand does not fit shared memory (n=%d k=%d)", n_out, k_red);
  p.stages = stages;
  p.split = exact ? 1 : 0;
  const size_t smem = fixed + (size_t)stages * (dup * A_STAGE + 3 * 8);
  const int ntiles = (m + TILE_M - 1) / TILE_M;
  const int grid = ntiles < HGB_NUM_SMS ? ntiles : HGB_NUM_SMS;
  cudaStream_t st = (cudaStream_t)stream;
  switch (n_out / 32) {
    case 1: launch_linear<1>(grid, smem, st, tm, p); break;
    case 2: launch_linear<2>(grid, smem, st, tm, p); break;
    case 3: launch_linear<3>(grid, smem, st, tm, p); break;
    case 4: launch_linear<4>(grid, smem, st, tm, p); break;
    case 5: launch_linear<5>(grid, smem, st, tm, p); break;
    case 6: launch_linear<6>(grid, smem, st, tm, p); break;
    case 7: launch_linear<7>(grid, smem, st, tm, p); break;
    default: launch_linear<8>(grid, smem, st, tm, p); break;
  }
  HGB_LAUNCH_CHECK("tc_linear");
  return HGB_OK;
}

// y[m, no] = act(a[m, kr] . B^T + bias) + addend;  B(r, c) = w[r, c] (trans_b = 0) or w[c, r] (trans_b = 1).
// no > 256: independent column pieces.  kr > 256: the pieces of the reduction accumulate through `addend` (linear layers
// only: an activation or a saved pre-activation needs the whole sum first).
extern "C" int hgb_tc_linear(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t trans_b, const float* bias, int32_t m,
                             int32_t n_out, int32_t k_red, int32_t act, float act_param, float* y, float* z, const float* addend,
                             const float* gsrc, int32_t gact, int32_t exact, hgb_stream_t stream) {
  HGB_REQUIRE(a && w && y && hgb_tc_linear_supported(m, n_out, k_red), "tc_linear: unsupported shape m=%d n=%d k=%d", m, n_out, k_red);
  HGB_REQUIRE(k_red <= 256 || (act == HGB_ACT_NONE && !z && !gsrc), "tc_linear: reduction length %d > 256 needs a plain linear layer", k_red);
  // piece sizes: the B piece (kc x nc fp32) stays resident in shared memory next to >= 2 A stages per consumer ring
  const int kc_max = k_red < 256 ? k_red : 256;
  int nc_max = (int)(((exact ? 64 : 160) * 1024) / (4 * (size_t)kc_max) / 32) * 32;     // split mode: two weight copies + two copies per A stage
  if (nc_max > 256) nc_max = 256;
  for (int c0 = 0; c0 < n_out; c0 += nc_max) {
    const int nc = n_out - c0 < nc_max ? n_out - c0 : nc_max;
    for (int k0 = 0; k0 < k_red; k0 += 256) {
      const int kc = k_red - k0 < 256 ? k_red - k0 : 256;
      // B piece: rows = output columns c0.., columns = reduction k0..
      const float* wp = trans_b ? w + (int64_t)k0 * ldw + c0 : w + (int64_t)c0 * ldw + k0;
      const float* add = k0 == 0 ? (addend ? addend + c0 : nullptr) : y + c0;
      int rc = tc_linear_piece(a + k0, lda, wp, ldw, trans_b, (bias && k0 == 0) ? bias + c0 : nullptr, m, nc, kc, act, act_param, y + c0,
                               z ? z + c0 : nullptr, add, gsrc ? gsrc + c0 : nullptr, gact, n_out, exact, stream);
      if (rc) return rc;
    }
  }
  return HGB_OK;
}

extern "C" int64_t hgb_tc_wgrad_workspace_bytes(int32_t n_out, int32_t k_out) { return (int64_t)HGB_NUM_SMS * n_out * (k_out + 1) * 4; }

// dw[no, ko] (row stride lddw) (+)= dz[m, no]^T x[m, ko];  db[no] (+)= column sums of dz (db may be NULL)
extern "C" int hgb_tc_wgrad(const float* dz, int64_t lddz, const float* x, int64_t ldx, int32_t m, int32_t n_out, int32_t k_out,
                            float* dw, int64_t lddw, float* db, int32_t accumulate, int32_t exact, void* workspace,
                            int64_t workspace_bytes, hgb_stream_t stream) {
  HGB_REQUIRE(dz && x && dw && workspace && m >= 128 && shape_ok(k_out, n_out) && k_out + 16 <= 256,
              "tc_wgrad: unsupported shape m=%d n=%d k=%d", m, n_out, k_out);
  HGB_REQUIRE(lddz % 4 == 0 && ldx % 4 == 0 && ((uintptr_t)dz % 16 == 0) && ((uintptr_t)x % 16 == 0), "tc_wgrad: operands must be 16-byte aligned");
  HGB_REQUIRE(workspace_bytes >= hgb_tc_wgrad_workspace_bytes(n_out, k_out), "tc_wgrad: workspace too small");
  WgParams p;
  p.m = m; p.no = n_out; p.ko = k_out;
  p.split = exact ? 1 : 0;
  // fp32-accurate mode: restart the register accumulators every 8 chunks (256 rows), so no chain of tensor-core additions grows long
  p.flush = exact ? 8 : 0;
  const int Q = k_out / 32;
  const int nsl_max = (n_out < WG_NA ? n_out : WG_NA) / 32;
  const size_t raw_bytes = (size_t)(nsl_max + Q) * WG_ROWS * 128;
  const size_t tb_bytes = (size_t)(WG_NA + k_out + 16) * 128 * (exact ? 2 : 1);
  const size_t budget = SMEM_MAX - 1024 - 256;
  int tbufs = 2;
  int stages = budget > 2 * tb_bytes ? (int)((budget - 2 * tb_bytes) / raw_bytes) : 0;
  if (stages < 2) {
    tbufs = 1;
    stages = (int)((budget - tb_bytes) / raw_bytes);
  }
  if (stages > 4) stages = 4;
  HGB_REQUIRE(stages >= 2, "tc_wgrad: stage does not fit shared memory");
  p.stages = stages;
  p.tbufs = tbufs;
  CUtensorMap tdz, tx;
  int rc = make_tmap(&tdz, dz, m, n_out, lddz, WG_ROWS, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  rc = make_tmap(&tx, x, m, k_out, ldx, WG_ROWS, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  const int total_chunks = (m + WG_ROWS - 1) / WG_ROWS;
  const int gy = (n_out + WG_NA - 1) / WG_NA;
  const int max_x = HGB_NUM_SMS / gy;
  int gx = total_chunks < max_x ? total_chunks : max_x;
  p.chunks_per_cta = (total_chunks + gx - 1) / gx;
  gx = (total_chunks + p.chunks_per_cta - 1) / p.chunks_per_cta;
  p.part = (float*)workspace;
  const size_t smem = 1024 + tbufs * tb_bytes + stages * raw_bytes + 2 * stages * 8;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(gx, gy);
  switch (Q) {
    case 1: launch_wgrad<1>(grid, smem, st, tdz, tx, p); break;
    case 2: launch_wgrad<2>(grid, smem, st, tdz, tx, p); break;
    case 3: launch_wgrad<3>(grid, smem, st, tdz, tx, p); break;
    case 4: launch_wgrad<4>(grid, smem, st, tdz, tx, p); break;
    case 5: launch_wgrad<5>(grid, smem, st, tdz, tx, p); break;
    case 6: launch_wgrad<6>(grid, smem, st, tdz, tx, p); break;
    default: launch_wgrad<7>(grid, smem, st, tdz, tx, p); break;
  }
  HGB_LAUNCH_CHECK("tc_wgrad");
  const int outs = n_out * (k_out + 1);
  tc_wgrad_reduce_kernel<<<(outs + 31) / 32, dim3(32, 8), 0, st>>>(p.part, gx, n_out, k_out, dw, lddw, db, accumulate);
  HGB_LAUNCH_CHECK("tc_wgrad_reduce");
  return HGB_OK;
}
