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
//                       row-major: warp-specialised, one warp's TMA lands row slabs, seven transposer warps turn them into a ring
//                       of K-major buffers (splitting into TF32 hi / lo in fp32-accurate mode), and the two MMA warpgroups only
//                       issue wgmma on them.  The bias gradient rides along as 16 extra "ones" rows of the B operand.
#include "hgb_tc.cuh"

namespace {

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
  int slots;            // output staging buffers per consumer warpgroup (2 or 4), one [64 x 32] sub-tile each
};

// hgb_tc_linear_graph_add: a separate parameter type, so the plain layers' kernels keep their parameter block and registers
struct LinParamsGA : LinParams {
  const float* gadd;    // [ng, no] (row stride ldg), never with addend: y = a.B^T + bias + gadd[graph(row)], where graph(row) is
  const int32_t* gptr;  //   the g with gptr[g] <= row < gptr[g + 1] (graph offsets [ng + 1], rows sorted by graph)
  int ng;
  int64_t ldg;
};
template <bool GA> struct LinParamsOf { using type = LinParams; };
template <> struct LinParamsOf<true> { using type = LinParamsGA; };

constexpr int TILE_M = 64;                       // rows per tile = one wgmma M
constexpr uint32_t A_STAGE = TILE_M * 128;       // one pipeline stage = one [64 x 32 fp32] k-block (8 KB)
constexpr uint32_t SUB_BYTES = TILE_M * 128;     // one output staging buffer = one [64 x 32 fp32] TMA store box (8 KB)
constexpr int LIN_THREADS = 384;

// epilogue kinds: the activation, picked once per sub-tile so that the element loop carries no dispatch
enum { EPI_NONE, EPI_RELU, EPI_SILU, EPI_SILU_ZD, EPI_TANH, EPI_OTHER };

// the epilogue of one output: v = accumulator + bias on entry; z receives what the z output stores
template <int K, bool GA>
__device__ __forceinline__ float lin_epilogue1(const LinParams& p, float v, float& z, float a, float g) {
  z = v;
  if (K == EPI_RELU) v = isnan(v) ? v : fmaxf(v, 0.f);     // torch.relu (clamp_min): NaN propagates
  if (K == EPI_SILU) v = __fdividef(v, 1.f + __expf(-v));
  if (K == EPI_SILU_ZD) {     // z receives silu'(pre) = s + y (1 - s): the backward then needs one multiply per element
    const float s = __fdividef(1.f, 1.f + __expf(-v));
    v *= s;
    z = fmaf(v, 1.f - s, s);
  }
  if (K == EPI_TANH) v = tanhf(v);
  if (K == EPI_OTHER) v = hgb_act(v, p.act, p.act_param);
  if (GA || p.addend) v += a;
  if (p.gsrc) {
    if (p.gact == HGB_ACT_RELU_SELECT) v = hgb_relu_select(v, g);
    else v *= p.gact == HGB_ACT_DERIV ? g : hgb_act_grad(g, g, p.gact, p.act_param);   // DERIV: gsrc already holds act'(.)
  }
  return v;
}

// Element loop over one [64 x 32] sub-tile of a warpgroup (tid 0..127): 4 float4 per thread, 8 threads per row.  ys holds the
// accumulators in the TMA SWIZZLE_128B layout and receives y in place; zs receives z.  a / g: this thread's addend / gsrc values.
template <int K, bool GA>
__device__ __forceinline__ void lin_epilogue_sub(const LinParams& p, const float* sb, uint8_t* ys, uint8_t* zs, int tid, const float4* a,
                                                 const float4* g) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int idx = j * 128 + tid, r = idx >> 3, q = idx & 7;
    const uint32_t off = (uint32_t)r * 128 + ((q ^ (r & 7)) << 4);
    float4 v = *reinterpret_cast<float4*>(ys + off), z;
    v.x = lin_epilogue1<K, GA>(p, v.x + sb[4 * q], z.x, a[j].x, g[j].x);
    v.y = lin_epilogue1<K, GA>(p, v.y + sb[4 * q + 1], z.y, a[j].y, g[j].y);
    v.z = lin_epilogue1<K, GA>(p, v.z + sb[4 * q + 2], z.z, a[j].z, g[j].z);
    v.w = lin_epilogue1<K, GA>(p, v.w + sb[4 * q + 3], z.w, a[j].w, g[j].w);
    *reinterpret_cast<float4*>(ys + off) = v;
    if (zs) *reinterpret_cast<float4*>(zs + off) = z;
  }
}

// the graph of row `row` (< m): the last g with gptr[g] <= row, so empty graphs (repeated offsets) are skipped
__device__ __forceinline__ int lin_graph_of(const LinParamsGA& p, int row) {
  int lo = 0, hi = p.ng;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(p.gptr + mid) <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// this thread's addend / gsrc values of sub-tile c (columns 32 c ..) of the tile at row0, in lin_epilogue_sub's element order;
// gid: the graphs of this thread's 4 rows (gadd only)
template <bool GA>
__device__ __forceinline__ void lin_load_operands(const typename LinParamsOf<GA>::type& p, int row0, int c, int tid, const int* gid, float4* a, float4* g) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int idx = j * 128 + tid, row = row0 + (idx >> 3);
    const int64_t o = (int64_t)row * p.ldy + c * 32 + (idx & 7) * 4;
    const bool in = row < p.m;
    if (p.addend) a[j] = in ? __ldg(reinterpret_cast<const float4*>(p.addend + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (GA)
      a[j] = in ? __ldg(reinterpret_cast<const float4*>(p.gadd + (int64_t)gid[j] * p.ldg + c * 32 + (idx & 7) * 4))
                : make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.gsrc) g[j] = in ? __ldg(reinterpret_cast<const float4*>(p.gsrc + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Shared memory (bytes; B = KB * NO * 128 per weight copy, A stage = 8 KB, x2 in split mode; SMEM_MAX = 232,448):
//   [B hi | B lo (split)] [2 warpgroups x slots x 8 KB output staging] [stages x A stage | A lo (split)] [3 x stages barriers] [bias]
// The host piece rule keeps B <= 160 KB in TF32 mode and 2 x 64 KB in split mode.  Tightest TF32 case, k_red = 256 and a 160-column
// piece: 1 KB alignment + 160 KB B + 32 KB staging (2 slots) + 0.7 KB bias / barriers leaves 33.7 KB = 4 A stages (2 per ring).
// Tightest split case, 64 KB of weights per copy: 1 KB + 128 KB B + 32 KB staging leaves 66 KB = 4 A stages of 16 KB.  Four slots
// per warpgroup (64 KB) are used when at least 4 stages still fit next to them: B <= 128 KB in TF32 mode, <= 48 KB per copy in split
// mode (every C2 layer has B <= 48 KB).
// GA: the per-graph addend (gadd) of hgb_tc_linear_graph_add; its own instantiations, so the plain layers keep their registers
template <int NC, bool SPLIT, bool GA>   // NO = 32 * NC output columns; SPLIT: the fp32-accurate mode
__global__ void __launch_bounds__(LIN_THREADS, 1) tc_linear_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                   const __grid_constant__ CUtensorMap tmap_y,
                                                                   const __grid_constant__ CUtensorMap tmap_z,
                                                                   const typename LinParamsOf<GA>::type p) {
  constexpr int NO = NC * 32;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int KB = p.kr >> 5;
  const uint32_t b_pad = ((uint32_t)KB * NO * 128 + 1023) & ~1023u;
  uint8_t* sB = smem;
  uint8_t* sBlo = sB + b_pad;                                 // split mode only
  uint8_t* sOut = sB + (SPLIT ? 2 : 1) * (size_t)b_pad;       // [2][slots] staging buffers, 1024-byte aligned (TMA swizzle)
  uint8_t* sA = sOut + (size_t)2 * p.slots * SUB_BYTES;
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
    const int tid = threadIdx.x & 127;  // thread within the warpgroup
    const uint32_t sA_addr = smem_u32(sA), sAlo_addr = smem_u32(sAlo), sB_addr = smem_u32(sB), sBlo_addr = smem_u32(sBlo);
    // output staging: a sub-tile takes one buffer (y) or two (y, z); `ahead` = how many sub-tiles' TMA stores may still be reading
    // their buffers when the next sub-tile is written
    uint8_t* sOwn = sOut + (size_t)cw * p.slots * SUB_BYTES;
    const int per_sub = p.z ? 2 : 1;
    const int ahead = p.slots / per_sub - 1;            // 0, 1 or 3
    const int kind = p.act == HGB_ACT_NONE ? EPI_NONE
                     : p.act == HGB_ACT_RELU ? EPI_RELU
                     : p.act == HGB_ACT_SILU ? (p.z && p.z_deriv ? EPI_SILU_ZD : EPI_SILU)
                     : p.act == HGB_ACT_TANH ? EPI_TANH
                                             : EPI_OTHER;
    const bool operands = GA || p.addend || p.gsrc;
    float acc[NC * 16];
    uint32_t sub = 0;                   // sub-tiles stored so far by this warpgroup
    int li = cw;
    for (int t = blockIdx.x + cw * gridDim.x; t < ntiles; t += 2 * gridDim.x, li += 2) {
      const int row0 = t * TILE_M;
      int gid[4] = {0, 0, 0, 0};
      if constexpr (GA) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int row = row0 + ((j * 128 + tid) >> 3);
          if (row < p.m) gid[j] = lin_graph_of(p, row);
        }
      }
      float4 opa[4], opg[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) opa[j] = opg[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      // the first sub-tile's addend / gsrc are in flight during the MMAs (at NC = 8 these 32 registers would spill: load after them)
      constexpr bool early = NC < 8;
      if (early && operands) lin_load_operands<GA>(p, row0, 0, tid, gid, opa, opg);
#pragma unroll
      for (int j = 0; j < NC * 16; ++j) acc[j] = 0.f;
      const uint32_t n0 = (uint32_t)(li >> 1) * KB;             // first item of this tile within ring cw
      for (int kb = 0; kb < KB; ++kb) {
        const uint32_t n = n0 + kb;
        const int s = cw * SR + n % SR;
        mbar_wait(SPLIT ? full2 + s : full + s, (n / SR) & 1);
        fence_regs<NC * 16>(acc);
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const uint64_t ad = make_desc(sA_addr + s * A_STAGE + k4 * 32);
          const uint32_t boff = (uint32_t)kb * NO * 128 + k4 * 32;  // every output column: 8-row groups of B are 1024 B apart
          const uint64_t bd = make_desc(sB_addr + boff);
          if (SPLIT) {          // small terms first: lo*hi + hi*lo + hi*hi
            wgmma_tf32<NC>(acc, make_desc(sAlo_addr + s * A_STAGE + k4 * 32), bd);
            wgmma_tf32<NC>(acc, ad, make_desc(sBlo_addr + boff));
          }
          wgmma_tf32<NC>(acc, ad, bd);
        }
        wgmma_commit();
        fence_regs<NC * 16>(acc);
        if (kb > 0) {                   // the MMAs of the previous k-block have read their stage: release it
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(empty + cw * SR + (n - 1) % SR);
        }
      }
      wgmma_wait<0>();
      fence_regs<NC * 16>(acc);
      if (lane == 0) mbar_arrive(empty + cw * SR + (n0 + KB - 1) % SR);
      if (!early && operands) lin_load_operands<GA>(p, row0, 0, tid, gid, opa, opg);
      // ===== epilogue, one [64 x 32] sub-tile at a time: accumulators -> swizzled staging buffer -> element loop in place -> TMA
      // store (rows >= m are clipped by the tensor map) =====
#pragma unroll 1
      for (int c = 0; c < NC; ++c, ++sub) {
        uint8_t* ys = sOwn + (size_t)((sub % (p.slots / per_sub)) * per_sub) * SUB_BYTES;
        uint8_t* zs = p.z ? ys + SUB_BYTES : nullptr;
        if (tid == 0) {
          if (ahead == 0) bulk_wait_read<0>(); else if (ahead == 1) bulk_wait_read<1>(); else bulk_wait_read<3>();
        }
        named_bar_sync(2 + cw, 128);    // the buffers are free (and no thread still reads them)
#pragma unroll
        for (int cc = 0; cc < NC; ++cc)
          if (cc == c) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = wq * 16 + (lane >> 2) + 8 * h, col = i * 8 + 2 * (lane & 3);
                *reinterpret_cast<float2*>(ys + kmajor_sw128_off(r, col, TILE_M)) =
                    make_float2(acc[16 * cc + 4 * i + 2 * h], acc[16 * cc + 4 * i + 2 * h + 1]);
              }
          }
        named_bar_sync(2 + cw, 128);
        const float* sb = sbias + c * 32;
        switch (kind) {
          case EPI_NONE: lin_epilogue_sub<EPI_NONE, GA>(p, sb, ys, zs, tid, opa, opg); break;
          case EPI_RELU: lin_epilogue_sub<EPI_RELU, GA>(p, sb, ys, zs, tid, opa, opg); break;
          case EPI_SILU: lin_epilogue_sub<EPI_SILU, GA>(p, sb, ys, zs, tid, opa, opg); break;
          case EPI_SILU_ZD: lin_epilogue_sub<EPI_SILU_ZD, GA>(p, sb, ys, zs, tid, opa, opg); break;
          case EPI_TANH: lin_epilogue_sub<EPI_TANH, GA>(p, sb, ys, zs, tid, opa, opg); break;
          default: lin_epilogue_sub<EPI_OTHER, GA>(p, sb, ys, zs, tid, opa, opg);
        }
        if (operands && c + 1 < NC) lin_load_operands<GA>(p, row0, c + 1, tid, gid, opa, opg);
        fence_proxy_async();            // the staged results are visible to the TMA
        named_bar_sync(2 + cw, 128);
        if (tid == 0) {
          tma_store_2d(&tmap_y, ys, c * 32, row0);
          if (zs) tma_store_2d(&tmap_z, zs, c * 32, row0);
          bulk_commit();
        }
      }
    }
    if (tid == 0) bulk_wait_all();      // the stores have completed before the CTA's shared memory goes away
  }
}

// ------------------------------------------------------------------------------------------------
// weight gradient: dW[NO, KO] (+ db[NO]) = sum_m dZ[m, NO]^T X[m, KO]
// ------------------------------------------------------------------------------------------------
struct WgParams {
  int m, no, ko;
  int chunks_per_cta;   // number of 32-row chunks each CTA reduces
  int stages;           // TMA ring of raw row slabs
  int tbufs;            // ring of K-major (transposed) operand buffers between the transposer warps and the MMA warpgroups
  int split;            // 1: fp32-accurate mode -- both operands are split into TF32 hi / lo twins and every k-step runs lo*hi + hi*lo + hi*hi
  int flush;            // > 0: the register accumulators are added into the partial every `flush` chunks and restarted, so each chain
                        //   of tensor-core additions stays short (the fp32-accurate mode)
  float* part;          // [gridDim.x, no, ko + 1]
};

constexpr int WG_ROWS = 32;                      // rows of dZ / X per chunk = one 128-byte K-major row of the transposed operands
constexpr int WG_NA = 128;                       // rows of dW per CTA (two MMA warpgroups x 64)
constexpr int WG_TRANSPOSERS = 7;                // with three, the transposition bounded the n_out = 128 and 192 calls
constexpr int WG_THREADS = 256 + 32 * (1 + WG_TRANSPOSERS);   // 2 MMA warpgroups + one TMA warp and WG_TRANSPOSERS transposer warps
constexpr int WG_AUX_REGS = 40, WG_MMA_REGS = 216;   // 256 x 40 + 256 x 216 = 64 K registers

// Warp-specialised pipeline, one chunk (32 rows of dZ and X) per step:
//   warp 8           TMA: raw row slabs into a ring of `stages` buffers (full / empty mbarriers)
//   warps 9..15      transpose each raw stage into the next K-major operand buffer of a ring of `tbufs` (tfull / tempty), splitting
//                    into TF32 hi / lo in fp32-accurate mode, and release the raw stage
//   warpgroups 0, 1  wait on tfull, issue the chunk's MMAs, and release the buffer once wgmma_wait shows they have read it
// The arithmetic is fixed by the chunk partition and the MMA sequence of each chunk, not by how the data gets there.
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
  const int n_mma_wg = (nrows + 63) >> 6;                 // warpgroups with dW rows in this CTA
  const uint32_t raw_bytes = (uint32_t)(nsl + Q) * SLAB;
  const uint32_t tb_bytes = HI_BYTES * (SPLIT ? 2 : 1);
  const int S = p.stages, T = p.tbufs;
  uint8_t* tbuf = smem;                                   // T x [A hi (128 rows) | B hi (NB rows) | A lo | B lo]
  uint8_t* raw = smem + (size_t)T * tb_bytes;             // S x [nsl dZ slabs | Q X slabs], row-major as loaded
  uint64_t* full = reinterpret_cast<uint64_t*>(raw + (size_t)S * raw_bytes);
  uint64_t* empty = full + S;
  uint64_t* tfull = empty + S;
  uint64_t* tempty = tfull + T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int total_chunks = (p.m + WG_ROWS - 1) / WG_ROWS;
  const int c_beg = blockIdx.x * p.chunks_per_cta;
  const int nchunks = max(0, min(total_chunks, c_beg + p.chunks_per_cta) - c_beg);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, WG_TRANSPOSERS); }
    for (int t = 0; t < T; ++t) { mbar_init(tfull + t, WG_TRANSPOSERS); mbar_init(tempty + t, 4 * n_mma_wg); }
    fence_barrier_init();
  }
  // rows of the operand buffers that no chunk writes, set once: A rows nrows..127 zero, B rows KO.. the ones rows (lo twins zero)
  {
    const int zrows = WG_NA - nrows, frows = zrows + 16;
    const int words = T * (SPLIT ? 2 : 1) * frows * 32;
    for (int i = threadIdx.x; i < words; i += blockDim.x) {
      const int rr = (i >> 5) % frows, half = (i >> 5) / frows;   // half: buffer * (SPLIT ? 2 : 1) + (lo twin)
      const int row = rr < zrows ? nrows + rr : WG_NA + KO + (rr - zrows);
      const bool lo = SPLIT && (half & 1);
      const int t = SPLIT ? half >> 1 : half;
      reinterpret_cast<float*>(tbuf + (size_t)t * tb_bytes + (lo ? HI_BYTES : 0) + (size_t)row * 128)[i & 31] =
          (!lo && rr >= zrows) ? 1.f : 0.f;
    }
  }
  fence_proxy_async();
  __syncthreads();

  if (warp >= 8) {
    regs_dec<WG_AUX_REGS>();
    if (warp == 8) {
      // ===== TMA producer: this CTA's dZ columns n0.. and all of X, 32 rows per chunk =====
      if (lane == 0) {
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
    // ===== transposers: operand row r (A: dZ column n0 + r; B: X column r - nrows) gets the 32 values of this chunk as one K-major
    // 128-byte row.  A unit is 32 consecutive rows (one per lane) x 4 consecutive m: four conflict-free column reads per lane and
    // one swizzled 16-byte store.  =====
    const int tw = warp - 9;
    const int units = (nsl + Q) * 8;
    for (int c = 0; c < nchunks; ++c) {
      const int s = c % S, t = c % T;
      uint8_t* tb = tbuf + (size_t)t * tb_bytes;
      const uint8_t* st = raw + (size_t)s * raw_bytes;
      mbar_wait(full + s, (c / S) & 1);
      mbar_wait(tempty + t, ((c / T) & 1) ^ 1);
#pragma unroll 4
      for (int u = tw; u < units; u += WG_TRANSPOSERS) {
        const int slab = u >> 3, m4 = u & 7;
        const float* src = reinterpret_cast<const float*>(st + (size_t)slab * SLAB) + lane + m4 * 4 * 32;
        const float4 v = make_float4(src[0], src[32], src[64], src[96]);
        const int orow = slab < nsl ? slab * 32 + lane : WG_NA + (slab - nsl) * 32 + lane;
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
      if (lane == 0) {
        mbar_arrive(empty + s);                           // the raw slabs are no longer needed
        mbar_arrive(tfull + t);                           // this warp's share of the K-major chunk is written
      }
    }
    return;
  }

  // ===== MMA warpgroups (threads 0..255): warpgroup wg owns dW rows n0 + 64 wg .. +63 =====
  regs_inc<WG_MMA_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  if (wg >= n_mma_wg) return;
  float acc[Q][16], accb[8];
  float* part = p.part + (size_t)blockIdx.x * p.no * (p.ko + 1);

  auto store = [&](bool first) {   // partial (first: =, then +=) accumulators
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
  };

  // fold groups: the accumulators start at zero, take `flush` chunks (all of them when flush = 0) and are added into the partial.
  // They are zeroed only here, with no MMA in flight: ptxas serialises every wgmma of a loop in which a non-wgmma instruction may write
  // an accumulator while a group is pending.  A CTA without chunks writes zeros.
  int c = 0;
  for (bool first = true;; first = false) {
#pragma unroll
    for (int q = 0; q < Q; ++q)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[q][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) accb[j] = 0.f;
    const int c_end = p.flush ? min(nchunks, c + p.flush) : nchunks;
    for (; c < c_end; ++c) {
      const int t = c % T;
      const uint32_t ta = smem_u32(tbuf + (size_t)t * tb_bytes);
      mbar_wait(tfull + t, (c / T) & 1);
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
      // release the buffer whose MMAs are known to be complete: the previous chunk's (one group may stay in flight), or with a
      // single buffer this chunk's
      if (T >= 2) {
        wgmma_wait<1>();
        if (c > 0 && lane == 0) mbar_arrive(tempty + (c - 1) % T);
      } else {
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(tempty + t);
      }
    }
    wgmma_wait<0>();
    fence_regs<Q * 16>(&acc[0][0]);
    fence_regs<8>(accb);
    store(first);
    if (c >= nchunks) break;
  }
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
bool shape_ok(int kr, int no) { return kr >= 32 && kr <= 256 && kr % 32 == 0 && no >= 32 && no <= 256 && no % 32 == 0; }

template <int NC, bool SPLIT, bool GA>
void launch_linear_t(int grid, size_t smem, cudaStream_t st, const CUtensorMap* tm, const typename LinParamsOf<GA>::type& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(tc_linear_kernel<NC, SPLIT, GA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
    attr_set = true;
  }
  tc_linear_kernel<NC, SPLIT, GA><<<grid, LIN_THREADS, smem, st>>>(tm[0], tm[1], tm[2], p);
}
template <int NC>
void launch_linear(int grid, size_t smem, cudaStream_t st, const CUtensorMap* tm, const LinParamsGA& p) {  // tm: a, y, z
  if (p.gadd) {
    if (p.split) launch_linear_t<NC, true, true>(grid, smem, st, tm, p); else launch_linear_t<NC, false, true>(grid, smem, st, tm, p);
  } else {
    const LinParams& q = p;
    if (q.split) launch_linear_t<NC, true, false>(grid, smem, st, tm, q); else launch_linear_t<NC, false, false>(grid, smem, st, tm, q);
  }
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
                           const float* gsrc, int32_t gact, int64_t ldy, int32_t exact, const float* gadd, int64_t ldg,
                           const int32_t* gptr, int32_t ng, hgb_stream_t stream) {
  HGB_REQUIRE(a && w && y && m >= 128 && shape_ok(k_red, n_out), "tc_linear: unsupported shape m=%d n=%d k=%d", m, n_out, k_red);
  HGB_REQUIRE(lda % 4 == 0 && ldy % 4 == 0 && ((uintptr_t)a % 16 == 0) && ((uintptr_t)y % 16 == 0) && (!z || (uintptr_t)z % 16 == 0) &&
                  (!addend || (uintptr_t)addend % 16 == 0) && (!gsrc || (uintptr_t)gsrc % 16 == 0) &&
                  (!gadd || ((uintptr_t)gadd % 16 == 0 && ldg % 4 == 0)),
              "tc_linear: operands must be 16-byte aligned with a row stride that is a multiple of 4");
  CUtensorMap tm[3];                               // A loads; y and z stores: [64 x 32] boxes, rows >= m clipped
  int rc = make_tmap(&tm[0], a, m, k_red, lda, TILE_M, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  LinParamsGA p;
  p.m = m; p.kr = k_red; p.no = n_out; p.w = w; p.ldw = ldw; p.trans_b = trans_b; p.bias = bias; p.act = act; p.act_param = act_param;
  p.y = y; p.z = z; p.addend = addend; p.ldy = ldy; p.gsrc = gsrc; p.gact = gact; p.z_deriv = (!gsrc && gact == HGB_ACT_DERIV) ? 1 : 0;
  p.gadd = gadd; p.gptr = gptr; p.ng = ng; p.ldg = ldg;
  rc = make_tmap(&tm[1], y, m, n_out, ldy, TILE_M, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_tmap(&tm[2], z ? z : y, m, n_out, ldy, TILE_M, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  const int KB = k_red / 32;
  const int dup = exact ? 2 : 1;                   // split mode keeps a hi and a lo copy of the weights and of every A stage
  const size_t b_bytes = ((size_t)KB * n_out * 128 + 1023) & ~(size_t)1023;
  int stages = 0, slots = 0;
  size_t fixed = 0;
  for (slots = 4; slots >= 2; slots -= 2) {        // four staging buffers per warpgroup where 4 A stages still fit, else two
    fixed = 1024 + dup * b_bytes + (size_t)2 * slots * SUB_BYTES + (size_t)n_out * 4 + 64;
    stages = fixed < SMEM_MAX ? (int)((SMEM_MAX - fixed) / (dup * A_STAGE + 3 * 8)) : 0;
    if (stages > 8) stages = 8;
    stages &= ~1;                                  // two equal rings, one per consumer warpgroup
    if (stages >= 4) break;
  }
  HGB_REQUIRE(stages >= 4, "tc_linear: weight operand does not fit shared memory (n=%d k=%d)", n_out, k_red);
  p.stages = stages;
  p.slots = slots;
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
// gadd (with gptr / ng / ldg) replaces addend for the first reduction piece: the per-graph row of hgb_tc_linear_graph_add
static int tc_linear_pieces(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t trans_b, const float* bias, int32_t m,
                            int32_t n_out, int32_t k_red, int32_t act, float act_param, float* y, float* z, const float* addend,
                            const float* gsrc, int32_t gact, int32_t exact, const float* gadd, int64_t ldg, const int32_t* gptr, int32_t ng,
                            hgb_stream_t stream) {
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
                               z ? z + c0 : nullptr, add, gsrc ? gsrc + c0 : nullptr, gact, n_out, exact,
                               (gadd && k0 == 0) ? gadd + c0 : nullptr, ldg, gptr, ng, stream);
      if (rc) return rc;
    }
  }
  return HGB_OK;
}

extern "C" int hgb_tc_linear(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t trans_b, const float* bias, int32_t m,
                             int32_t n_out, int32_t k_red, int32_t act, float act_param, float* y, float* z, const float* addend,
                             const float* gsrc, int32_t gact, int32_t exact, hgb_stream_t stream) {
  return tc_linear_pieces(a, lda, w, ldw, trans_b, bias, m, n_out, k_red, act, act_param, y, z, addend, gsrc, gact, exact, nullptr, 0,
                          nullptr, 0, stream);
}

// y[m, no] = a[m, kr] . w^T + gadd[graph(row)]: the concat_node projector Linear(H + G, H) on [h | graph_attr[batch]] with the
// graph-attribute columns folded into the per-graph row gadd = graph_attr . W_g^T + b [ng, no] (row stride ldg)
extern "C" int hgb_tc_linear_graph_add(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t m, int32_t n_out, int32_t k_red,
                                       const float* gadd, int64_t ldg, const int32_t* gptr, int32_t ng, float* y, int32_t exact,
                                       hgb_stream_t stream) {
  HGB_REQUIRE(a && w && y && gadd && gptr && ng >= 1 && hgb_tc_linear_supported(m, n_out, k_red),
              "tc_linear_graph_add: unsupported shape m=%d n=%d k=%d graphs=%d", m, n_out, k_red, ng);
  return tc_linear_pieces(a, lda, w, ldw, 0, nullptr, m, n_out, k_red, HGB_ACT_NONE, 0.f, y, nullptr, nullptr, nullptr, 0, exact, gadd, ldg,
                          gptr, ng, stream);
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
  // shared memory: up to three K-major buffers (each transposed chunk then waits on no MMA still reading the buffer it reuses), as
  // long as two raw stages fit beside them; every byte left over deepens the TMA ring.  Each buffer and stage has two mbarriers.
  const size_t budget = SMEM_MAX - 1024;
  int tbufs = 3;
  while (tbufs > 1 && (size_t)tbufs * (tb_bytes + 16) + 2 * (raw_bytes + 16) > budget) --tbufs;
  const size_t left = budget > (size_t)tbufs * (tb_bytes + 16) ? budget - (size_t)tbufs * (tb_bytes + 16) : 0;
  const int stages = (int)(left / (raw_bytes + 16));
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
  const size_t smem = 1024 + tbufs * (tb_bytes + 16) + stages * (raw_bytes + 16);
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
