// libhgb.so -- neighbour aggregation gathered straight into a degree-grouped wgmma Linear: torch_geometric's SAGEConv
// (aggr "mean", root_weight, hydragnn/models/SAGEStack.py) and MFConv (aggr "add", one weight pair per clamped in-degree,
// hydragnn/models/MFCStack.py).  sm_90a only.
//
//   forward     out[i] = [h_i | x_i] . [W_l,g | W_r,g]^T + b_g      h_i = sum (SAGE: mean) of x_j over the in-edges j -> i,
//                                                                   g = the row's weight group (MFC: min(in-degree, max_degree))
//   data bwd 1  [g_h | g_xr][i] = g_out[i] . [W_l,g | W_r,g]        (g_h divided by max(deg, 1) in mean mode)
//
// One CTA per 64-row tile of a row order in which the weight groups are contiguous (order [n], grp_ptr [groups + 1]); the tile
// table [tiles][2] = (group, first row) comes from hgb_nbr_tiles, so no tile scans the groups and the host reads no group size.
// All eight warps build the A tile [64 x ka] in shared memory, already in the K-major SWIZZLE_128B layout wgmma reads: in the
// forward the neighbour rows x[src] of each target summed in the order of its by-target CSR segment (ascending edge id), then
// the node's own row; in the data backward the rows of g_out.  Every padding column is zero.  The weight operand streams in
// 32-deep k-blocks, double-buffered when shared memory allows it: warpgroup 1 stages block kb + 1 while warpgroup 0 runs the
// wgmma of block kb (one full-width instruction per k-step, as hgb_tc_linear).  The epilogue scatters each row to its node.
// No atomics: repeated runs are bit-identical.
#include "hgb_tc.cuh"

namespace {

constexpr int NB_ROWS = 64;                    // rows per tile = one wgmma M
constexpr int NB_THREADS = 256;
constexpr uint32_t NB_SLAB = NB_ROWS * 128;   // one 32-column block of the A tile

__device__ __forceinline__ float nb_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

struct NbrParams {
  int gather;               // 1: forward (neighbour sum + root row), 0: rows of x (the data backward)
  int kin, kpad, ka;        // forward: feature width, its 32-padded width, ka = 2 kpad; backward: n_out, -, ka = round32(n_out)
  const float* x;           // [n, kin]
  const int32_t* rowptr;    // by-target CSR offsets [n + 1]: the segments (forward) and the in-degrees (mean scale)
  const int32_t* src;       // source node of every by-target CSR slot (forward)
  int mean;
  const int32_t* order;     // [n] row -> node (NULL: identity)
  const int32_t* tiles;     // [tiles][2] = (group, first row); group < 0: surplus tile
  const int32_t* grp_ptr;   // [groups + 1]
  const float* w;           // [groups, npad, ka] K-major weight operand, zero padded
  int npad;
  const float* bias;        // [groups, n0] or NULL
  float* y0;                // padded output columns [0, csplit) -> y0 [n, n0]
  int n0, csplit;
  float* y1;                // columns [csplit, csplit + n1) -> y1 [n, n1] (NULL: none)
  int n1;
  int scale0;               // divide the y0 columns by max(deg, 1) (the mean's backward)
  float* hx;                // optional [n, ka] copy of the A tile rows, in row order (the weight gradient's operand)
  int split;                // 3xTF32
  int nbuf;                 // weight k-block buffers (1 or 2)
};

template <bool SPLIT>
__device__ __forceinline__ void nb_put(uint8_t* hi, uint8_t* lo, uint32_t off, float v) {
  if (SPLIT) {
    const float h = nb_tf32(v);
    *reinterpret_cast<float*>(hi + off) = h;
    *reinterpret_cast<float*>(lo + off) = nb_tf32(v - h);
  } else {
    *reinterpret_cast<float*>(hi + off) = v;
  }
}

// weight k-block kb of group g -> buffer (hi, lo): rows = output columns, 32 reduction columns
template <bool SPLIT>
__device__ __forceinline__ void nb_stage_b(const NbrParams& p, int g, int kb, uint8_t* hi, uint8_t* lo, int t0, int nt) {
  const float* wg = p.w + ((int64_t)g * p.npad) * p.ka + kb * 32;
  for (int i = t0; i < p.npad * 32; i += nt) {
    const int r = i >> 5, c = i & 31;
    nb_put<SPLIT>(hi, lo, kmajor_sw128_off(r, c, p.npad), __ldg(wg + (int64_t)r * p.ka + c));
  }
}

template <int NC, bool SPLIT>
__global__ void __launch_bounds__(NB_THREADS) nbr_linear_kernel(const NbrParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ int s_node[NB_ROWS];
  __shared__ float s_inv[NB_ROWS];
  const int g = p.tiles[2 * blockIdx.x], row0 = p.tiles[2 * blockIdx.x + 1];
  if (g < 0) return;                                           // surplus tile (uniform across the block)
  const int rows = min(NB_ROWS, p.grp_ptr[g + 1] - row0);
  const int KB = p.ka >> 5;
  const uint32_t a_bytes = (uint32_t)KB * NB_SLAB, b_bytes = (uint32_t)p.npad * 128;
  uint8_t* sA = smem;
  uint8_t* sAlo = sA + a_bytes;                                // split mode only
  uint8_t* sB = sA + (SPLIT ? 2 : 1) * a_bytes;                // nbuf x [hi | lo (split)]
  const uint32_t b_stride = (SPLIT ? 2 : 1) * b_bytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x < NB_ROWS) {
    const int r = threadIdx.x;
    int node = -1;
    float inv = 1.f;
    if (r < rows) {
      node = p.order ? p.order[row0 + r] : row0 + r;
      inv = 1.f / (float)max(p.rowptr[node + 1] - p.rowptr[node], 1);
    }
    s_node[r] = node;
    s_inv[r] = inv;
  }
  // the first weight block loads while the A tile is gathered
  nb_stage_b<SPLIT>(p, g, 0, sB, sB + b_bytes, threadIdx.x, NB_THREADS);
  __syncthreads();

  // ===== A tile: warp w builds rows w, w + 8, ...; lane l owns columns l, l + 32, ... =====
  for (int r = warp; r < NB_ROWS; r += NB_THREADS / 32) {
    const int node = s_node[r];
    int e0 = 0, e1 = 0;
    if (node >= 0 && p.gather) { e0 = p.rowptr[node]; e1 = p.rowptr[node + 1]; }
    for (int cb = 0; cb < KB; ++cb) {
      const int c = cb * 32 + lane;
      float v = 0.f;
      if (node >= 0) {
        if (!p.gather) {
          if (c < p.kin) v = __ldg(p.x + (int64_t)node * p.kin + c);
        } else if (c < p.kpad) {
          if (c < p.kin) {
            // neighbour sum in CSR order: four rows in flight, added one after the other
            int e = e0;
            for (; e + 3 < e1; e += 4) {
              const int s0 = __ldg(p.src + e), s1 = __ldg(p.src + e + 1), s2 = __ldg(p.src + e + 2), s3 = __ldg(p.src + e + 3);
              const float v0 = __ldg(p.x + (int64_t)s0 * p.kin + c), v1 = __ldg(p.x + (int64_t)s1 * p.kin + c);
              const float v2 = __ldg(p.x + (int64_t)s2 * p.kin + c), v3 = __ldg(p.x + (int64_t)s3 * p.kin + c);
              v += v0; v += v1; v += v2; v += v3;
            }
            for (; e < e1; ++e) v += __ldg(p.x + (int64_t)__ldg(p.src + e) * p.kin + c);
            if (p.mean) v /= (float)max(e1 - e0, 1);
          }
        } else if (c - p.kpad < p.kin) {
          v = __ldg(p.x + (int64_t)node * p.kin + (c - p.kpad));
        }
        if (p.hx) p.hx[(int64_t)(row0 + r) * p.ka + c] = v;
      }
      nb_put<SPLIT>(sA, sAlo, kmajor_sw128_off(r, c, NB_ROWS), v);
    }
  }
  fence_proxy_async();
  __syncthreads();

  // ===== k loop: warpgroup 0 multiplies, warpgroup 1 stages the next weight block (or everyone does, single-buffered) =====
  float acc[NC * 16];
#pragma unroll
  for (int j = 0; j < NC * 16; ++j) acc[j] = 0.f;
  const int wg = warp >> 2;
  for (int kb = 0; kb < KB; ++kb) {
    uint8_t* bcur = sB + (size_t)(p.nbuf == 2 ? (kb & 1) : 0) * b_stride;
    if (wg == 0) {
      const uint32_t a_hi = smem_u32(sA) + kb * NB_SLAB, a_lo = smem_u32(sAlo) + kb * NB_SLAB;
      const uint32_t b_hi = smem_u32(bcur), b_lo = b_hi + b_bytes;
      fence_regs<NC * 16>(acc);
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t ad = make_desc(a_hi + k4 * 32), bd = make_desc(b_hi + k4 * 32);
        if (SPLIT) {                                           // small terms first: lo*hi + hi*lo + hi*hi
          wgmma_tf32<NC>(acc, make_desc(a_lo + k4 * 32), bd);
          wgmma_tf32<NC>(acc, ad, make_desc(b_lo + k4 * 32));
        }
        wgmma_tf32<NC>(acc, ad, bd);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<NC * 16>(acc);
    } else if (p.nbuf == 2 && kb + 1 < KB) {
      uint8_t* bn = sB + (size_t)((kb + 1) & 1) * b_stride;
      nb_stage_b<SPLIT>(p, g, kb + 1, bn, bn + b_bytes, threadIdx.x - 128, 128);
      fence_proxy_async();
    }
    __syncthreads();
    if (p.nbuf == 1 && kb + 1 < KB) {
      nb_stage_b<SPLIT>(p, g, kb + 1, sB, sB + b_bytes, threadIdx.x, NB_THREADS);
      fence_proxy_async();
      __syncthreads();
    }
  }

  // ===== epilogue (warpgroup 0): d[16 cc + 4 i + 2 h + e] = D(16 wq + lane/4 + 8 h, 32 cc + 8 i + 2 (lane % 4) + e) =====
  if (wg != 0) return;
  const int wq = warp & 3;
  const float* bias = p.bias ? p.bias + (int64_t)g * p.n0 : nullptr;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wq * 16 + (lane >> 2) + 8 * h;
    const int node = s_node[r];
    if (node < 0) continue;
    const float sc = p.scale0 ? s_inv[r] : 1.f;
#pragma unroll
    for (int cc = 0; cc < NC; ++cc)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = cc * 32 + i * 8 + 2 * (lane & 3) + e;
          const float v = acc[16 * cc + 4 * i + 2 * h + e];
          if (c < p.csplit) {
            if (c < p.n0) p.y0[(int64_t)node * p.n0 + c] = p.scale0 ? v * sc : (bias ? v + __ldg(bias + c) : v);
          } else if (p.y1 && c - p.csplit < p.n1) {
            p.y1[(int64_t)node * p.n1 + (c - p.csplit)] = v;
          }
        }
  }
}

// tile -> (group, first row) for rows grouped by grp_ptr; entries past the last tile get group -1
__global__ void nbr_tiles_kernel(const int32_t* __restrict__ grp_ptr, int groups, int ntiles, int32_t* __restrict__ tiles) {
  __shared__ int start[129];                 // first tile of every group, start[groups] = tiles in use
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int q = 0; q < groups; ++q) {
      start[q] = acc;
      acc += (grp_ptr[q + 1] - grp_ptr[q] + NB_ROWS - 1) / NB_ROWS;
    }
    start[groups] = acc;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < ntiles; t += blockDim.x) {
    int lo = 0, hi = groups;                 // the group q with start[q] <= t < start[q + 1]: binary search over the starts
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (start[mid] <= t) lo = mid; else hi = mid;
    }
    const bool used = t < start[groups];
    tiles[2 * t] = used ? lo : -1;
    tiles[2 * t + 1] = used ? grp_ptr[lo] + (t - start[lo]) * NB_ROWS : 0;
  }
}

size_t nb_smem(int ka, int npad, int split, int nbuf) {
  return 1024 + (size_t)(split ? 2 : 1) * ((size_t)ka * NB_ROWS * 4 + (size_t)nbuf * npad * 128);
}

template <int NC, bool SPLIT>
void nb_launch_t(int grid, size_t smem, cudaStream_t st, const NbrParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    // the static row tables (512 B) count against the same per-block limit
    cudaFuncSetAttribute(nbr_linear_kernel<NC, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX - 1024);
    attr_set = true;
  }
  nbr_linear_kernel<NC, SPLIT><<<grid, NB_THREADS, smem, st>>>(p);
}
template <int NC>
void nb_launch_nc(int grid, size_t smem, cudaStream_t st, const NbrParams& p) {
  if (p.split) nb_launch_t<NC, true>(grid, smem, st, p); else nb_launch_t<NC, false>(grid, smem, st, p);
}

int nb_run(NbrParams& p, int n, int groups, hgb_stream_t stream) {
  p.nbuf = nb_smem(p.ka, p.npad, p.split, 2) + 1024 <= SMEM_MAX ? 2 : 1;   // 1 KB for the static tables
  const size_t smem = nb_smem(p.ka, p.npad, p.split, p.nbuf);
  const int grid = (n + NB_ROWS - 1) / NB_ROWS + groups;   // worst case; surplus tiles exit
  cudaStream_t st = (cudaStream_t)stream;
  switch (p.npad / 32) {
    case 1: nb_launch_nc<1>(grid, smem, st, p); break;
    case 2: nb_launch_nc<2>(grid, smem, st, p); break;
    case 3: nb_launch_nc<3>(grid, smem, st, p); break;
    case 4: nb_launch_nc<4>(grid, smem, st, p); break;
    case 5: nb_launch_nc<5>(grid, smem, st, p); break;
    case 6: nb_launch_nc<6>(grid, smem, st, p); break;
    case 7: nb_launch_nc<7>(grid, smem, st, p); break;
    default: nb_launch_nc<8>(grid, smem, st, p); break;
  }
  HGB_LAUNCH_CHECK("nbr_linear");
  return HGB_OK;
}

int r32(int v) { return (v + 31) & ~31; }

}  // namespace

extern "C" int hgb_nbr_linear_supported(int32_t k, int32_t n_out, int32_t groups) {
  return (k >= 1 && k <= 128 && n_out >= 1 && n_out <= 256 && groups >= 1 && groups <= 128) ? 1 : 0;
}

extern "C" int hgb_nbr_tiles(const int32_t* grp_ptr, int32_t groups, int32_t n, int32_t* tiles, hgb_stream_t stream) {
  HGB_REQUIRE(grp_ptr && tiles && groups >= 1 && groups <= 128 && n >= 0, "nbr_tiles: bad arguments");
  const int ntiles = (n + NB_ROWS - 1) / NB_ROWS + groups;
  nbr_tiles_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(grp_ptr, groups, ntiles, tiles);
  HGB_LAUNCH_CHECK("nbr_tiles");
  return HGB_OK;
}

extern "C" int hgb_nbr_linear_fwd(const float* x, int32_t n, int32_t k, const int32_t* rowptr, const int32_t* src, int64_t e,
                                  int32_t mean, const int32_t* order, const int32_t* grp_ptr, const int32_t* tiles, int32_t groups,
                                  const float* w, const float* bias, int32_t n_out, float* out, float* hx, int32_t exact,
                                  hgb_stream_t stream) {
  HGB_REQUIRE(hgb_nbr_linear_supported(k, n_out, groups), "nbr_linear_fwd: unsupported shape k=%d n_out=%d groups=%d", k, n_out, groups);
  HGB_REQUIRE(n >= 0 && e >= 0 && e <= INT32_MAX, "nbr_linear_fwd: bad sizes n=%d e=%lld", n, (long long)e);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(x && rowptr && (src || e == 0) && grp_ptr && tiles && w && out, "nbr_linear_fwd: missing operand");
  NbrParams p = {};
  p.gather = 1; p.kin = k; p.kpad = r32(k); p.ka = 2 * p.kpad; p.x = x; p.rowptr = rowptr; p.src = src; p.mean = mean ? 1 : 0;
  p.order = order; p.tiles = tiles; p.grp_ptr = grp_ptr; p.w = w; p.npad = r32(n_out); p.bias = bias;
  p.y0 = out; p.n0 = n_out; p.csplit = p.npad; p.hx = hx; p.split = exact ? 1 : 0;
  return nb_run(p, n, groups, stream);
}

extern "C" int hgb_nbr_linear_bwd_data(const float* g_out, int32_t n, int32_t n_out, const int32_t* rowptr, int32_t mean,
                                       const int32_t* order, const int32_t* grp_ptr, const int32_t* tiles, int32_t groups,
                                       const float* wt, int32_t k, float* g_h, float* g_xr, int32_t exact, hgb_stream_t stream) {
  HGB_REQUIRE(hgb_nbr_linear_supported(k, n_out, groups), "nbr_linear_bwd_data: unsupported shape k=%d n_out=%d groups=%d", k, n_out,
              groups);
  HGB_REQUIRE(n >= 0, "nbr_linear_bwd_data: bad size n=%d", n);
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(g_out && rowptr && grp_ptr && tiles && wt && g_h && g_xr, "nbr_linear_bwd_data: missing operand");
  NbrParams p = {};
  p.gather = 0; p.kin = n_out; p.ka = r32(n_out); p.x = g_out; p.rowptr = rowptr; p.mean = 0;
  p.order = order; p.tiles = tiles; p.grp_ptr = grp_ptr; p.w = wt; p.npad = 2 * r32(k);
  p.y0 = g_h; p.n0 = k; p.csplit = r32(k); p.y1 = g_xr; p.n1 = k; p.scale0 = mean ? 1 : 0; p.split = exact ? 1 : 0;
  return nb_run(p, n, groups, stream);
}
