// libhgb.so -- error plumbing, prefix scan, CSR construction.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "hgb_common.cuh"

#include <cub/device/device_radix_sort.cuh>

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void hgb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void hgb_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" int hgb_version(void) { return 114; }
extern "C" const char* hgb_last_error(void) { return g_err; }
extern "C" int64_t hgb_launch_count(void) { return g_launches.load(); }

// ------------------------------------------------------------------------------------------------
// exclusive scan (three small kernels; n <= 2^31).  Block = 1024 items.
// ------------------------------------------------------------------------------------------------
#define SCAN_B 1024

__device__ __forceinline__ int block_exclusive_scan_1024(int v, int* total) {
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = warp_tot[lane];
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    warp_tot[lane] = winc - w;  // exclusive over warps
    if (lane == 31) *total = winc;
  }
  __syncthreads();
  return inc - v + warp_tot[wid];
}

__global__ void scan_block_kernel(const int32_t* __restrict__ in, int32_t* __restrict__ out, int64_t n,
                                  int32_t* __restrict__ block_sums) {
  __shared__ int total;
  int64_t i = (int64_t)blockIdx.x * SCAN_B + threadIdx.x;
  int v = i < n ? in[i] : 0;
  int ex = block_exclusive_scan_1024(v, &total);
  if (i < n) out[i] = ex;
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// single block: exclusive scan of block sums in place (nb arbitrary: serial over chunks of 1024)
__global__ void scan_sums_kernel(int32_t* __restrict__ sums, int nb, int32_t* __restrict__ grand_total) {
  __shared__ int total;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += SCAN_B) {
    int i = base + threadIdx.x;
    int v = i < nb ? sums[i] : 0;
    int ex = block_exclusive_scan_1024(v, &total);
    int c = carry;
    if (i < nb) sums[i] = ex + c;
    __syncthreads();
    if (threadIdx.x == 0) carry = c + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) *grand_total = carry;
}

__global__ void scan_add_kernel(int32_t* __restrict__ out, int64_t n, const int32_t* __restrict__ sums,
                                const int32_t* __restrict__ grand_total) {
  int64_t i = (int64_t)blockIdx.x * SCAN_B + threadIdx.x;
  if (i < n) out[i] += sums[blockIdx.x];
  if (i == 0) out[n] = *grand_total;
}

extern "C" int64_t hgb_exclusive_scan_workspace_bytes(int64_t n) { return 4 * ((n + SCAN_B - 1) / SCAN_B + 2); }

extern "C" int hgb_exclusive_scan_i32(const int32_t* in, int32_t* out, int64_t n, void* workspace,
                                      hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && out && workspace, "exclusive_scan: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  int nb = (int)((n + SCAN_B - 1) / SCAN_B);
  int32_t* sums = (int32_t*)workspace;
  int32_t* total = sums + nb + 1;
  if (nb == 0) {
    cudaMemsetAsync(out, 0, sizeof(int32_t), st);
    return HGB_OK;
  }
  scan_block_kernel<<<nb, SCAN_B, 0, st>>>(in, out, n, sums);
  HGB_LAUNCH_CHECK("scan_block");
  scan_sums_kernel<<<1, SCAN_B, 0, st>>>(sums, nb, total);
  HGB_LAUNCH_CHECK("scan_sums");
  scan_add_kernel<<<nb, SCAN_B, 0, st>>>(out, n, sums, total);
  HGB_LAUNCH_CHECK("scan_add");
  return HGB_OK;
}

// ------------------------------------------------------------------------------------------------
// CSR view of an index vector (stable)
// ------------------------------------------------------------------------------------------------
__global__ void csr_hist_kernel(const int64_t* __restrict__ idx, int64_t e, int32_t n, int32_t* __restrict__ idx32,
                                int32_t* __restrict__ count, int32_t* __restrict__ bad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k = idx[i];
    if (k < 0 || k >= n) {
      atomicOr(bad, 2);     // HGB guard bit "index outside [0, n)" (hydragnn_b200.ops.GUARD_BAD_INDEX)
      k = 0;
    }
    idx32[i] = (int32_t)k;
    atomicAdd(&count[k], 1);
  }
}

__global__ void iota_i32_kernel(int32_t* __restrict__ out, int64_t e) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) out[i] = (int32_t)i;
}

static inline int csr_key_bits(int32_t n) {
  int bits = 1;
  while (bits < 31 && (1ll << bits) < (int64_t)n) ++bits;
  return bits;
}

static inline size_t csr_sort_temp_bytes(int64_t e, int32_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)(e > 0 ? e : 1), 0, csr_key_bits(n));
  return (bytes + 255) & ~(size_t)255;
}

extern "C" int64_t hgb_csr_workspace_bytes(int64_t e, int32_t n) {
  // counts (n + 8) | iota [e] | sorted keys [e] | scan workspace | radix-sort temporaries
  return 4 * ((int64_t)n + 8) + 8 * ((e + 63) & ~63ll) + hgb_exclusive_scan_workspace_bytes(n) + 256 +
         (int64_t)csr_sort_temp_bytes(e, n) + 256;
}

// Stable by construction: a least-significant-digit radix sort of (key = idx, value = edge id) keeps equal keys in ascending edge
// id, whatever the segment lengths (the round-1 per-segment insertion sort was quadratic in the longest segment).
extern "C" int hgb_csr_build(const int64_t* idx, int64_t e, int32_t n, int32_t* idx32, int32_t* rowptr,
                             int32_t* perm, int32_t* guard_flag, void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && n >= 0 && rowptr && workspace, "csr_build: bad arguments");
  HGB_REQUIRE(e < (1ll << 31), "csr_build: more than 2^31 - 1 entries");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t epad = (e + 63) & ~63ll;
  int32_t* count = (int32_t*)workspace;           // n + 8 (slot n: bad-index flag of this call)
  int32_t* iota = count + n + 8;
  int32_t* keys_out = iota + epad;
  char* scan_ws = (char*)(keys_out + epad);
  scan_ws = (char*)(((uintptr_t)scan_ws + 255) & ~(uintptr_t)255);
  char* sort_ws = scan_ws + ((hgb_exclusive_scan_workspace_bytes(n) + 255) & ~255ll);
  cudaMemsetAsync(count, 0, 4 * ((int64_t)n + 8), st);
  if (e > 0) {
    csr_hist_kernel<<<hgb_grid_for(e, 256), 256, 0, st>>>(idx, e, n, idx32, count, guard_flag ? guard_flag : count + n);
    HGB_LAUNCH_CHECK("csr_hist");
  }
  int rc = hgb_exclusive_scan_i32(count, rowptr, n, scan_ws, stream);
  if (rc) return rc;
  if (e > 0) {
    iota_i32_kernel<<<hgb_grid_for(e, 256), 256, 0, st>>>(iota, e);
    HGB_LAUNCH_CHECK("csr_iota");
    size_t temp = csr_sort_temp_bytes(e, n);
    cudaError_t err = cub::DeviceRadixSort::SortPairs((void*)sort_ws, temp, (const int32_t*)idx32, keys_out, (const int32_t*)iota,
                                                      perm, (int)e, 0, csr_key_bits(n), st);
    if (err != cudaSuccess) {
      hgb_set_error("csr_build: radix sort failed: %s", cudaGetErrorString(err));
      return HGB_ECUDA;
    }
    // (the radix-sort kernels are library code and are not counted as libhgb launches)
  }
  return HGB_OK;
}

// Stable CSR fill for index vectors whose entries are GROUPED: the edges of graph g are the contiguous range
// [edge_ptr[node_ptr[g]], edge_ptr[node_ptr[g + 1]]) and only reference nodes of graph g (what the engine's radius-graph kernels
// emit: edges sorted by target, graphs never interact).  One warp per graph walks its edges 32 at a time; equal keys inside a
// warp-step are ranked with match_any (lower lanes first), so every segment comes out in ascending edge id -- no sort at all.
__global__ void csr_fill_grouped_kernel(const int32_t* __restrict__ idx32, const int32_t* __restrict__ node_ptr,
                                        const int32_t* __restrict__ edge_ptr, int g, const int32_t* __restrict__ rowptr,
                                        int32_t* __restrict__ cursor, int32_t* __restrict__ perm) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int k = blockIdx.x * wpb + (threadIdx.x >> 5); k < g; k += gridDim.x * wpb) {
    const int e0 = edge_ptr[node_ptr[k]], e1 = edge_ptr[node_ptr[k + 1]];
    for (int base = e0; base < e1; base += 32) {
      const int e = base + lane;
      const bool on = e < e1;
      const int key = on ? idx32[e] : -1 - lane;                 // distinct dummies: never match a real key
      const unsigned peers = __match_any_sync(0xffffffffu, key);
      const int rank = __popc(peers & ((1u << lane) - 1u));
      int cur = 0;
      if (on) cur = cursor[key];
      __syncwarp();
      if (on) {
        perm[rowptr[key] + cur + rank] = e;
        if (rank == 0) cursor[key] = cur + __popc(peers);
      }
      __syncwarp();
    }
  }
}

extern "C" int64_t hgb_csr_grouped_workspace_bytes(int64_t e, int32_t n) {
  return 4 * ((int64_t)n + 8) * 2 + hgb_exclusive_scan_workspace_bytes(n) + 512;
}

extern "C" int hgb_csr_build_grouped(const int64_t* idx, int64_t e, int32_t n, const int32_t* node_ptr, const int32_t* edge_ptr,
                                     int32_t g, int32_t* idx32, int32_t* rowptr, int32_t* perm, int32_t* guard_flag,
                                     void* workspace, hgb_stream_t stream) {
  HGB_REQUIRE(e >= 0 && n >= 0 && g >= 0 && node_ptr && edge_ptr && rowptr && workspace, "csr_build_grouped: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* count = (int32_t*)workspace;           // n + 8
  int32_t* cursor = count + n + 8;                // n + 8
  char* scan_ws = (char*)(cursor + n + 8);
  scan_ws = (char*)(((uintptr_t)scan_ws + 255) & ~(uintptr_t)255);
  cudaMemsetAsync(count, 0, 4 * ((int64_t)n + 8) * 2, st);
  if (e > 0) {
    csr_hist_kernel<<<hgb_grid_for(e, 256), 256, 0, st>>>(idx, e, n, idx32, count, guard_flag ? guard_flag : count + n);
    HGB_LAUNCH_CHECK("csr_hist");
  }
  int rc = hgb_exclusive_scan_i32(count, rowptr, n, scan_ws, stream);
  if (rc) return rc;
  if (e > 0 && g > 0) {
    csr_fill_grouped_kernel<<<hgb_grid_for(g, 8), 256, 0, st>>>(idx32, node_ptr, edge_ptr, g, rowptr, cursor, perm);
    HGB_LAUNCH_CHECK("csr_fill_grouped");
  }
  return HGB_OK;
}

// out[p] = idx[perm[p]]  (the neighbour of every CSR slot, so the fused kernels do one dependent index load less)
__global__ void gather_i32_kernel(const int32_t* __restrict__ idx, const int32_t* __restrict__ perm, int64_t e, int32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) out[i] = idx[perm[i]];
}
extern "C" int hgb_gather_i32(const int32_t* idx, const int32_t* perm, int64_t e, int32_t* out, hgb_stream_t stream) {
  if (e == 0) return HGB_OK;
  HGB_REQUIRE(idx && perm && out, "gather_i32: null pointer");
  gather_i32_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(idx, perm, e, out);
  HGB_LAUNCH_CHECK("gather_i32");
  return HGB_OK;
}

// ------------------------------------------------------------------------------------------------
// device-side collate (replaces the index bookkeeping of PyG Batch.from_data_list, hydragnn/preprocess/load_data.py:157-164):
// batch[i] = graph of node i, and edge_index with per-graph node offsets added, both from [G+1] offset vectors.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ptr_search(const int32_t* __restrict__ ptr, int g, int64_t i) {   // largest k with ptr[k] <= i
  int lo = 0, hi = g;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (ptr[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void collate_batch_vector_kernel(const int32_t* __restrict__ ptr, int g, int64_t n, int64_t* __restrict__ batch) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) batch[i] = ptr_search(ptr, g, i);
}

__global__ void collate_offset_edges_kernel(const int64_t* __restrict__ local, const int32_t* __restrict__ eptr,
                                            const int32_t* __restrict__ nptr, int g, int64_t e, int64_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t off = nptr[ptr_search(eptr, g, i)];
    out[i] = local[i] + off;
    out[e + i] = local[e + i] + off;
  }
}

extern "C" int hgb_collate_batch_vector(const int32_t* ptr, int32_t g, int64_t n, int64_t* batch, hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && n >= 0 && ptr && (n == 0 || batch), "collate_batch_vector: bad arguments");
  if (n == 0) return HGB_OK;
  collate_batch_vector_kernel<<<hgb_grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(ptr, g, n, batch);
  HGB_LAUNCH_CHECK("collate_batch_vector");
  return HGB_OK;
}

extern "C" int hgb_collate_offset_edges(const int64_t* edge_index_local, const int32_t* edge_ptr, const int32_t* node_ptr, int32_t g,
                                        int64_t e, int64_t* edge_index, hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && e >= 0 && edge_ptr && node_ptr && (e == 0 || (edge_index_local && edge_index)), "collate_offset_edges: bad arguments");
  if (e == 0) return HGB_OK;
  collate_offset_edges_kernel<<<hgb_grid_for(e, 256), 256, 0, (cudaStream_t)stream>>>(edge_index_local, edge_ptr, node_ptr, g, e, edge_index);
  HGB_LAUNCH_CHECK("collate_offset_edges");
  return HGB_OK;
}
