// libhgb.so -- the branch-weighted energy of a multi-branch interatomic potential
// (examples/multidataset_hpo_sc26/inference_fused.py: _weighted_average :547-563, _fused_energy_forces :508-544).
//
//   E_gb = e[g, b]                          (graph head: R = G rows)
//   E_gb = sum_{i in g} e[i, b]             (node head: R atoms grouped by graph, gptr [G + 1])
//   E_g  = sum_b w[g, b] E_gb
//
// and the seeds of the heads' backward, seeds[r, b] = w[g(r), b] dE[g].  One warp per graph: lane j sums branch j's atoms in
// ascending order, then every lane adds the lanes' w E_gb in ascending branch order by shuffle.  No atomics, so every run gives
// the same bits.
#include "hgb_common.cuh"

namespace {

constexpr int MIX_WARPS = 8;

__global__ void __launch_bounds__(MIX_WARPS * 32) branch_mix_fwd_kernel(const float* __restrict__ e, const int32_t* __restrict__ gptr,
                                                                        const float* __restrict__ w, int g, int b,
                                                                        float* __restrict__ eb, float* __restrict__ out) {
  const int gi = blockIdx.x * MIX_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gi >= g) return;                                         // uniform across the warp
  const int lo = gptr ? gptr[gi] : gi, hi = gptr ? gptr[gi + 1] : gi + 1;
  float acc = 0.f;
  for (int b0 = 0; b0 < b; b0 += 32) {
    const int j = b0 + lane;
    float v = 0.f;
    if (j < b) {
      float s = 0.f;
      for (int i = lo; i < hi; ++i) s += e[(int64_t)i * b + j];
      if (gptr) eb[(int64_t)gi * b + j] = s;
      v = w[(int64_t)gi * b + j] * s;
    }
    const int cnt = min(32, b - b0);
    for (int q = 0; q < cnt; ++q) acc += __shfl_sync(0xffffffffu, v, q);
  }
  if (lane == 0) out[gi] = acc;
}

__global__ void __launch_bounds__(MIX_WARPS * 32) branch_mix_bwd_kernel(const float* __restrict__ dout, const int32_t* __restrict__ gptr,
                                                                        const float* __restrict__ w, int g, int b,
                                                                        float* __restrict__ seeds) {
  const int gi = blockIdx.x * MIX_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gi >= g) return;
  const int64_t lo = gptr ? gptr[gi] : gi, hi = gptr ? gptr[gi + 1] : gi + 1;
  const float d = dout[gi];
  const float* wg = w + (int64_t)gi * b;
  for (int64_t k = lo * b + lane; k < hi * b; k += 32) seeds[k] = wg[k % b] * d;   // the graph's rows are contiguous
}

}  // namespace

extern "C" int hgb_branch_mix_fwd(const float* e, const int32_t* gptr, const float* w, int32_t g, int32_t r, int32_t b, float* eb,
                                  float* out, hgb_stream_t stream) {
  // empty tensors may come with null pointers: a pointer is needed only when there is something to read or write through it
  HGB_REQUIRE(g >= 0 && r >= 0 && b >= 1 && (gptr || r == g) && (g == 0 || (w && out && (eb || !gptr))) && (r == 0 || e),
              "branch_mix_fwd: bad arguments");
  if (g == 0) return HGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (r == 0) {                                                // every graph is empty: E_gb = E_g = 0, no kernel
    if (cudaMemsetAsync(out, 0, sizeof(float) * (size_t)g, st) != cudaSuccess ||
        cudaMemsetAsync(eb, 0, sizeof(float) * (size_t)g * b, st) != cudaSuccess) {
      hgb_set_error("branch_mix_fwd: memset failed");
      return HGB_ECUDA;
    }
    return HGB_OK;
  }
  branch_mix_fwd_kernel<<<(g + MIX_WARPS - 1) / MIX_WARPS, MIX_WARPS * 32, 0, st>>>(e, gptr, w, g, b, eb, out);
  HGB_LAUNCH_CHECK("branch_mix_fwd");
  return HGB_OK;
}

extern "C" int hgb_branch_mix_bwd(const float* dout, const int32_t* gptr, const float* w, int32_t g, int32_t r, int32_t b,
                                  float* seeds, hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && r >= 0 && b >= 1 && (gptr || r == g) && (g == 0 || (dout && w)) && (r == 0 || seeds),
              "branch_mix_bwd: bad arguments");
  if (g == 0 || r == 0) return HGB_OK;
  branch_mix_bwd_kernel<<<(g + MIX_WARPS - 1) / MIX_WARPS, MIX_WARPS * 32, 0, (cudaStream_t)stream>>>(dout, gptr, w, g, b, seeds);
  HGB_LAUNCH_CHECK("branch_mix_bwd");
  return HGB_OK;
}
