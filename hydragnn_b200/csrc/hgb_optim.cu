// libhgb.so -- losses (value + gradient in one pass) and PReLU; the optimizer steps are in hgb_optim_flat.cu.
#include "hgb_common.cuh"

// single block: deterministic tree reduction; count is small (number of targets in the batch)
__global__ void loss_fwd_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ target, int64_t count, int mode,
                                    float gscale, float* __restrict__ loss, float* __restrict__ gpred,
                                    const int32_t* __restrict__ valid_rows, int row_width) {
  __shared__ float sm[1024];
  float acc = 0.f;
  const int64_t total = count;
  if (valid_rows) {          // capacity-padded batch: only the first *valid_rows rows are real (hydragnn_b200/padded.py)
    const int64_t v = (int64_t)valid_rows[0] * row_width;
    count = v < count ? (v > 0 ? v : 0) : count;    // no real row: loss 0, gpred all zero
    for (int64_t i = count + threadIdx.x; gpred && i < total; i += blockDim.x) gpred[i] = 0.f;
  }
  const float inv = 1.f / (float)(count > 0 ? count : 1);
  for (int64_t i = threadIdx.x; i < count; i += blockDim.x) {
    const float d = pred[i] - target[i];
    if (mode == 0) {
      acc += d * d;
      if (gpred) gpred[i] = 2.f * d * inv * gscale;
    } else {
      acc += fabsf(d);
      if (gpred) gpred[i] = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * inv * gscale;
    }
  }
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = sm[0] * inv;
}

extern "C" int hgb_loss_fwd_bwd(const float* pred, const float* target, int64_t count, int32_t mode, float gscale, float* loss,
                                float* gpred, const int32_t* valid_rows, int32_t row_width, hgb_stream_t stream) {
  HGB_REQUIRE(count > 0 && pred && target && loss && (mode == 0 || mode == 1), "loss_fwd_bwd: bad arguments");
  HGB_REQUIRE(!valid_rows || row_width > 0, "loss_fwd_bwd: row_width must be positive with valid_rows");
  loss_fwd_bwd_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(pred, target, count, mode, gscale, loss, gpred, valid_rows, row_width);
  HGB_LAUNCH_CHECK("loss_fwd_bwd");
  return HGB_OK;
}

// Gaussian negative log-likelihood (torch.nn.GaussianNLLLoss, full=False, reduction="mean"), value and both gradients in one
// launch.  Node heads have millions of elements, so the grid has many CTAs: each CTA sums its grid-stride share in a fixed
// order into one fp64 partial; the CTA that finishes last (an atomic ticket decides which one, no value is accumulated
// atomically) sums the partials in index order.  The grid depends on `count` only, so repeated calls give the same bits.
constexpr int GNLL_THREADS = 256;
constexpr int GNLL_PER_THREAD = 8;
constexpr int GNLL_MAX_BLOCKS = 1024;

static int gnll_blocks(int64_t count) { return hgb_grid_for(count, GNLL_THREADS * GNLL_PER_THREAD, GNLL_MAX_BLOCKS); }

__device__ __forceinline__ double gnll_block_sum(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < GNLL_THREADS / 32; ++w) s += sm[w];
  __syncthreads();
  return s;        // valid in thread 0
}

__global__ void __launch_bounds__(GNLL_THREADS) gnll_fwd_bwd_kernel(
    const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ target, int64_t count, float eps,
    float* __restrict__ loss, float* __restrict__ gmean, float* __restrict__ gvar, double* __restrict__ partial,
    unsigned int* __restrict__ ticket, const int32_t* __restrict__ valid_rows, int row_width) {
  __shared__ double sm[GNLL_THREADS / 32];
  __shared__ bool last;
  int64_t n = count;
  if (valid_rows) {          // capacity-padded batch: only the first *valid_rows rows are real (hydragnn_b200/padded.py)
    const int64_t v = (int64_t)valid_rows[0] * row_width;
    n = v < count ? (v > 0 ? v : 0) : count;
  }
  // the loss is the mean of 0.5 (log v_c + d^2 / v_c), v_c = max(var, eps); the clamp passes the gradient through unchanged:
  // dL/dmean = d / v_c / n, dL/dvar = 0.5 (1 / v_c - d^2 / v_c^2) / n.  Evaluated in fp64, rounded once to fp32.
  const double inv = 1.0 / (double)(n > 0 ? n : 1);
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * GNLL_THREADS;
  for (int64_t i = (int64_t)blockIdx.x * GNLL_THREADS + threadIdx.x; i < count; i += stride) {
    if (i < n) {
      const double d = (double)mean[i] - (double)target[i];
      const double vc = fmax((double)var[i], (double)eps);
      const double q = d / vc;
      acc += log(vc) + d * q;
      gmean[i] = (float)(q * inv);
      gvar[i] = (float)(0.5 * (1.0 - d * q) / vc * inv);
    } else {
      gmean[i] = 0.f;
      gvar[i] = 0.f;
    }
  }
  const double s = gnll_block_sum(acc, sm);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double t = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += GNLL_THREADS) t += __ldcg(partial + b);
  t = gnll_block_sum(t, sm);
  if (threadIdx.x == 0) {
    loss[0] = n > 0 ? (float)(0.5 * t * inv) : 0.f;
    *ticket = 0u;
  }
}

extern "C" int64_t hgb_gnll_workspace_bytes(int64_t count) {
  return count > 0 ? (int64_t)sizeof(double) * (gnll_blocks(count) + 1) : 0;
}

extern "C" int hgb_gnll_fwd_bwd(const float* mean, const float* var, const float* target, int64_t count, float eps, float* loss,
                                float* gmean, float* gvar, void* workspace, const int32_t* valid_rows, int32_t row_width,
                                hgb_stream_t stream) {
  HGB_REQUIRE(count > 0 && mean && var && target && loss && gmean && gvar && workspace, "gnll_fwd_bwd: bad arguments");
  HGB_REQUIRE(eps > 0.f, "gnll_fwd_bwd: eps must be positive");
  HGB_REQUIRE(!valid_rows || row_width > 0, "gnll_fwd_bwd: row_width must be positive with valid_rows");
  const int blocks = gnll_blocks(count);
  double* partial = (double*)workspace;
  unsigned int* ticket = (unsigned int*)(partial + blocks);
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st);
  gnll_fwd_bwd_kernel<<<blocks, GNLL_THREADS, 0, st>>>(mean, var, target, count, eps, loss, gmean, gvar, partial, ticket,
                                                        valid_rows, row_width);
  HGB_LAUNCH_CHECK("gnll_fwd_bwd");
  return HGB_OK;
}

// torch.nn.PReLU() with its one learnable slope a, read from device memory on every launch (never by the host: the slope
// changes every optimiser step and a captured graph replays with whatever value it holds then).  Same arithmetic as ATen's
// prelu: y = z > 0 ? z : a z, dz = z > 0 ? g : a g (z = 0 and NaN take the slope branch), dL/da = sum over !(z > 0) of z g.
// The slope gradient is reduced as hgb_gnll_fwd_bwd reduces its loss: a grid that depends on `count` only, each CTA's share
// summed in a fixed order in fp64, the last CTA to finish adding the partials in index order.
__global__ void __launch_bounds__(GNLL_THREADS) prelu_fwd_kernel(const float* __restrict__ z, int64_t count,
                                                                 const float* __restrict__ slope, float* __restrict__ y) {
  const float a = __ldg(slope);
  const int64_t stride = (int64_t)gridDim.x * GNLL_THREADS;
  for (int64_t i = (int64_t)blockIdx.x * GNLL_THREADS + threadIdx.x; i < count; i += stride) {
    const float v = z[i];
    y[i] = v > 0.f ? v : a * v;
  }
}

template <bool SLOPE>
__global__ void __launch_bounds__(GNLL_THREADS) prelu_bwd_kernel(
    const float* __restrict__ g, const float* __restrict__ z, int64_t count, const float* __restrict__ slope,
    float* __restrict__ dz, float* __restrict__ dslope, double* __restrict__ partial, unsigned int* __restrict__ ticket) {
  const float a = __ldg(slope);
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * GNLL_THREADS;
  for (int64_t i = (int64_t)blockIdx.x * GNLL_THREADS + threadIdx.x; i < count; i += stride) {
    const float v = z[i], gi = g[i];
    const bool pos = v > 0.f;
    dz[i] = pos ? gi : a * gi;
    if (SLOPE && !pos) acc += (double)v * (double)gi;       // exact product of two floats, summed in fp64
  }
  if (!SLOPE) return;
  __shared__ double sm[GNLL_THREADS / 32];
  __shared__ bool last;
  const double s = gnll_block_sum(acc, sm);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double t = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += GNLL_THREADS) t += __ldcg(partial + b);
  t = gnll_block_sum(t, sm);
  if (threadIdx.x == 0) {
    dslope[0] = (float)t;
    *ticket = 0u;
  }
}

extern "C" int hgb_prelu_fwd(const float* z, int64_t count, const float* slope, float* y, hgb_stream_t stream) {
  HGB_REQUIRE(count > 0 && z && slope && y, "prelu_fwd: bad arguments");
  prelu_fwd_kernel<<<gnll_blocks(count), GNLL_THREADS, 0, (cudaStream_t)stream>>>(z, count, slope, y);
  HGB_LAUNCH_CHECK("prelu_fwd");
  return HGB_OK;
}

extern "C" int64_t hgb_prelu_workspace_bytes(int64_t count) { return hgb_gnll_workspace_bytes(count); }

extern "C" int hgb_prelu_bwd(const float* g, const float* z, int64_t count, const float* slope, float* dz, float* dslope,
                             void* workspace, int32_t skip_slope, hgb_stream_t stream) {
  HGB_REQUIRE(count > 0 && g && z && slope && dz, "prelu_bwd: bad arguments");
  HGB_REQUIRE(skip_slope || (dslope && workspace), "prelu_bwd: dslope and workspace are needed unless skip_slope");
  const int blocks = gnll_blocks(count);
  cudaStream_t st = (cudaStream_t)stream;
  if (skip_slope) {
    prelu_bwd_kernel<false><<<blocks, GNLL_THREADS, 0, st>>>(g, z, count, slope, dz, nullptr, nullptr, nullptr);
  } else {
    double* partial = (double*)workspace;
    unsigned int* ticket = (unsigned int*)(partial + blocks);
    cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st);
    prelu_bwd_kernel<true><<<blocks, GNLL_THREADS, 0, st>>>(g, z, count, slope, dz, dslope, partial, ticket);
  }
  HGB_LAUNCH_CHECK("prelu_bwd");
  return HGB_OK;
}
