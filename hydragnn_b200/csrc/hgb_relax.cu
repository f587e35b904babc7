// libhgb.so -- one FIRE iteration of a batched structure relaxation
// (examples/multidataset_hpo_sc26/structure_optimization_ASE.py :385-439 with ase.optimize.FIRE, ASE 3.26, maxstep given).
//
// One CTA per structure.  After the model has evaluated E_k and F_k at x_k, the CTA of a running structure
//   1. computes m_k = sqrt(max_i |F_i|^2), writes E_k and m_k into row k of the histories and applies the script's rules in
//      its order: revert (k >= 2, m_{k-1} > 0, (m_k - m_{k-1}) / m_{k-1} > threshold: x = x_{k-1}), converged (k >= 1,
//      m_k < fmax), max steps (k == max_steps).  Row 0 is the start x_0, to which no rule applies;
//   2. if the structure still runs, moves it to x_{k+1} with ASE's FIRE step on F_k.
// Every sum over a structure's 3N components is fp64: each thread adds its strided atoms in ascending order, then a fixed
// tree over the CTA -- no atomics on values, so every run gives the same bits.
#include "hgb_common.cuh"

namespace {

constexpr int RELAX_THREADS = 256;
// ase.optimize.FIRE defaults
constexpr double FIRE_DTMAX = 1.0, FIRE_FINC = 1.1, FIRE_FDEC = 0.5, FIRE_ASTART = 0.1, FIRE_FA = 0.99;
constexpr int FIRE_NMIN = 5;
constexpr int RELAX_RUNNING = 0, RELAX_CONVERGED = 1, RELAX_REVERTED = 2, RELAX_MAX_STEPS = 3;

// sum (op 0) or max (op 1) of one value per thread over the CTA, in a fixed order; every thread gets the result
template <int OP>
__device__ __forceinline__ double cta_reduce(double v, double* sh) {
  const int t = threadIdx.x;
  sh[t] = v;
  __syncthreads();
  for (int s = RELAX_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) sh[t] = OP == 0 ? sh[t] + sh[t + s] : fmax(sh[t], sh[t + s]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(RELAX_THREADS) fire_kernel(
    const int32_t* __restrict__ valid, const int32_t* __restrict__ gptr, const float* __restrict__ energy,
    const float* __restrict__ forces, double* __restrict__ x, double* __restrict__ v, double* __restrict__ x_prev,
    double* __restrict__ fire, int32_t* __restrict__ istate, double* __restrict__ e_hist, double* __restrict__ f_hist,
    int64_t hist_stride, float* __restrict__ e_out, float* __restrict__ f_out, float* __restrict__ pos, double ftol,
    double maxstep, int32_t max_steps, int32_t revert, double threshold, const int32_t* __restrict__ guard,
    int32_t* __restrict__ live) {
  __shared__ double sh[RELAX_THREADS];
  __shared__ int decision;
  const int gi = blockIdx.x, t = threadIdx.x;
  if (gi == 0 && t == 0) live[1] = *guard;            // the neighbour build of this iteration ran before this kernel
  if (gi >= valid[0]) return;                          // filler graphs: never touched
  int32_t* st = istate + 3 * gi;                       // status, k, FIRE's n
  if (st[0] != RELAX_RUNNING) return;                  // frozen: uniform over the CTA
  double* fs = fire + 3 * gi;                          // dt, a, m_{k-1}
  const int64_t lo = 3 * (int64_t)gptr[gi], hi = 3 * (int64_t)gptr[gi + 1];
  const int k = st[1];

  // ---- bookkeeping of the evaluation at x_k ---------------------------------------------------------------------------------
  double mx = 0.0, vf = 0.0, ff = 0.0, vv = 0.0;
  for (int64_t i = lo + 3 * t; i < hi; i += 3 * RELAX_THREADS) {
    const double f0 = forces[i], f1 = forces[i + 1], f2 = forces[i + 2];
    const double v0 = v[i], v1 = v[i + 1], v2 = v[i + 2];
    mx = fmax(mx, f0 * f0 + f1 * f1 + f2 * f2);
    vf += f0 * v0 + f1 * v1 + f2 * v2;
    ff += f0 * f0 + f1 * f1 + f2 * f2;
    vv += v0 * v0 + v1 * v1 + v2 * v2;
  }
  mx = cta_reduce<1>(mx, sh);
  vf = cta_reduce<0>(vf, sh);
  ff = cta_reduce<0>(ff, sh);
  vv = cta_reduce<0>(vv, sh);
  const double m = sqrt(mx);
  if (t == 0) {
    e_hist[(int64_t)k * hist_stride + gi] = (double)energy[gi];
    f_hist[(int64_t)k * hist_stride + gi] = m;
    int s = RELAX_RUNNING;
    const double mp = fs[2];
    if (revert && k >= 2 && mp > 0.0 && (m - mp) / mp > threshold) s = RELAX_REVERTED;
    else if (k >= 1 && m < ftol) s = RELAX_CONVERGED;
    else if (k >= max_steps) s = RELAX_MAX_STEPS;
    if (s != RELAX_RUNNING) st[0] = s;
    else atomicAdd(live, 1);                          // a count of structures, not a value: the order does not matter
    if (s != RELAX_REVERTED) e_out[gi] = energy[gi];   // a reverted structure keeps E_{k-1} and F_{k-1}
    decision = s;
  }
  __syncthreads();
  const int s = decision;
  if (s == RELAX_REVERTED) {
    for (int64_t i = lo + t; i < hi; i += RELAX_THREADS) {
      x[i] = x_prev[i];
      pos[i] = (float)x_prev[i];
    }
    return;
  }
  for (int64_t i = lo + t; i < hi; i += RELAX_THREADS) f_out[i] = forces[i];
  if (s != RELAX_RUNNING) return;

  // ---- FIRE step x_k -> x_{k+1} (ase/optimize/fire.py FIRE.step) -----------------------------------------------------------
  double dt = fs[0], a = fs[1];
  int nst = st[2];
  bool mixv = false, zerov = false;
  if (k > 0) {                                         // at k = 0 FIRE's v is None: v = 0 and no update of dt, a, n
    if (vf > 0.0) {
      mixv = true;
      if (nst > FIRE_NMIN) {
        dt = fmin(dt * FIRE_FINC, FIRE_DTMAX);
        a *= FIRE_FA;
      }
      nst += 1;
    } else {
      zerov = true;
      a = FIRE_ASTART;
      dt *= FIRE_FDEC;
      nst = 0;
    }
  }
  const double nf = sqrt(ff), nv = sqrt(vv), ca = 1.0 - fs[1], a0 = fs[1];
  // v = (1 - a) v + ((a f) / |f|) |v| with the a before its decay; v += dt f; dr = dt v.  The elementwise steps are rounded
  // one by one, as numpy evaluates them (no contraction into fma).
  double dd = 0.0;
  for (int64_t i = lo + t; i < hi; i += RELAX_THREADS) {
    const double f = forces[i];
    double vi = (k == 0 || zerov) ? 0.0 : v[i];
    if (mixv) vi = __dadd_rn(__dmul_rn(ca, vi), __dmul_rn(__ddiv_rn(__dmul_rn(a0, f), nf), nv));
    vi = __dadd_rn(vi, __dmul_rn(dt, f));
    v[i] = vi;
    const double dr = __dmul_rn(dt, vi);
    dd += dr * dr;
  }
  dd = cta_reduce<0>(dd, sh);
  const double ndr = sqrt(dd);
  const bool clamp = ndr > maxstep;
  for (int64_t i = lo + t; i < hi; i += RELAX_THREADS) {
    double dr = __dmul_rn(dt, v[i]);
    if (clamp) dr = __ddiv_rn(__dmul_rn(maxstep, dr), ndr);
    const double xi = x[i], xn = __dadd_rn(xi, dr);
    x_prev[i] = xi;
    x[i] = xn;
    pos[i] = (float)xn;
  }
  if (t == 0) {
    fs[0] = dt;
    fs[1] = a;
    fs[2] = m;
    st[1] = k + 1;
    st[2] = nst;
  }
}

}  // namespace

extern "C" int hgb_fire_step(const int32_t* valid, const int32_t* gptr, int32_t g_cap, const float* energy, const float* forces,
                             double* x, double* v, double* x_prev, double* fire, int32_t* istate, double* e_hist, double* f_hist,
                             int64_t hist_stride, float* e_out, float* f_out, float* pos, double ftol, double maxstep,
                             int32_t max_steps, int32_t revert, double threshold, const int32_t* guard, int32_t* live,
                             hgb_stream_t stream) {
  HGB_REQUIRE(g_cap >= 1 && hist_stride >= g_cap && valid && gptr && energy && forces && x && v && x_prev && fire && istate &&
                  e_hist && f_hist && e_out && f_out && pos && guard && live && ftol >= 0.0 && maxstep > 0.0 && max_steps >= 1 &&
                  (revert == 0 || revert == 1),
              "fire_step: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(live, 0, 2 * sizeof(int32_t), st) != cudaSuccess) {
    hgb_set_error("fire_step: memset failed");
    return HGB_ECUDA;
  }
  fire_kernel<<<g_cap, RELAX_THREADS, 0, st>>>(valid, gptr, energy, forces, x, v, x_prev, fire, istate, e_hist, f_hist, hist_stride,
                                               e_out, f_out, pos, ftol, maxstep, max_steps, revert, threshold, guard, live);
  HGB_LAUNCH_CHECK("fire_step");
  return HGB_OK;
}
