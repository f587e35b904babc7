// libhgb.so -- the flat-buffer steps of every optimizer hydragnn/utils/optimizer/optimizer.py selects: SGD, Adam, AdamW,
// Adamax, Adagrad, Adadelta and RMSprop, one kernel template over one flat parameter / gradient / state buffer set:
//   * lr and grad_scale come from hyper_dev {lr, grad_scale} when it is given (a captured step follows a scheduler);
//   * the step count is read from step_dev (1-based inside the update) and incremented by a second launch after it;
//   * the gradient is multiplied by grad_scale before anything else (1/world after the flat all-reduce).
// All but AdamW follow torch.optim's single-tensor algorithm (foreach=False) element by element, in the same operation order:
// scalar coefficients (bias corrections, Adagrad's decayed lr) are computed once per thread in fp64 and rounded to fp32, as
// torch computes them in Python doubles; the elementwise arithmetic is fp32, as ATen's opmath for fp32 tensors.  AdamW keeps
// the fp32 hyperparameters and fp32 coefficients of its C entry point.
#include "hgb_common.cuh"

namespace {

constexpr int FLAT_THREADS = 256;

// ATen's lerp: self + w (end - self) for |w| < 0.5, else end - (end - self) (1 - w)
__device__ __forceinline__ float aten_lerp(float self, float end, float w) {
  const float d = end - self;
  return fabsf(w) < 0.5f ? self + w * d : end - d * (1.f - w);
}

// One element's update.  p, the scaled gradient g and up to three state values s0..s2 (in the order the entry point names
// them); a rule leaves the states it does not use untouched.  A sum of two products is written out with explicit roundings
// (torch's in-place mul_ then addcmul_ / add_): left to the compiler, the float4 body and the scalar loop could contract it into
// different fmas and give different bits for the same element.
struct SgdRule {
  float momentum, one_minus_dampening, wd;
  bool nesterov, first;
  // torch copies the gradient into a buffer it does not have yet: decided from the device step count, so every replay of a
  // captured step after the first one takes the momentum branch
  __device__ __forceinline__ void coef(float, double t) { first = t == 1.0; }
  __device__ __forceinline__ void apply(float lr, float& p, float g, float& buf, float&, float&) const {
    if (wd != 0.f) g = g + wd * p;
    if (momentum != 0.f) {
      buf = first ? g : __fmaf_rn(one_minus_dampening, g, __fmul_rn(buf, momentum));
      g = nesterov ? __fmaf_rn(momentum, buf, g) : buf;
    }
    p = p - lr * g;
  }
};

struct AdamRule {
  double b1, b2;
  float w1, b2f, w2, eps, wd;
  bool amsgrad;
  float neg_step_size, bc2_sqrt;
  __device__ __forceinline__ void coef(float lr, double t) {
    const double bc1 = 1.0 - pow(b1, t), bc2 = 1.0 - pow(b2, t);
    neg_step_size = (float)(-((double)lr / bc1));
    bc2_sqrt = (float)sqrt(bc2);
  }
  __device__ __forceinline__ void apply(float, float& p, float g, float& m, float& v, float& vmax) const {
    if (wd != 0.f) g = g + wd * p;
    m = aten_lerp(m, g, w1);                               // exp_avg.lerp_(grad, 1 - beta1)
    v = __fmaf_rn(w2 * g, g, __fmul_rn(v, b2f));
    float vv = v;
    if (amsgrad) {
      vmax = fmaxf(vmax, v);
      vv = vmax;
    }
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    p = p + neg_step_size * (m / denom);
  }
};

// torch.optim.AdamW's update with fp32 hyperparameters and fp32 bias corrections (not Adam's lerp and fp64 coefficients):
//   p *= 1 - lr wd;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= lr / (1 - b1^t) m / (sqrt(v) rsqrt(1 - b2^t) + eps)
// Every contraction is explicit, so the float4 body and the scalar loop give the same bits.
struct AdamWRule {
  float b1, b2, w1, w2, eps, wd;
  float decay, step_size, inv_sqrt_bc2;
  __device__ __forceinline__ void coef(float lr, double t) {
    const float tf = (float)t;
    decay = __fmaf_rn(-lr, wd, 1.f);
    step_size = __fdiv_rn(lr, 1.f - powf(b1, tf));
    inv_sqrt_bc2 = rsqrtf(1.f - powf(b2, tf));
  }
  __device__ __forceinline__ void apply(float, float& p, float g, float& m, float& v, float&) const {
    m = __fmaf_rn(g, w1, __fmul_rn(m, b1));
    v = __fmaf_rn(g, __fmul_rn(g, w2), __fmul_rn(v, b2));
    p = __fsub_rn(__fmul_rn(p, decay), __fdiv_rn(__fmul_rn(step_size, m), __fmaf_rn(sqrtf(v), inv_sqrt_bc2, eps)));
  }
};

struct AdamaxRule {
  double b1;
  float w1, b2f, eps, wd;
  float neg_clr;
  __device__ __forceinline__ void coef(float lr, double t) { neg_clr = (float)(-((double)lr / (1.0 - pow(b1, t)))); }
  __device__ __forceinline__ void apply(float, float& p, float g, float& m, float& u, float&) const {
    if (wd != 0.f) g = g + wd * p;
    m = aten_lerp(m, g, w1);
    u = fmaxf(u * b2f, fabsf(g) + eps);
    p = p + neg_clr * (m / u);
  }
};

struct AdagradRule {
  double lr_decay;
  float eps, wd;
  float neg_clr;
  __device__ __forceinline__ void coef(float lr, double t) { neg_clr = (float)(-((double)lr / (1.0 + (t - 1.0) * lr_decay))); }
  __device__ __forceinline__ void apply(float, float& p, float g, float& sum, float&, float&) const {
    if (wd != 0.f) g = g + wd * p;
    sum = sum + g * g;
    const float std = sqrtf(sum) + eps;
    p = p + neg_clr * (g / std);
  }
};

struct AdadeltaRule {
  float rho, w, eps, wd;
  __device__ __forceinline__ void coef(float, double) {}
  __device__ __forceinline__ void apply(float lr, float& p, float g, float& sq, float& acc, float&) const {
    if (wd != 0.f) g = g + wd * p;
    sq = __fmaf_rn(w * g, g, __fmul_rn(sq, rho));
    const float std = sqrtf(sq + eps);
    const float delta = sqrtf(acc + eps) / std * g;
    acc = __fmaf_rn(w * delta, delta, __fmul_rn(acc, rho));
    p = p - lr * delta;
  }
};

struct RmspropRule {
  float alpha, w, eps, wd, momentum;
  bool centered;
  __device__ __forceinline__ void coef(float, double) {}
  __device__ __forceinline__ void apply(float lr, float& p, float g, float& sq, float& buf, float& ga) const {
    if (wd != 0.f) g = g + wd * p;
    sq = __fmaf_rn(w * g, g, __fmul_rn(sq, alpha));
    float avg;
    if (centered) {
      ga = aten_lerp(ga, g, w);                            // grad_avg.lerp_(grad, 1 - alpha)
      avg = sqrtf(__fmaf_rn(-ga, ga, sq));
    } else {
      avg = sqrtf(sq);
    }
    avg = avg + eps;
    if (momentum > 0.f) {
      buf = __fadd_rn(__fmul_rn(buf, momentum), g / avg);
      p = p - lr * buf;
    } else {
      p = p - lr * (g / avg);
    }
  }
};

__device__ __forceinline__ float4 ld4(const float* a, int64_t i) { return reinterpret_cast<const float4*>(a)[i]; }
__device__ __forceinline__ void st4(float* a, int64_t i, float4 v) { reinterpret_cast<float4*>(a)[i] = v; }

// vec: every buffer is 16-byte aligned, so the first count / 4 * 4 elements go as float4 and the rest one by one.
template <class Rule>
__global__ void __launch_bounds__(FLAT_THREADS) flat_step_kernel(Rule r, float* __restrict__ p, const float* __restrict__ g,
                                                                 float* __restrict__ s0, float* __restrict__ s1,
                                                                 float* __restrict__ s2, int64_t count, float lr, float gscale,
                                                                 const float* __restrict__ step_dev,
                                                                 const float* __restrict__ hyper_dev, bool vec) {
  if (hyper_dev) {
    lr = hyper_dev[0];
    gscale = hyper_dev[1];
  }
  r.coef(lr, (double)step_dev[0] + 1.0);
  const int64_t stride = (int64_t)gridDim.x * FLAT_THREADS;
  const int64_t tid = (int64_t)blockIdx.x * FLAT_THREADS + threadIdx.x;
  const int64_t nvec = vec ? count / 4 : 0;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t i = tid; i < nvec; i += stride) {
    float4 pv = ld4(p, i), gv = ld4(g, i);
    float4 a = s0 ? ld4(s0, i) : z4, b = s1 ? ld4(s1, i) : z4, c = s2 ? ld4(s2, i) : z4;
    r.apply(lr, pv.x, __fmul_rn(gv.x, gscale), a.x, b.x, c.x);
    r.apply(lr, pv.y, __fmul_rn(gv.y, gscale), a.y, b.y, c.y);
    r.apply(lr, pv.z, __fmul_rn(gv.z, gscale), a.z, b.z, c.z);
    r.apply(lr, pv.w, __fmul_rn(gv.w, gscale), a.w, b.w, c.w);
    st4(p, i, pv);
    if (s0) st4(s0, i, a);
    if (s1) st4(s1, i, b);
    if (s2) st4(s2, i, c);
  }
  for (int64_t i = nvec * 4 + tid; i < count; i += stride) {
    float pv = p[i], a = s0 ? s0[i] : 0.f, b = s1 ? s1[i] : 0.f, c = s2 ? s2[i] : 0.f;
    r.apply(lr, pv, __fmul_rn(g[i], gscale), a, b, c);
    p[i] = pv;
    if (s0) s0[i] = a;
    if (s1) s1[i] = b;
    if (s2) s2[i] = c;
  }
}

__global__ void flat_step_count_kernel(float* step_dev) { step_dev[0] += 1.f; }

bool aligned16(const void* a) { return a == nullptr || (reinterpret_cast<uintptr_t>(a) & 15u) == 0; }

template <class Rule>
int launch(const char* name, const Rule& r, float* p, const float* g, float* s0, float* s1, float* s2, int64_t count, float lr,
           float gscale, float* step_dev, const float* hyper_dev, hgb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (count > 0) {
    const bool vec = aligned16(p) && aligned16(g) && aligned16(s0) && aligned16(s1) && aligned16(s2);
    const int64_t work = vec ? (count + 3) / 4 : count;
    flat_step_kernel<Rule><<<hgb_grid_for(work, FLAT_THREADS), FLAT_THREADS, 0, st>>>(r, p, g, s0, s1, s2, count, lr, gscale,
                                                                                   step_dev, hyper_dev, vec);
    HGB_LAUNCH_CHECK(name);
  }
  flat_step_count_kernel<<<1, 1, 0, st>>>(step_dev);
  HGB_LAUNCH_CHECK(name);
  return HGB_OK;
}

}  // namespace

extern "C" int hgb_sgd_step(float* p, const float* g, float* momentum_buffer, int64_t count, float lr, double momentum,
                            double dampening, int32_t nesterov, double weight_decay, float grad_scale, float* step_dev,
                            const float* hyper_dev, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g)), "sgd_step: bad arguments");
  HGB_REQUIRE(count == 0 || momentum == 0.0 || momentum_buffer, "sgd_step: momentum != 0 needs momentum_buffer");
  HGB_REQUIRE(!nesterov || (momentum > 0.0 && dampening == 0.0), "sgd_step: nesterov needs momentum > 0 and dampening 0");
  const SgdRule r{(float)momentum, (float)(1.0 - dampening), (float)weight_decay, nesterov != 0, false};
  return launch("sgd_step", r, p, g, momentum == 0.0 ? nullptr : momentum_buffer, nullptr, nullptr, count, lr, grad_scale, step_dev,
                hyper_dev, stream);
}

extern "C" int hgb_adam_step(float* p, const float* g, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, int64_t count,
                             float lr, double beta1, double beta2, double eps, double weight_decay, int32_t amsgrad,
                             float grad_scale, float* step_dev, const float* hyper_dev, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && exp_avg && exp_avg_sq)), "adam_step: bad arguments");
  HGB_REQUIRE(count == 0 || !amsgrad || max_exp_avg_sq, "adam_step: amsgrad needs max_exp_avg_sq");
  const AdamRule r{beta1, beta2, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, (float)weight_decay,
                   amsgrad != 0, 0.f, 0.f};
  return launch("adam_step", r, p, g, exp_avg, exp_avg_sq, amsgrad ? max_exp_avg_sq : nullptr, count, lr, grad_scale, step_dev,
                hyper_dev, stream);
}

extern "C" int hgb_adamw_step(float* p, const float* g, float* m, float* v, int64_t count, float lr, float beta1, float beta2,
                              float eps, float weight_decay, float grad_scale, float* step_dev, const float* hyper_dev,
                              hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && m && v)), "adamw_step: bad arguments");
  const AdamWRule r{beta1, beta2, 1.f - beta1, 1.f - beta2, eps, weight_decay, 0.f, 0.f, 0.f};
  return launch("adamw_step", r, p, g, m, v, nullptr, count, lr, grad_scale, step_dev, hyper_dev, stream);
}

extern "C" int hgb_adamax_step(float* p, const float* g, float* exp_avg, float* exp_inf, int64_t count, float lr, double beta1,
                               double beta2, double eps, double weight_decay, float grad_scale, float* step_dev,
                               const float* hyper_dev, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && exp_avg && exp_inf)), "adamax_step: bad arguments");
  const AdamaxRule r{beta1, (float)(1.0 - beta1), (float)beta2, (float)eps, (float)weight_decay, 0.f};
  return launch("adamax_step", r, p, g, exp_avg, exp_inf, nullptr, count, lr, grad_scale, step_dev, hyper_dev, stream);
}

extern "C" int hgb_adagrad_step(float* p, const float* g, float* sum, int64_t count, float lr, double lr_decay, double weight_decay,
                                double eps, float grad_scale, float* step_dev, const float* hyper_dev, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && sum)), "adagrad_step: bad arguments");
  const AdagradRule r{lr_decay, (float)eps, (float)weight_decay, 0.f};
  return launch("adagrad_step", r, p, g, sum, nullptr, nullptr, count, lr, grad_scale, step_dev, hyper_dev, stream);
}

extern "C" int hgb_adadelta_step(float* p, const float* g, float* square_avg, float* acc_delta, int64_t count, float lr, double rho,
                                 double eps, double weight_decay, float grad_scale, float* step_dev, const float* hyper_dev,
                                 hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && square_avg && acc_delta)), "adadelta_step: bad arguments");
  const AdadeltaRule r{(float)rho, (float)(1.0 - rho), (float)eps, (float)weight_decay};
  return launch("adadelta_step", r, p, g, square_avg, acc_delta, nullptr, count, lr, grad_scale, step_dev, hyper_dev, stream);
}

extern "C" int hgb_rmsprop_step(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg, int64_t count,
                                float lr, double alpha, double eps, double weight_decay, double momentum, int32_t centered,
                                float grad_scale, float* step_dev, const float* hyper_dev, hgb_stream_t stream) {
  HGB_REQUIRE(count >= 0 && step_dev && (count == 0 || (p && g && square_avg)), "rmsprop_step: bad arguments");
  HGB_REQUIRE(count == 0 || momentum <= 0.0 || momentum_buffer, "rmsprop_step: momentum > 0 needs momentum_buffer");
  HGB_REQUIRE(count == 0 || !centered || grad_avg, "rmsprop_step: centered needs grad_avg");
  const RmspropRule r{(float)alpha, (float)(1.0 - alpha), (float)eps, (float)weight_decay, (float)momentum, centered != 0};
  return launch("rmsprop_step", r, p, g, square_avg, momentum > 0.0 ? momentum_buffer : nullptr, centered ? grad_avg : nullptr,
                count, lr, grad_scale, step_dev, hyper_dev, stream);
}
