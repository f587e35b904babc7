// libhgb.so -- FiLM conditioning of node features on per-graph terms (hydragnn/models/Base.py _apply_graph_conditioning,
// mode "film"), over rows sorted by graph.  sm_90a only.
//
//   forward    y[r] = h[r] * (1 + tanh s[g]) + t[g]                 g = graph of row r, [s | t] = st[g] ([ng, 2c])
//   backward   dh[r] = dy[r] * (1 + tanh s[g])
//              ds[g] = (1 - tanh^2 s[g]) * sum_{r in g} dy[r] h[r],  dt[g] = sum_{r in g} dy[r]
//
// One CTA per FILM_CHUNK-row chunk, one thread per column, rows walked in order so the graph of a row is found by advancing
// through the offsets (one binary search per chunk).  The per-graph sums are fixed-order segmented reductions without atomics:
// a graph that lies inside one chunk is summed and written by that chunk; a graph that spans chunks leaves one partial per chunk
// (the chunk's "tail" slot in its first chunk, the "head" slot in every later one) and film_bwd_finish adds them in chunk order.
// Repeated runs are bit-identical.
#include "hgb_common.cuh"

namespace {

constexpr int FILM_CHUNK = 64;

__device__ __forceinline__ int film_graph_of(const int32_t* gptr, int ng, int row) {
  int lo = 0, hi = ng;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(gptr + mid) <= row) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void film_fwd_kernel(const float* __restrict__ h, int n, int c, const float* __restrict__ st, int64_t ldst,
                                const int32_t* __restrict__ gptr, int ng, float* __restrict__ y) {
  const int r0 = blockIdx.x * FILM_CHUNK, r1 = min(r0 + FILM_CHUNK, n);
  const int g0 = film_graph_of(gptr, ng, r0);
  for (int col = threadIdx.x; col < c; col += blockDim.x) {
    int g = g0, gend = __ldg(gptr + g + 1);
    float sc = 1.f + tanhf(__ldg(st + (int64_t)g * ldst + col)), sh = __ldg(st + (int64_t)g * ldst + c + col);
    for (int r = r0; r < r1; ++r) {
      if (r >= gend) {
        while (__ldg(gptr + g + 1) <= r) ++g;
        gend = __ldg(gptr + g + 1);
        sc = 1.f + tanhf(__ldg(st + (int64_t)g * ldst + col));
        sh = __ldg(st + (int64_t)g * ldst + c + col);
      }
      const int64_t o = (int64_t)r * c + col;
      y[o] = __ldg(h + o) * sc + sh;
    }
  }
}

// partials: head / tail [nchunks, 2c] (ds sums in columns [0, c), dt sums in [c, 2c))
__global__ void film_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ h, int n, int c, const float* __restrict__ st,
                                int64_t ldst, const int32_t* __restrict__ gptr, int ng, float* __restrict__ dh, float* __restrict__ dst,
                                float* __restrict__ head, float* __restrict__ tail) {
  const int chunk = blockIdx.x;
  const int r0 = chunk * FILM_CHUNK, r1 = min(r0 + FILM_CHUNK, n);
  const int g0 = film_graph_of(gptr, ng, r0);
  for (int col = threadIdx.x; col < c; col += blockDim.x) {
    int g = g0, gend = __ldg(gptr + g + 1);
    float tn = tanhf(__ldg(st + (int64_t)g * ldst + col));
    float as = 0.f, at = 0.f;
    auto flush = [&]() {
      const int a = __ldg(gptr + g), e = __ldg(gptr + g + 1);
      if (a >= r0 && e <= r1) {
        dst[(int64_t)g * 2 * c + col] = as * (1.f - tn * tn);
        dst[(int64_t)g * 2 * c + c + col] = at;
      } else {
        float* part = (a < r0 ? head : tail) + (int64_t)chunk * 2 * c;
        part[col] = as;
        part[c + col] = at;
      }
    };
    for (int r = r0; r < r1; ++r) {
      if (r >= gend) {
        if (dst) flush();
        as = at = 0.f;
        while (__ldg(gptr + g + 1) <= r) ++g;
        gend = __ldg(gptr + g + 1);
        tn = tanhf(__ldg(st + (int64_t)g * ldst + col));
      }
      const int64_t o = (int64_t)r * c + col;
      const float d = __ldg(dy + o);
      if (dh) dh[o] = d * (1.f + tn);
      as = fmaf(d, __ldg(h + o), as);
      at += d;
    }
    if (dst) flush();
  }
}

// the graphs that span chunks (and the empty ones): tail of the first chunk + heads of the later chunks, in chunk order
__global__ void film_bwd_finish_kernel(int c, const float* __restrict__ st, int64_t ldst, const int32_t* __restrict__ gptr,
                                       float* __restrict__ dst, const float* __restrict__ head, const float* __restrict__ tail) {
  const int g = blockIdx.x;
  const int a = __ldg(gptr + g), e = __ldg(gptr + g + 1);
  const int cf = a / FILM_CHUNK, cl = (e - 1) / FILM_CHUNK;
  if (e > a && cf == cl) return;                      // written by its chunk
  for (int col = threadIdx.x; col < c; col += blockDim.x) {
    float as = 0.f, at = 0.f;
    if (e > a) {
      as = tail[(int64_t)cf * 2 * c + col];
      at = tail[(int64_t)cf * 2 * c + c + col];
      for (int k = cf + 1; k <= cl; ++k) {
        as += head[(int64_t)k * 2 * c + col];
        at += head[(int64_t)k * 2 * c + c + col];
      }
    }
    const float tn = tanhf(__ldg(st + (int64_t)g * ldst + col));
    dst[(int64_t)g * 2 * c + col] = as * (1.f - tn * tn);
    dst[(int64_t)g * 2 * c + c + col] = at;
  }
}

int film_threads(int c) { return c >= 128 ? 128 : ((c + 31) / 32) * 32; }

}  // namespace

extern "C" int64_t hgb_film_bwd_workspace_bytes(int32_t n, int32_t c) {
  const int64_t chunks = ((int64_t)n + FILM_CHUNK - 1) / FILM_CHUNK;
  return 2 * chunks * 2 * (int64_t)c * 4;
}

extern "C" int hgb_film_fwd(const float* h, int32_t n, int32_t c, const float* st, int64_t ldst, const int32_t* gptr, int32_t ng, float* y,
                            hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && c >= 1 && ng >= 1 && ldst >= 2 * c && (n == 0 || (h && st && gptr && y)), "film_fwd: bad arguments n=%d c=%d ng=%d",
              n, c, ng);
  if (n == 0) return HGB_OK;
  film_fwd_kernel<<<(n + FILM_CHUNK - 1) / FILM_CHUNK, film_threads(c), 0, (cudaStream_t)stream>>>(h, n, c, st, ldst, gptr, ng, y);
  HGB_LAUNCH_CHECK("film_fwd");
  return HGB_OK;
}

extern "C" int hgb_film_bwd(const float* dy, const float* h, int32_t n, int32_t c, const float* st, int64_t ldst, const int32_t* gptr,
                            int32_t ng, float* dh, float* dst, void* ws, int64_t ws_bytes, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && c >= 1 && ng >= 1 && ldst >= 2 * c && st && gptr && (n == 0 || (dy && h)), "film_bwd: bad arguments n=%d c=%d ng=%d",
              n, c, ng);
  HGB_REQUIRE(!dst || (ws && ws_bytes >= hgb_film_bwd_workspace_bytes(n, c)), "film_bwd: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t chunks = ((int64_t)n + FILM_CHUNK - 1) / FILM_CHUNK;
  float* head = reinterpret_cast<float*>(ws);
  float* tail = dst ? head + chunks * 2 * c : nullptr;
  if (n > 0 && (dh || dst)) {
    film_bwd_kernel<<<(unsigned)chunks, film_threads(c), 0, s>>>(dy, h, n, c, st, ldst, gptr, ng, dh, dst, head, tail);
    HGB_LAUNCH_CHECK("film_bwd");
  }
  if (dst) {
    film_bwd_finish_kernel<<<ng, film_threads(c), 0, s>>>(c, st, ldst, gptr, dst, head, tail);
    HGB_LAUNCH_CHECK("film_bwd_finish");
  }
  return HGB_OK;
}
