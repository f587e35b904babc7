// libhgb.so -- radius graphs (open boundary and periodic), batched over graphs.
//
// Graphs on this path are tiny (9..200 atoms, SURVEY 8d), so the neighbour search is a brute-force
// scan of the query's own graph: one thread per query/target node, candidates visited in ascending
// index.  That reproduces the visitation order of torch_cluster's CUDA kernel, which is what fixes
// WHICH neighbours survive the max_neighbours cap (oracle/radius_graph.py restates the rule).
// Integer outputs are bit-exact against the oracle: the accept test uses explicitly rounded
// multiplies/adds (no FMA contraction).
#include "hgb_common.cuh"

__device__ __forceinline__ int find_graph(const int32_t* __restrict__ gptr, int g, int i) {
  int lo = 0, hi = g;  // invariant: gptr[lo] <= i < gptr[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (gptr[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

template <bool FILL>
__global__ void radius_open_kernel(const float* __restrict__ pos, const int32_t* __restrict__ gptr, int n, int g,
                                   float r, int cap, int loop, int32_t* __restrict__ deg,
                                   const int32_t* __restrict__ rowptr, int64_t e, int64_t* __restrict__ ei) {
  const float r2 = __fmul_rn(r, r);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int k = find_graph(gptr, g, i);
    const int lo = gptr[k], hi = gptr[k + 1];
    const float xi = pos[3 * i], yi = pos[3 * i + 1], zi = pos[3 * i + 2];
    int matches = 0, out = 0;
    int64_t base = FILL ? rowptr[i] : 0;
    for (int j = lo; j < hi && matches < cap; ++j) {
      float dx = __fsub_rn(pos[3 * j], xi), dy = __fsub_rn(pos[3 * j + 1], yi), dz = __fsub_rn(pos[3 * j + 2], zi);
      float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d2 < r2) {
        ++matches;
        if (loop || j != i) {
          if (FILL && base + out < e) {   // e may be a caller-promised count (captured steps): never write past it
            ei[base + out] = j;
            ei[e + base + out] = i;
          }
          ++out;
        }
      }
    }
    if (!FILL) deg[i] = out;
  }
}

extern "C" int hgb_radius_graph_count(const float* pos, const int32_t* graph_ptr, int32_t n, int32_t g, float r,
                                      int32_t max_neighbors, int32_t loop, int32_t* deg, hgb_stream_t stream) {
  if (n == 0) return HGB_OK;
  HGB_REQUIRE(n > 0 && g >= 0 && r > 0.f && max_neighbors > 0 && deg, "radius_graph_count: bad arguments");
  int cap = loop ? max_neighbors : (max_neighbors == INT32_MAX ? max_neighbors : max_neighbors + 1);
  radius_open_kernel<false><<<hgb_grid_for(n, 128), 128, 0, (cudaStream_t)stream>>>(pos, graph_ptr, n, g, r, cap, loop,
                                                                                   deg, nullptr, 0, nullptr);
  HGB_LAUNCH_CHECK("radius_open_count");
  return HGB_OK;
}

extern "C" int hgb_radius_graph_fill(const float* pos, const int32_t* graph_ptr, int32_t n, int32_t g, float r,
                                     int32_t max_neighbors, int32_t loop, const int32_t* rowptr, int64_t e,
                                     int64_t* edge_index, hgb_stream_t stream) {
  if (n == 0 || e == 0) return HGB_OK;
  HGB_REQUIRE(n > 0 && g >= 0 && r > 0.f && max_neighbors > 0 && rowptr, "radius_graph_fill: bad arguments");
  int cap = loop ? max_neighbors : (max_neighbors == INT32_MAX ? max_neighbors : max_neighbors + 1);
  radius_open_kernel<true><<<hgb_grid_for(n, 128), 128, 0, (cudaStream_t)stream>>>(pos, graph_ptr, n, g, r, cap, loop,
                                                                                  nullptr, rowptr, e, edge_index);
  HGB_LAUNCH_CHECK("radius_open_fill");
  return HGB_OK;
}

// ------------------------------------------------------------------------------------------------
// periodic
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double ldpos(const void* pos, int is64, int64_t i) {
  return is64 ? ((const double*)pos)[i] : (double)((const float*)pos)[i];
}

// image range per graph: nimg[k] = ceil(cutoff / height_k + frac_spread_k) + 1 for periodic axes
__global__ void pbc_range_kernel(const void* __restrict__ pos, int is64, const int32_t* __restrict__ gptr,
                                 const double* __restrict__ cell, const int32_t* __restrict__ pbc,
                                 const double* __restrict__ cutoff, int g, int32_t* __restrict__ nimg) {
  const int k = blockIdx.x;
  if (k >= g) return;
  const double* c = cell + 9 * k;
  double inv[9];
  const double det = c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6]) + c[2] * (c[3] * c[7] - c[4] * c[6]);
  const double id = 1.0 / det;
  inv[0] = (c[4] * c[8] - c[5] * c[7]) * id; inv[1] = (c[2] * c[7] - c[1] * c[8]) * id; inv[2] = (c[1] * c[5] - c[2] * c[4]) * id;
  inv[3] = (c[5] * c[6] - c[3] * c[8]) * id; inv[4] = (c[0] * c[8] - c[2] * c[6]) * id; inv[5] = (c[2] * c[3] - c[0] * c[5]) * id;
  inv[6] = (c[3] * c[7] - c[4] * c[6]) * id; inv[7] = (c[1] * c[6] - c[0] * c[7]) * id; inv[8] = (c[0] * c[4] - c[1] * c[3]) * id;
  __shared__ double smin[3][128], smax[3][128];
  double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
  for (int i = gptr[k] + threadIdx.x; i < gptr[k + 1]; i += blockDim.x) {
    double p0 = ldpos(pos, is64, 3 * (int64_t)i), p1 = ldpos(pos, is64, 3 * (int64_t)i + 1), p2 = ldpos(pos, is64, 3 * (int64_t)i + 2);
    for (int a = 0; a < 3; ++a) {  // frac = pos @ inv(cell)
      double f = p0 * inv[a] + p1 * inv[3 + a] + p2 * inv[6 + a];
      mn[a] = fmin(mn[a], f);
      mx[a] = fmax(mx[a], f);
    }
  }
  for (int a = 0; a < 3; ++a) { smin[a][threadIdx.x] = mn[a]; smax[a][threadIdx.x] = mx[a]; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double vol = fabs(det);
    for (int a = 0; a < 3; ++a) {
      int out = 0;
      if (pbc[3 * k + a] && gptr[k + 1] > gptr[k]) {
        double lo = 1e300, hi = -1e300;
        for (int t = 0; t < blockDim.x; ++t) { lo = fmin(lo, smin[a][t]); hi = fmax(hi, smax[a][t]); }
        const double* u = c + 3 * ((a + 1) % 3);
        const double* w = c + 3 * ((a + 2) % 3);
        double cx = u[1] * w[2] - u[2] * w[1], cy = u[2] * w[0] - u[0] * w[2], cz = u[0] * w[1] - u[1] * w[0];
        double height = vol / sqrt(cx * cx + cy * cy + cz * cz);
        out = (int)ceil(cutoff[k] / height + (hi - lo)) + 1;
      }
      nimg[3 * k + a] = out;
    }
  }
}

struct PbcCand {
  double len;
  int src, sx, sy, sz;
};
__device__ __forceinline__ bool cand_less(const PbcCand& a, const PbcCand& b) {
  if (a.len != b.len) return a.len < b.len;
  if (a.src != b.src) return a.src < b.src;
  if (a.sx != b.sx) return a.sx < b.sx;
  if (a.sy != b.sy) return a.sy < b.sy;
  return a.sz < b.sz;
}

template <bool FILL>
__global__ void radius_pbc_kernel(const void* __restrict__ pos, int is64, const int32_t* __restrict__ gptr,
                                  const double* __restrict__ cell, const int32_t* __restrict__ nimg,
                                  const double* __restrict__ cutoff, int n, int g, int32_t* __restrict__ count,
                                  const int32_t* __restrict__ candptr, int64_t cand_cap, int32_t* __restrict__ csrc,
                                  int32_t* __restrict__ cshift, double* __restrict__ clen) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int k = find_graph(gptr, g, j);
    const int lo = gptr[k], hi = gptr[k + 1];
    const double* c = cell + 9 * k;
    const double c2 = __dmul_rn(cutoff[k], cutoff[k]);
    const int n0 = nimg[3 * k], n1 = nimg[3 * k + 1], n2 = nimg[3 * k + 2];
    const double xj = ldpos(pos, is64, 3 * (int64_t)j), yj = ldpos(pos, is64, 3 * (int64_t)j + 1), zj = ldpos(pos, is64, 3 * (int64_t)j + 2);
    // Image pruning.  The reference enumerates every image in [-n_a, n_a]^3 and keeps |v| < cutoff.  With fractional
    // coordinates f = pos inv(cell), a displacement v = pos_j - pos_i + S cell has |v| >= |f_j,a - f_i,a + S_a| / |b_a|
    // (b_a = column a of inv(cell)), so only S_a in [-r|b_a| - df_a, r|b_a| - df_a] can pass: the same candidate set (the
    // interval is widened by 1e-9 before rounding), two orders of magnitude fewer distance evaluations.
    double inv[9];
    {
      const double det = c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6]) + c[2] * (c[3] * c[7] - c[4] * c[6]);
      const double id = 1.0 / det;
      inv[0] = (c[4] * c[8] - c[5] * c[7]) * id; inv[1] = (c[2] * c[7] - c[1] * c[8]) * id; inv[2] = (c[1] * c[5] - c[2] * c[4]) * id;
      inv[3] = (c[5] * c[6] - c[3] * c[8]) * id; inv[4] = (c[0] * c[8] - c[2] * c[6]) * id; inv[5] = (c[2] * c[3] - c[0] * c[5]) * id;
      inv[6] = (c[3] * c[7] - c[4] * c[6]) * id; inv[7] = (c[1] * c[6] - c[0] * c[7]) * id; inv[8] = (c[0] * c[4] - c[1] * c[3]) * id;
    }
    double rb[3], fj[3];
    const int nn[3] = {n0, n1, n2};
    for (int a = 0; a < 3; ++a) {
      rb[a] = cutoff[k] * sqrt(inv[a] * inv[a] + inv[3 + a] * inv[3 + a] + inv[6 + a] * inv[6 + a]) * (1.0 + 1e-9) + 1e-9;
      fj[a] = xj * inv[a] + yj * inv[3 + a] + zj * inv[6 + a];
    }
    int cnt = 0;
    const int base = FILL ? candptr[j] : 0;
    for (int i = lo; i < hi; ++i) {
      const double xi = ldpos(pos, is64, 3 * (int64_t)i), yi = ldpos(pos, is64, 3 * (int64_t)i + 1), zi = ldpos(pos, is64, 3 * (int64_t)i + 2);
      const double bx = __dsub_rn(xj, xi);
      const double by = __dsub_rn(yj, yi);
      const double bz = __dsub_rn(zj, zi);
      int slo[3], shi[3];
      bool empty = false;
      for (int a = 0; a < 3; ++a) {
        const double df = fj[a] - (xi * inv[a] + yi * inv[3 + a] + zi * inv[6 + a]);
        const double slack = 1e-9 * (1.0 + fabs(df));
        slo[a] = max(-nn[a], (int)ceil(-rb[a] - df - slack));
        shi[a] = min(nn[a], (int)floor(rb[a] - df + slack));
        empty |= slo[a] > shi[a];
      }
      if (empty) continue;
      for (int sx = slo[0]; sx <= shi[0]; ++sx)
        for (int sy = slo[1]; sy <= shi[1]; ++sy)
          for (int sz = slo[2]; sz <= shi[2]; ++sz) {
            if (i == j && sx == 0 && sy == 0 && sz == 0) continue;
            // shift = (sx*c0 + sy*c1) + sz*c2, every operation rounded (matches oracle/radius_graph.py)
            double hx = __dadd_rn(__dadd_rn(__dmul_rn(sx, c[0]), __dmul_rn(sy, c[3])), __dmul_rn(sz, c[6]));
            double hy = __dadd_rn(__dadd_rn(__dmul_rn(sx, c[1]), __dmul_rn(sy, c[4])), __dmul_rn(sz, c[7]));
            double hz = __dadd_rn(__dadd_rn(__dmul_rn(sx, c[2]), __dmul_rn(sy, c[5])), __dmul_rn(sz, c[8]));
            double vx = __dadd_rn(bx, hx), vy = __dadd_rn(by, hy), vz = __dadd_rn(bz, hz);
            double d2 = __dadd_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)), __dmul_rn(vz, vz));
            if (d2 < c2) {
              if (FILL && base + cnt < cand_cap) {   // cand_cap may be a caller-promised count (captured steps)
                csrc[base + cnt] = i;
                cshift[3 * (int64_t)(base + cnt)] = sx;
                cshift[3 * (int64_t)(base + cnt) + 1] = sy;
                cshift[3 * (int64_t)(base + cnt) + 2] = sz;
                clen[base + cnt] = __dsqrt_rn(d2);
              }
              ++cnt;
            }
          }
    }
    if (!FILL) {
      count[j] = cnt;
    } else {
      // sort this target's candidates by (len, src, S): insertion sort, segments are short
      if (base + cnt > cand_cap) cnt = cand_cap > base ? (int)(cand_cap - base) : 0;
      for (int a = 1; a < cnt; ++a) {
        PbcCand v{clen[base + a], csrc[base + a], cshift[3 * (int64_t)(base + a)], cshift[3 * (int64_t)(base + a) + 1],
                  cshift[3 * (int64_t)(base + a) + 2]};
        int b = a - 1;
        while (b >= 0) {
          PbcCand w{clen[base + b], csrc[base + b], cshift[3 * (int64_t)(base + b)], cshift[3 * (int64_t)(base + b) + 1],
                    cshift[3 * (int64_t)(base + b) + 2]};
          if (!cand_less(v, w)) break;
          clen[base + b + 1] = w.len; csrc[base + b + 1] = w.src;
          cshift[3 * (int64_t)(base + b + 1)] = w.sx; cshift[3 * (int64_t)(base + b + 1) + 1] = w.sy; cshift[3 * (int64_t)(base + b + 1) + 2] = w.sz;
          --b;
        }
        clen[base + b + 1] = v.len; csrc[base + b + 1] = v.src;
        cshift[3 * (int64_t)(base + b + 1)] = v.sx; cshift[3 * (int64_t)(base + b + 1) + 1] = v.sy; cshift[3 * (int64_t)(base + b + 1) + 2] = v.sz;
      }
    }
  }
}

__global__ void radius_pbc_emit_kernel(const int32_t* __restrict__ gptr, const double* __restrict__ cell, int n, int g,
                                       const int32_t* __restrict__ candptr, const int32_t* __restrict__ csrc,
                                       const int32_t* __restrict__ cshift, int maxn, const int32_t* __restrict__ outptr,
                                       int64_t e, int64_t* __restrict__ ei, int32_t* __restrict__ cell_shift,
                                       void* __restrict__ edge_shifts, int sh64) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int k = find_graph(gptr, g, j);
    const double* c = cell + 9 * k;
    const int cb = candptr[j];
    const int ob = outptr[j], m = outptr[j + 1] - ob;
    for (int t = 0; t < m; ++t) {
      const int64_t o = ob + t;
      if (o >= e) break;                       // e may be a caller-promised count (captured steps)
      ei[o] = csrc[cb + t];
      ei[e + o] = j;
      const int sx = cshift[3 * (int64_t)(cb + t)], sy = cshift[3 * (int64_t)(cb + t) + 1], sz = cshift[3 * (int64_t)(cb + t) + 2];
      cell_shift[3 * o] = sx; cell_shift[3 * o + 1] = sy; cell_shift[3 * o + 2] = sz;
      for (int a = 0; a < 3; ++a) {
        double h = __dadd_rn(__dadd_rn(__dmul_rn(sx, c[a]), __dmul_rn(sy, c[3 + a])), __dmul_rn(sz, c[6 + a]));
        if (sh64) ((double*)edge_shifts)[3 * o + a] = h; else ((float*)edge_shifts)[3 * o + a] = (float)h;
      }
    }
  }
}

extern "C" int hgb_radius_pbc_range(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr, const double* cell,
                                    const int32_t* pbc, const double* cutoff, int32_t n, int32_t g, int32_t* nimg,
                                    hgb_stream_t stream) {
  HGB_REQUIRE(g >= 0 && cell && pbc && cutoff && nimg, "radius_pbc_range: bad arguments");
  if (g == 0) return HGB_OK;
  pbc_range_kernel<<<g, 128, 0, (cudaStream_t)stream>>>(pos, pos_is_f64, graph_ptr, cell, pbc, cutoff, g, nimg);
  HGB_LAUNCH_CHECK("pbc_range");
  return HGB_OK;
}

extern "C" int hgb_radius_pbc_count(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr, const double* cell,
                                    const int32_t* nimg, const double* cutoff, int32_t n, int32_t g,
                                    int32_t* cand_count, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && cell && nimg && cutoff && cand_count, "radius_pbc_count: bad arguments");
  if (n == 0) return HGB_OK;
  radius_pbc_kernel<false><<<hgb_grid_for(n, 64), 64, 0, (cudaStream_t)stream>>>(
      pos, pos_is_f64, graph_ptr, cell, nimg, cutoff, n, g, cand_count, nullptr, 0, nullptr, nullptr, nullptr);
  HGB_LAUNCH_CHECK("radius_pbc_count");
  return HGB_OK;
}

extern "C" int hgb_radius_pbc_fill(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr, const double* cell,
                                   const int32_t* nimg, const double* cutoff, int32_t n, int32_t g,
                                   const int32_t* candptr, int64_t cand_capacity, int32_t* cand_src, int32_t* cand_shift,
                                   double* cand_len, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && candptr && cand_src && cand_shift && cand_len, "radius_pbc_fill: bad arguments");
  if (n == 0) return HGB_OK;
  radius_pbc_kernel<true><<<hgb_grid_for(n, 64), 64, 0, (cudaStream_t)stream>>>(
      pos, pos_is_f64, graph_ptr, cell, nimg, cutoff, n, g, nullptr, candptr, cand_capacity, cand_src, cand_shift, cand_len);
  HGB_LAUNCH_CHECK("radius_pbc_fill");
  return HGB_OK;
}

extern "C" int hgb_radius_pbc_emit(const int32_t* graph_ptr, const double* cell, int32_t n, int32_t g,
                                   const int32_t* candptr, const int32_t* cand_src, const int32_t* cand_shift,
                                   int32_t max_neighbors, const int32_t* outptr, int64_t e, int64_t* edge_index,
                                   int32_t* cell_shift, void* edge_shifts, int32_t shifts_is_f64, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && candptr && outptr, "radius_pbc_emit: bad arguments");
  if (n == 0 || e == 0) return HGB_OK;
  radius_pbc_emit_kernel<<<hgb_grid_for(n, 128), 128, 0, (cudaStream_t)stream>>>(
      graph_ptr, cell, n, g, candptr, cand_src, cand_shift, max_neighbors, outptr, e, edge_index, cell_shift,
      edge_shifts, shifts_is_f64);
  HGB_LAUNCH_CHECK("radius_pbc_emit");
  return HGB_OK;
}

// Degrees of a capacity-sized periodic build: deg[j] = min(count[j], k, cand_cap - candptr[j]) (at least 0), so that
// hgb_radius_pbc_emit reads no candidate past the cand_cap that hgb_radius_pbc_fill wrote; guard bit 1 when the candidates
// overflowed (some target's list is then cut short even if the edges fit).
__global__ void pbc_cap_degree_kernel(const int32_t* __restrict__ count, const int32_t* __restrict__ candptr, int n, int32_t k,
                                      int64_t cand_cap, int32_t* __restrict__ deg, int32_t* __restrict__ flag) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && candptr[n] > cand_cap) atomicOr(flag, 1);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int64_t room = cand_cap - candptr[j];
    int d = count[j] < k ? count[j] : k;
    if (room < d) d = room > 0 ? (int)room : 0;
    deg[j] = d;
  }
}
extern "C" int hgb_radius_pbc_cap_degree(const int32_t* cand_count, const int32_t* candptr, int32_t n, int32_t max_neighbors,
                                         int64_t cand_capacity, int32_t* deg, int32_t* flag, hgb_stream_t stream) {
  HGB_REQUIRE(n >= 0 && max_neighbors >= 0 && cand_capacity >= 0 && candptr && flag && (n == 0 || (cand_count && deg)),
              "radius_pbc_cap_degree: bad arguments");
  pbc_cap_degree_kernel<<<hgb_grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(cand_count, candptr, n, max_neighbors,
                                                                                 cand_capacity, deg, flag);
  HGB_LAUNCH_CHECK("radius_pbc_cap_degree");
  return HGB_OK;
}

// zero rows [min(*e_real, e_cap), e_cap) of cell_shift [e_cap, 3] int32 and edge_shifts [e_cap, 3] (the dummy edges' shifts);
// guard bit 1 when the edges overflowed
__global__ void pbc_zero_tail_kernel(const int32_t* __restrict__ e_real, int64_t e_cap, int32_t* __restrict__ cell_shift,
                                     void* __restrict__ edge_shifts, int sh64, int32_t* __restrict__ flag) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && e_real[0] > e_cap) atomicOr(flag, 1);
  const int64_t lo = 3 * min((int64_t)e_real[0], e_cap);
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < 3 * e_cap; i += (int64_t)gridDim.x * blockDim.x) {
    cell_shift[i] = 0;
    if (sh64) ((double*)edge_shifts)[i] = 0.0; else ((float*)edge_shifts)[i] = 0.f;
  }
}
extern "C" int hgb_radius_pbc_zero_tail(const int32_t* e_real, int64_t e_cap, int32_t* cell_shift, void* edge_shifts,
                                        int32_t shifts_is_f64, int32_t* flag, hgb_stream_t stream) {
  HGB_REQUIRE(e_real && flag && e_cap >= 0 && (e_cap == 0 || (cell_shift && edge_shifts)), "radius_pbc_zero_tail: bad arguments");
  pbc_zero_tail_kernel<<<hgb_grid_for(3 * e_cap, 256), 256, 0, (cudaStream_t)stream>>>(e_real, e_cap, cell_shift, edge_shifts,
                                                                                       shifts_is_f64, flag);
  HGB_LAUNCH_CHECK("radius_pbc_zero_tail");
  return HGB_OK;
}

// out[i] = min(in[i], cap)   (degree after the nearest-k truncation)
__global__ void clamp_i32_kernel(const int32_t* __restrict__ in, int32_t cap, int64_t n, int32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = in[i] < cap ? in[i] : cap;
}
extern "C" int hgb_clamp_i32(const int32_t* in, int32_t cap, int64_t n, int32_t* out, hgb_stream_t stream) {
  if (n == 0) return HGB_OK;
  clamp_i32_kernel<<<hgb_grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(in, cap, n, out);
  HGB_LAUNCH_CHECK("clamp_i32");
  return HGB_OK;
}

// Device-side guard for captured steps that size their outputs from an earlier run of the same shape: *flag |= bit when
// *value != expected (read back asynchronously by the host; see hydragnn_b200/ops.py::check_guard).
__global__ void expect_i32_kernel(const int32_t* __restrict__ value, int32_t expected, int32_t bit, int32_t* __restrict__ flag) {
  if (*value != expected) atomicOr(flag, bit);
}
extern "C" int hgb_expect_i32(const int32_t* value, int32_t expected, int32_t bit, int32_t* flag, hgb_stream_t stream) {
  HGB_REQUIRE(value && flag, "expect_i32: bad arguments");
  expect_i32_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(value, expected, bit, flag);
  HGB_LAUNCH_CHECK("expect_i32");
  return HGB_OK;
}

// dummy edges between consecutive filler nodes for the unused tail of a capacity-padded edge list
__global__ void pad_edges_kernel(const int32_t* __restrict__ e_real, const int32_t* __restrict__ n_real, int n_cap, int64_t e_cap,
                                 int64_t* __restrict__ ei, int32_t* __restrict__ flag) {
  const int64_t er = e_real[0];
  const int nr = n_real[0];
  const int p = n_cap - nr;                       // filler nodes (the host guarantees >= 2)
  if (blockIdx.x == 0 && threadIdx.x == 0 && (er > e_cap || p < 2)) atomicOr(flag, 1);
  if (p < 2) return;
  for (int64_t m = er + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < e_cap; m += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)((m - er) % p);
    ei[m] = nr + k;                               // source
    ei[e_cap + m] = nr + (k + 1) % p;             // target
  }
}
extern "C" int hgb_pad_edges(const int32_t* e_real, const int32_t* n_real, int32_t n_cap, int64_t e_cap, int64_t* edge_index,
                             int32_t* flag, hgb_stream_t stream) {
  HGB_REQUIRE(e_real && n_real && edge_index && flag && n_cap >= 2 && e_cap >= 0, "pad_edges: bad arguments");
  if (e_cap == 0) return HGB_OK;
  pad_edges_kernel<<<hgb_grid_for(e_cap / 8 + 1, 256), 256, 0, (cudaStream_t)stream>>>(e_real, n_real, n_cap, e_cap, edge_index, flag);
  HGB_LAUNCH_CHECK("pad_edges");
  return HGB_OK;
}
