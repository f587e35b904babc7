/* hgb.h -- C-ABI of libhgb.so, the sm_90a (H100) hot-path library of hydragnn-b200.
 *
 * The reference (ORNL/HydraGNN) is 100 % Python and has no FFI boundary of its own: every
 * GPU instruction on its hot path is issued by ATen or a third-party wheel (torch_scatter,
 * torch_cluster, PyG).  Each entry point below therefore cites the *reference call site* (or
 * third-party kernel it reaches) that it replaces, file:line relative to the reference tree.
 *
 * Conventions
 *   - plain C: raw DEVICE pointers into caller-owned buffers, sizes, a cudaStream_t.  No torch
 *     types, no allocation, no retained pointers, no global mutable state, no implicit
 *     synchronisation: every call only enqueues work on `stream`.
 *   - every function returns HGB_OK (0) or a negative HGB_E* code; hgb_last_error() returns a
 *     thread-local message for the last failure on the calling thread.
 *   - matrices are dense row-major fp32 unless stated; index arrays handed over by the host
 *     framework are int64 (PyG convention), internal ones int32.
 *   - reductions are deterministic (fixed summation order given the same inputs).
 */
#ifndef HGB_H
#define HGB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* hgb_stream_t; /* cudaStream_t */

#define HGB_OK 0
#define HGB_EINVAL (-1)
#define HGB_ECUDA (-2)
#define HGB_ECAPACITY (-3)

/* activation codes (hydragnn/utils/model/model.py:30-46 plus the ones hard-wired in the stacks) */
#define HGB_ACT_DERIV 100 /* not an activation: "the tensor already holds act'(.)" (hgb_tc_linear, hgb_act_bwd) */
#define HGB_ACT_NONE 0
#define HGB_ACT_RELU 1
#define HGB_ACT_SILU 2
#define HGB_ACT_TANH 3
#define HGB_ACT_SIGMOID 4
#define HGB_ACT_LRELU 5 /* slope in `act_param` */
#define HGB_ACT_ELU 6
#define HGB_ACT_SELU 7

/* pooling codes (hydragnn/models/Base.py:147-170) */
#define HGB_POOL_ADD 0
#define HGB_POOL_MEAN 1
#define HGB_POOL_MAX 2

int hgb_version(void);
const char* hgb_last_error(void);
/* number of kernels this library has launched from the calling process (bench.py gpu_launches) */
int64_t hgb_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Graph construction
 * ------------------------------------------------------------------------------------------ */

/* Replaces torch_cluster.radius_graph reached through PyG RadiusGraph
 * (hydragnn/preprocess/graph_samples_checks_and_updates.py:112-117,128-133).
 * pos [n,3] fp32, graph_ptr [g+1] int32 (nodes of graph k are graph_ptr[k]..graph_ptr[k+1]).
 * Pass 1 writes deg [n] (in-degree of every query/target node after the max_neighbors cap).  */
int hgb_radius_graph_count(const float* pos, const int32_t* graph_ptr, int32_t n, int32_t g,
                           float r, int32_t max_neighbors, int32_t loop, int32_t* deg,
                           hgb_stream_t stream);
/* Pass 2: rowptr [n+1] = exclusive scan of deg; writes edge_index [2,e] int64
 * (row 0 = neighbour/source, row 1 = query/target; grouped by target ascending, sources ascending). */
int hgb_radius_graph_fill(const float* pos, const int32_t* graph_ptr, int32_t n, int32_t g, float r,
                          int32_t max_neighbors, int32_t loop, const int32_t* rowptr, int64_t e,
                          int64_t* edge_index, hgb_stream_t stream);

/* Periodic variant: replaces RadiusGraphPBC.__call__ (graph_samples...py:149-256: vesin neighbour
 * list + _limit_neighbors nearest-k) for a whole batch.  pos [n,3] fp32 or fp64 (pos_is_f64),
 * cell [g,3,3] fp64 (rows are lattice vectors), pbc [g,3] int32, cutoff [g] fp64 (per-graph so the
 * caller can run the reference's radius-growth retry).  Distances are evaluated in fp64 as the
 * reference does (vesin works in double).
 * Pass 0: nimg [g,3] = number of periodic images to scan along each lattice vector.               */
int hgb_radius_pbc_range(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr,
                         const double* cell, const int32_t* pbc, const double* cutoff, int32_t n,
                         int32_t g, int32_t* nimg, hgb_stream_t stream);
/* Pass 1 counts all candidates (src, S) per target node (no cap yet).                            */
int hgb_radius_pbc_count(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr,
                         const double* cell, const int32_t* nimg, const double* cutoff, int32_t n,
                         int32_t g, int32_t* cand_count, hgb_stream_t stream);
/* Pass 2: candptr [n+1] = exclusive scan of cand_count; fills cand_src [c] int32, cand_shift [c,3]
 * int32, cand_len [c] fp64 and sorts every target's segment by (len, src, Sx, Sy, Sz).
 * cand_capacity = c, the number of entries the three buffers hold (nothing is written past it).   */
int hgb_radius_pbc_fill(const void* pos, int32_t pos_is_f64, const int32_t* graph_ptr,
                        const double* cell, const int32_t* nimg, const double* cutoff, int32_t n,
                        int32_t g, const int32_t* candptr, int64_t cand_capacity, int32_t* cand_src,
                        int32_t* cand_shift, double* cand_len, hgb_stream_t stream);
/* Pass 3: keeps the first min(count, max_neighbors) candidates of every target.  outptr [n+1] =
 * exclusive scan of min(cand_count, max_neighbors) (hgb_clamp_i32 + scan).  Writes edge_index
 * [2,e] int64 (src; dst), cell_shift [e,3] int32 and edge_shifts [e,3] fp32/fp64 = S @ cell
 * (graph_samples...py:239-247).                                                                   */
int hgb_radius_pbc_emit(const int32_t* graph_ptr, const double* cell, int32_t n, int32_t g,
                        const int32_t* candptr, const int32_t* cand_src, const int32_t* cand_shift,
                        int32_t max_neighbors, const int32_t* outptr, int64_t e, int64_t* edge_index,
                        int32_t* cell_shift, void* edge_shifts, int32_t shifts_is_f64,
                        hgb_stream_t stream);
/* out[i] = min(in[i], cap) */
int hgb_clamp_i32(const int32_t* in, int32_t cap, int64_t n, int32_t* out, hgb_stream_t stream);
/* Capacity padding of a captured neighbour build (hydragnn_b200/padded.py): edge_index [2, e_cap] holds *e_real real
 * edges (written by hgb_radius_graph_fill with e = e_cap); slots [*e_real, e_cap) are filled with dummy edges between
 * consecutive FILLER nodes n_real .. n_cap-1 (atoms of the masked filler graphs), so every kernel of the step runs on
 * static shapes.  Sets guard bit 1 in *flag when *e_real > e_cap.                                                       */
int hgb_pad_edges(const int32_t* e_real, const int32_t* n_real, int32_t n_cap, int64_t e_cap, int64_t* edge_index,
                  int32_t* flag, hgb_stream_t stream);
/* Device-side guard for CUDA-graph-captured steps whose output sizes were promised by the caller
 * (edge counts measured on an earlier run): *flag |= bit when *value != expected.  The host reads
 * the flag asynchronously (hydragnn_b200.ops.check_guard); replaces the host read of the count at
 * graph_samples_checks_and_updates.py:128-133 that a captured step cannot do.                      */
int hgb_expect_i32(const int32_t* value, int32_t expected, int32_t bit, int32_t* flag,
                   hgb_stream_t stream);

/* exclusive prefix sum of int32 (out has n+1 entries, out[n] = total).  workspace: >= 4*(n/1024+2) bytes */
int hgb_exclusive_scan_i32(const int32_t* in, int32_t* out, int64_t n, void* workspace,
                           hgb_stream_t stream);
int64_t hgb_exclusive_scan_workspace_bytes(int64_t n);

/* Builds a CSR view of an arbitrary index vector: rowptr [n+1], perm [e] such that the edges whose
 * idx == k are perm[rowptr[k] .. rowptr[k+1]) in ascending edge id (stable).  Also writes idx32 [e].
 * This is what lets every scatter of the reference (ATen scatter_add_/index_add_,
 * hydragnn/models/EGCLStack.py:294-300, hydragnn/models/PAINNStack.py:263-266) run as an
 * atomics-free segmented reduction.  workspace: hgb_csr_workspace_bytes(e, n).
 * guard_flag (optional, device int32): bit 2 is OR-ed in when an entry lies outside [0, n) (such
 * entries are counted under node 0 so that nothing is written out of bounds).                      */
int hgb_csr_build(const int64_t* idx, int64_t e, int32_t n, int32_t* idx32, int32_t* rowptr,
                  int32_t* perm, int32_t* guard_flag, void* workspace, hgb_stream_t stream);
int64_t hgb_csr_workspace_bytes(int64_t e, int32_t n);
/* The same CSR view for index vectors that are GROUPED by graph (what the radius-graph kernels of this library emit: edges
 * sorted by target, graph k's edges = [edge_ptr[node_ptr[k]], edge_ptr[node_ptr[k+1]]) and referencing only its own nodes):
 * one warp per graph fills the segments in ascending edge id with warp-level ranking -- no sort.  node_ptr [g+1], edge_ptr [n+1]. */
int hgb_csr_build_grouped(const int64_t* idx, int64_t e, int32_t n, const int32_t* node_ptr, const int32_t* edge_ptr,
                          int32_t g, int32_t* idx32, int32_t* rowptr, int32_t* perm, int32_t* guard_flag,
                          void* workspace, hgb_stream_t stream);
int64_t hgb_csr_grouped_workspace_bytes(int64_t e, int32_t n);
/* out[p] = idx[perm[p]]: the neighbour node of every CSR slot */
int hgb_gather_i32(const int32_t* idx, const int32_t* perm, int64_t e, int32_t* out, hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Gather / segmented reductions (mutual adjoints)
 * ------------------------------------------------------------------------------------------ */

/* out[e, :] = x[idx[e], :]      -- aten::index at hydragnn/models/EGCLStack.py:284 etc. */
int hgb_gather_rows(const float* x, const int32_t* idx, int64_t e, int32_t c, float* out,
                    hgb_stream_t stream);
/* out[k, :] = sum over p in [rowptr[k], rowptr[k+1]) of m[perm[p], :]   (perm may be NULL = identity)
 * -- ATen scatter_add_ / index_add_ / torch_scatter.scatter_add.  Algorithmic bytes:
 * E*C*4 + E*4 + N*C*4 (SURVEY 8d "scatter primitive").                                          */
int hgb_segment_sum(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c,
                    float* out, hgb_stream_t stream);
/* the same with an output row stride ldo >= c (writes a column block of a wider matrix) */
int hgb_segment_sum_strided(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n,
                            int32_t c, float* out, int32_t ldo, hgb_stream_t stream);
/* PNA min / max aggregators (PyG DegreeScalerAggregation, hydragnn/models/PNAEqStack.py:396-400): for every
 * (segment, channel) the EDGE id of the minimum / maximum (first wins on ties, -1 for an empty segment); the
 * values and their gradients are gathers at those ids.  argmin / argmax are [n,c] int64.                    */
int hgb_segment_argminmax(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c,
                          int64_t* argmin, int64_t* argmax, hgb_stream_t stream);
/* graph pooling over sorted `batch` (graph_ptr [g+1]); mode HGB_POOL_*.  argmax [g,c] int32 is
 * written for HGB_POOL_MAX (may be NULL otherwise).  -- PyG global_*_pool, Base.py:147-170.     */
int hgb_pool_fwd(const float* x, const int32_t* graph_ptr, int32_t g, int32_t c, int32_t mode,
                 float* out, int32_t* argmax, hgb_stream_t stream);
int hgb_pool_bwd(const float* gout, const int32_t* graph_ptr, const int32_t* argmax, int32_t n,
                 int32_t g, int32_t c, int32_t mode, float* gx, hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Dense layers: the cuBLAS call sites behind every nn.Linear of the path -- hydragnn/models/EGCLStack.py:207-240
 * (edge / node / coord MLPs), hydragnn/models/PAINNStack.py:92-98,204-218,281-296 (embeddings, message and update
 * MLPs), hydragnn/models/Base.py:604-663,929-940 (shared layers, heads, MLPNode), mace_utils/modules/blocks.py:61-89,
 * 307-367 (o3.Linear, radial MLP)
 * ------------------------------------------------------------------------------------------ */

/* C[m,n] = op(A) . op(B); op = transpose when the flag is set; lda/ldb/ldc are row strides.
 * beta_one != 0 accumulates into C.  workspace (split-K partials): hgb_gemm_workspace_bytes.     */
int hgb_gemm(const float* a, const float* b, float* c, int32_t m, int32_t n, int32_t k,
             int32_t trans_a, int32_t trans_b, int64_t lda, int64_t ldb, int64_t ldc, int32_t beta_one,
             void* workspace, int64_t workspace_bytes, hgb_stream_t stream);
int64_t hgb_gemm_workspace_bytes(int32_t m, int32_t n, int32_t k, int32_t trans_a);
/* y = act(x . W^T + b); x [m,k] with row stride ldx, W [n,k] with row stride ldw (so a column block
 * of a wider weight matrix can be applied without a copy), b [n] or NULL, y [m,n] dense; z
 * (pre-activation, dense [m,n]) is written when non-NULL (needed by the SiLU backward).           */
int hgb_linear_fwd(const float* x, const float* w, const float* b, int32_t m, int32_t n, int32_t k,
                   int64_t ldx, int64_t ldw, int32_t act, float act_param, float* y, float* z,
                   hgb_stream_t stream);
/* Tiny-K (k <= 8, n <= 256) linear layers: the reference's first PaiNN layer runs at node_size = input_dim
 * (quirk Q4, hydragnn/models/PAINNStack.py:81-87), so Linear(1->F), Linear(2->1) ... appear at M = nodes.
 * fwd: y = act(x W^T + b).  bwd: ONE pass over (dy, y|z, x) applies act', writes dx [m,k] (optional) and
 * reduces dW [n,k] / db [n] deterministically (no dz tensor is materialised).                                 */
int hgb_linear_smallk_supported(int32_t n, int32_t k);
int hgb_linear_smallk_fwd(const float* x, int64_t ldx, const float* w, int64_t ldw, const float* b, int32_t m,
                          int32_t n, int32_t k, int32_t act, float act_param, float* y, float* z,
                          hgb_stream_t stream);
int hgb_linear_smallk_bwd(const float* dy, const float* y, const float* z, const float* x, int64_t ldx,
                          const float* w, int64_t ldw, int32_t m, int32_t n, int32_t k, int32_t act,
                          float act_param, float* dx, float* dw, int64_t lddw, float* db, void* workspace,
                          hgb_stream_t stream);
int64_t hgb_linear_smallk_bwd_workspace_bytes(int32_t m, int32_t n, int32_t k);

/* Tensor-core (wgmma TF32, register accumulators, TMA-fed) versions of the same dense layers for the
 * large-M shapes of the node / edge MLPs: m >= 128, n_out and k_red multiples of 32 and <= 256.  Used under
 * precision="bf16" (TF32 products, fp32 accumulation: tighter than the bf16 autocast of the reference).
 * y[m,n_out] = act(a[m,k_red] . B^T + bias) with B(r,c) = w[r,c] (trans_b = 0: forward, w is [n_out,k_red])
 * or B(r,c) = w[c,r] (trans_b = 1: the data gradient dX = dZ . W, w is [k_red,n_out]).  `addend` [m,n_out]
 * (optional) is added after the activation: gradient accumulation without an extra pass.  `gsrc` [m,n_out]
 * (optional): the result is multiplied by act'(gsrc) with activation code `gact` -- the GEMM is then the data
 * gradient THROUGH the activation that produced this layer's input (gsrc = its saved pre-activation for SiLU,
 * its output for the others; gact = HGB_ACT_DERIV: gsrc already holds act'), which removes the separate
 * activation-backward pass.  Forward calls with gsrc = NULL, gact = HGB_ACT_DERIV, act = SiLU and z != NULL store
 * silu'(pre-activation) in z instead of the pre-activation.  n_out, k_red up to 1024 are cut into <= 256 pieces.
 * exact != 0: fp32-accurate mode for the fp32 configs -- every operand is split in shared memory into a TF32 hi / lo
 * pair (three producer-side warps split each A stage as the TMA lands it) and each k-step issues hi*hi + lo*hi + hi*lo
 * ("3xTF32", error ~1e-6 relative against fp64, tests/test_gpu_round2.py).                                             */
int hgb_tc_linear_supported(int32_t m, int32_t n_out, int32_t k_red);
int hgb_tc_linear(const float* a, int64_t lda, const float* w, int64_t ldw, int32_t trans_b, const float* bias,
                  int32_t m, int32_t n_out, int32_t k_red, int32_t act, float act_param, float* y, float* z,
                  const float* addend, const float* gsrc, int32_t gact, int32_t exact, hgb_stream_t stream);
/* dw[n_out,k_out] (row stride lddw) (+)= dz[m,n_out]^T . x[m,k_out] and db[n_out] (+)= column sums of dz
 * (db may be NULL) in one pass: row slabs of both operands arrive by TMA and are transposed to K-major in shared
 * memory, the bias gradient rides along as extra all-ones rows of the B operand.  Deterministic two-stage reduce.
 * exact = 1: fp32-accurate (both operands split into TF32 hi / lo twins during the transposition, three products per
 * k-step, the register accumulators folded into the partial every 256 rows to keep the chains short); exact = 0:
 * plain TF32.                                                                                                        */
int hgb_tc_wgrad(const float* dz, int64_t lddz, const float* x, int64_t ldx, int32_t m, int32_t n_out,
                 int32_t k_out, float* dw, int64_t lddw, float* db, int32_t accumulate, int32_t exact,
                 void* workspace, int64_t workspace_bytes, hgb_stream_t stream);
int64_t hgb_tc_wgrad_workspace_bytes(int32_t n_out, int32_t k_out);
/* dz = dy * act'(.) evaluated from y (or from z for SiLU, which must then be non-NULL).           */
int hgb_act_bwd(const float* dy, const float* y, const float* z, int64_t count, int32_t act,
                float act_param, float* dz, hgb_stream_t stream);
/* elementwise activation value (order 0) or its order-th derivative (1..2) at x                   */
int hgb_act_deriv(const float* x, int64_t count, int32_t act, float act_param, int32_t order,
                  float* out, hgb_stream_t stream);
/* out[j] = sum_i x[i, j]  (bias gradient).  workspace: hgb_colsum_workspace_bytes(m, n).          */
int hgb_colsum(const float* x, int32_t m, int32_t n, float* out, void* workspace, hgb_stream_t stream);
int64_t hgb_colsum_workspace_bytes(int32_t m, int32_t n);

/* ------------------------------------------------------------------------------------------
 * Edge geometry  (hydragnn/utils/model/operations.py:21-36 and the RBF / cutoff chains of
 * hydragnn/models/PAINNStack.py:331-352)
 * ------------------------------------------------------------------------------------------ */

/* vec = pos[col] - pos[row] + shift; len = |vec|; unit = vec / (len + eps).  Any output may be NULL. */
int hgb_edge_geom_fwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts,
                      int64_t e, float eps, float* vec, float* len, float* unit, hgb_stream_t stream);
/* g_vec = g_vec_in + g_len * vec/len + d(unit)/d(vec)^T g_unit   (NULL gradients are zero).       */
int hgb_edge_geom_bwd(const float* vec, const float* len, float eps, const float* g_vec_in,
                      const float* g_len, const float* g_unit, int64_t e, float* g_vec,
                      hgb_stream_t stream);
/* PaiNN edge embedding: one 48-byte record per edge, epack [e,12] = { sin(n pi d/rc)/d * fcut(d) for n = 1..r
 * (zero padded to 8), fcut(d), dir = unit/len (quirk Q2, PAINNStack.py:257) }.  r <= 8.                     */
int hgb_painn_edge_embed_fwd(const float* unit, const float* len, int64_t e, int32_t r, float cutoff,
                             float* epack, hgb_stream_t stream);
/* backward of the above: g_epack [e,12] -> (g_unit [e,3], g_len [e])                                       */
int hgb_painn_edge_embed_bwd(const float* unit, const float* len, const float* g_epack, int64_t e, int32_t r,
                             float cutoff, float* g_unit, float* g_len, hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * PaiNN  (hydragnn/models/PAINNStack.py:194-328)
 * ------------------------------------------------------------------------------------------ */

/* Fused message: for every node i, over its CSR segment (edges with edge[:,0] == i; nbr [e] holds the source
 * node edge[:,1] of every CSR slot, perm [e] its edge id):
 *   W = Wf . rbfc[e] + bf * fc[e] (* efilt[e]);  f = W * phi[nbr];  (g_v, g_e, m_s) = split(f)
 *   s_out[i] = s[i] + sum m_s;  v_out[i,k] = v[i,k] + sum (v[nbr,k] * g_v + g_e * dir[e,k])
 * Replaces filter GEMM + 2 gathers + 2 index_add_ (PAINNStack.py:239-270); nothing per-edge is written, no
 * atomics, summation in ascending edge id.  Algorithmic bytes: E*(6F*4 + 8 + 48) + N*(8F*4 + 4).
 * phi [n,3f], s [n,f], v [n,3,f], wf [3f,r], bf [3f], efilt [e,3f] or NULL.                                 */
int hgb_painn_message_fwd(const float* phi, const float* s, const float* v, const int32_t* rowptr,
                          const int32_t* perm, const int32_t* nbr, const float* epack, const float* rec,
                          const float* wf, const float* bf, const float* efilt, int32_t n, int32_t f, int32_t r,
                          float* s_out, float* v_out, hgb_stream_t stream);
/* CSR-ordered 64-byte edge records rec [e,16] = { epack[perm[p]] (12), nbr[p] (int bits), perm[p] (int bits), 0, 0 }:
 * a node's records are contiguous and carry the gather index.  When `rec` is passed to hgb_painn_message_fwd and
 * f % 64 == 0, the shared-memory-tiled kernel is used: the phi / v rows of 32 consecutive nodes are staged with
 * cp.async.bulk (double buffered) and neighbour rows are gathered from shared memory.                          */
int hgb_painn_edge_records(const float* epack, const int32_t* perm, const int32_t* nbr, int64_t e, float* rec,
                           hgb_stream_t stream);
/* Backward of the fused message, as a segmented reduction over the CSR of edge[:,1] (the gather side);
 * nbr_agg [e] = edge[:,0] of every slot of that CSR.  gs_out [n,f], gv_out [n,3,f] are the incoming gradients.
 * Outputs: gphi [n,3f]; gv [n,3,f] (= gv_out + gathered part; gs_in == gs_out is the caller's); gwf [3f,r],
 * gbf [3f] (via workspace partials); optional g_epack [e,12] (zero-initialised by the caller when f > 64) and
 * g_efilt [e,3f] (iff efilt).  `rec` (optional): by-col CSR edge records -> shared-memory-tiled kernel.       */
int hgb_painn_message_bwd(const float* gs_out, const float* gv_out, const float* phi, const float* v,
                          const int32_t* rowptr_src, const int32_t* perm_src, const int32_t* nbr_agg,
                          const float* epack, const float* rec, const float* wf, const float* bf, const float* efilt, int32_t n,
                          int32_t f, int32_t r, float* gphi, float* gv, float* gwf, float* gbf, float* g_epack,
                          float* g_efilt, void* workspace, int64_t workspace_bytes, hgb_stream_t stream);
int64_t hgb_painn_message_bwd_workspace_bytes(int32_t n, int32_t f, int32_t r);

/* Update block glue (PAINNStack.py:298-328).  uv, vv are update_U(v), update_V(v) as [3n, f] matrices with row
 * stride `ld` (ld = f: two separate tensors; ld = 2f: the two halves of ONE [3n, 2f] matrix produced by a single
 * GEMM against the stacked weights [U; V]); guv / gvv use the same stride.
 * pre:  mlp_in [n,2f] = [ |vv| over the 3 components , s ]                                        */
int hgb_painn_update_pre_fwd(const float* vv, int64_t ld, const float* s, int32_t n, int32_t f, float* mlp_in,
                             hgb_stream_t stream);
/* post: a [n,(2|3)f] from update_mlp.  s_out = s + a_sv * sum_k(uv*vv) + a_ss;
 *       v_out = v + a_vv * uv (skipped when last != 0: a = (a_sv, a_ss), v_out may be NULL)        */
int hgb_painn_update_post_fwd(const float* a, const float* uv, const float* vv, int64_t ld, const float* s,
                              const float* v, int32_t n, int32_t f, int32_t last, float* s_out,
                              float* v_out, hgb_stream_t stream);
/* backward of pre+post in one pass.  Inputs: gs_out, gv_out (NULL when last), g_mlp_in [n,2f]
 * (gradient that came back through update_mlp), a, uv, vv, mlp_in.  Outputs: ga [n,(2|3)f] is
 * produced by *_post_bwd_a (needed before the MLP backward can run), then the rest; gv (optional)
 * receives a copy of gv_out (the direct path), callers may instead hand gv_out to the dgrad as addend.  */
int hgb_painn_update_post_bwd_a(const float* gs_out, const float* gv_out, const float* uv,
                                const float* vv, int64_t ld, int32_t n, int32_t f, int32_t last, float* ga,
                                hgb_stream_t stream);
int hgb_painn_update_bwd(const float* gs_out, const float* gv_out, const float* g_mlp_in,
                         const float* a, const float* uv, const float* vv, int64_t ld, const float* mlp_in,
                         int32_t n, int32_t f, int32_t last, float* guv, float* gvv, float* gs,
                         float* gv, hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * GPS global attention  (hydragnn/globalAtt/gps.py:126-133; ATen SDPA inside nn.MultiheadAttention)
 * ------------------------------------------------------------------------------------------ */

/* Dense multi-head self-attention over ONE sequence of n tokens (quirk Q1: the reference never passes
 * graph_batch, so the whole mini-batch attends to itself).  qkv [n,3f] is the packed in-projection
 * [q | k | v], head h owns columns h*d..h*d+d-1 (d = f/heads in {1,2,4,8,16,32}); out [n,f]; lse [n,heads]
 * (log-sum-exp of the scaled scores, kept for the backward).  Flash-style: no [n,n] matrix reaches HBM.    */
int hgb_mha_fwd(const float* qkv, int32_t n, int32_t f, int32_t heads, float* out, float* lse,
                hgb_stream_t stream);
int hgb_mha_bwd(const float* qkv, const float* out, const float* lse, const float* gout, int32_t n, int32_t f,
                int32_t heads, float* gqkv, hgb_stream_t stream);

/* The same attention on the tensor cores for head_dim == 8 (the GPS configuration of qm9.json / C5: 64 channels, 8 heads):
 * mma.sync m16n8k8 TF32 with fp32 accumulation; one score block of 16 queries x 8 keys per instruction, the accumulator
 * layout of S re-used as the A operand of P V through a key permutation (no shuffles).  exact != 0: every product as three
 * TF32 products of a hi/lo split (fp32-level accuracy, the fp32 configs); exact == 0: plain TF32 (precision="bf16").
 * delta_ws: n * heads floats of scratch.  Same lse / layout contract as hgb_mha_fwd / hgb_mha_bwd.                       */
int32_t hgb_mha_tc_supported(int32_t f, int32_t heads);
int hgb_mha_tc_fwd(const float* qkv, int32_t n, int32_t f, int32_t heads, int32_t exact, float* out, float* lse,
                   hgb_stream_t stream);
int hgb_mha_tc_bwd(const float* qkv, const float* out, const float* lse, const float* gout, int32_t n, int32_t f,
                   int32_t heads, int32_t exact, float* delta_ws, float* gqkv, hgb_stream_t stream);

/* Closed (any-order differentiable) MACE primitives for the force-training path and for shapes outside the fused first-order
 * kernels (replace the torch.einsum compositions of round 1; hydragnn/utils/model/mace_utils/modules/blocks.py:386-397,
 * symmetric_contraction.py:217-239).  cg [ni, nj, nk]: real coupling tensor of ONE tensor-product path (each <= 7).
 *   tp_path mode 0:  out [e, nk, f] = p2[e, f] * sum_ij cg[i, j, k] p0[e, i, f] p1[e, j]            (a, y, w)
 *           mode 1:  out [e, nj]    = sum_f p2[e, f] sum_ik cg[i, j, k] p0[e, i, f] p1[e, k, f]      (a, g, w)
 *           mode 2:  out [e, f]     = sum_ijk cg[i, j, k] p0[e, i, f] p1[e, j] p2[e, k, f]            (a, y, g)
 *   chan_contract mode 0: out [n, f, p]     = sum_i p0[n, f, p, i] p1[n, i, f]
 *                 mode 1: out [n, f, p, ni] = p0[n, f, p] p1[n, i, f]
 *                 mode 2: out [n, ni, f]    = sum_p p0[n, f, p] p1[n, f, p, i]
 * Each family is closed under differentiation (the derivative of every mode is another mode, possibly with cg permuted).  */
int hgb_mace_tp_path(int32_t mode, const float* p0, const float* p1, const float* p2, const float* cg, int64_t e, int32_t f,
                     int32_t ni, int32_t nj, int32_t nk, float* out, hgb_stream_t stream);
int hgb_mace_chan_contract(int32_t mode, const float* p0, const float* p1, int64_t n, int32_t f, int32_t p, int32_t ni,
                           float* out, hgb_stream_t stream);

/* MACE edge embedding in one pass per edge (SURVEY K2): vec = pos[col] - pos[row] + shift -> real spherical harmonics
 * sh [e, (lmax+1)^2] (component normalisation, e3nn axis convention; MACEStack.py:455-466) and the Bessel basis times the
 * polynomial cutoff radial [e, num_bessel] (mace_utils/modules/radial.py:18-60,110-148; blocks.py:164-177).  lmax <= 3.
 * bwd: g_vec [e, 3] = d L / d vec from g_sh / g_radial (either may be NULL); hgb_edge_vec_scatter turns it into d L / d pos.  */
int hgb_mace_edge_embed_fwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, int64_t e, int32_t lmax,
                            int32_t num_bessel, float r_max, float p, float* sh, float* radial, hgb_stream_t stream);
int hgb_mace_edge_embed_bwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts, const float* g_sh,
                            const float* g_radial, int64_t e, int32_t lmax, int32_t num_bessel, float r_max, float p, float* g_vec,
                            hgb_stream_t stream);

/* Grouped dense layers for multi-branch decoding (hydragnn/models/Base.py:770-780 graph heads, :816-840 node heads,
 * hydragnn/models/MultiTaskModelMP.py): rows sorted by dataset branch, rowptr [groups + 1] on the device, every 64-row tile
 * picks the weight matrix of its group -- one launch per layer instead of a boolean-mask loop over `dataset_name.unique()`.
 * trans_w == 0: y [m, n] = act(x [m, k] W_g^T + b_g), w [groups, n, k], bias [groups, n] (optional), z = pre-activation (optional).
 * trans_w != 0: y [m, n] = x [m, k] W_g with w [groups, k, n] (the data gradient; no bias / act).                          */
int hgb_grouped_linear(const float* x, int64_t ldx, const float* w, const float* bias, const int32_t* rowptr, int32_t groups,
                       int32_t m, int32_t n, int32_t k, int32_t trans_w, int32_t act, float act_param, float* y, float* z,
                       hgb_stream_t stream);
/* dw [groups, n, k] = per-group dy [m, n]^T x [m, k]; db [groups, n] (optional) = per-group column sums of dy */
int hgb_grouped_wgrad(const float* dy, const float* x, int64_t ldx, const int32_t* rowptr, int32_t groups, int32_t m, int32_t n,
                      int32_t k, float* dw, float* db, hgb_stream_t stream);

/* fp32-ACCURATE tensor-core GEMMs for the exact-fp32 mode (nn.Linear forward / dgrad / wgrad of every stack under
 * precision "fp32", e.g. EGCLStack.py:245-263, PNAEqStack.py:326-476, Base.py heads): mma.sync m16n8k8 TF32 with every
 * product expanded into the four products of a hi/lo split and the long sums kept in fp32 registers (csrc/hgb_gemm3.cu).
 * Same operand convention as hgb_gemm; bias / act / z (pre-activation) only for trans_a == 0.
 * hgb_gemm3_supported tells which shapes take this path (large m or a long reduction; everything else stays on hgb_gemm). */
int32_t hgb_gemm3_supported(int32_t m, int32_t n, int32_t k, int32_t trans_a, int32_t trans_b, int64_t lda,
                            int64_t ldb, int64_t ldc);
int64_t hgb_gemm3_workspace_bytes(int32_t m, int32_t n, int32_t k, int32_t trans_a);
int hgb_gemm3(const float* a, const float* b, float* c, int32_t m, int32_t n, int32_t k, int32_t trans_a,
              int32_t trans_b, int64_t lda, int64_t ldb, int64_t ldc, int32_t beta_one, const float* bias,
              int32_t act, float act_param, float* z, void* workspace, hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused EGNN edge block (hydragnn/models/EGCLStack.py:245-258 edge_model, :256-263 the scatter of
 * node_model, :278-291 forward; unsorted_segment_sum :294-300).  The first Linear of edge_mlp is
 * applied per node by the caller: pq [n, 2h] = [x W0[:, :fin]^T | x W0[:, fin:2fin]^T]; the kernels
 * see z1_e = P[row] + Q[col] + s_e w_d + b0 with s_e = |pos[col] - pos[row] + shift| (quirk Q3).
 * CSR = by edge_index[0] (the aggregation index): rowptr [n+1], perm [e] (edge ids), nbr [e] =
 * edge_index[1][perm].  masks [e, 2] uint64 (CSR order): ReLU patterns of z1 and z2, written by the
 * forward and read by every derivative kernel (the block is piecewise linear).  h in {32, 64}.
 * nodes_per_tile in [1, 32]: consecutive nodes per CTA tile (pick ~ 128 / mean degree).
 * ------------------------------------------------------------------------------------------ */
int32_t hgb_egnn_edge_supported(int32_t h);
int64_t hgb_egnn_edge_workspace_bytes(int32_t n, int32_t h, int32_t nodes_per_tile);
/* tangent == 0:  out[i] = sum_{row(e)=i} relu(W1 relu(z1_e) + b1)          (writes masks)
 * tangent != 0:  out[i] = sum_{row(e)=i} mask2 * (W1 (mask1 * (P[row] + Q[col] + s_e w_d)))   (reads masks;
 *                b0 / b1 ignored) -- the JVP of the block, which is the adjoint of hgb_egnn_edge_bwd_data
 *                with respect to its g_out (needed by the force loss, create.py:718-724).                    */
int hgb_egnn_edge_fwd(const float* pq, const float* s, const float* wd, const float* b0, const float* w1,
                      const float* b1, const int32_t* rowptr, const int32_t* perm, const int32_t* nbr,
                      int32_t n, int32_t h, int32_t nodes_per_tile, int32_t tangent, uint64_t* masks,
                      float* out, hgb_stream_t stream);
/* gz1_e = mask1 * (W1^T (mask2 * g_out[row(e)])).  Writes g_p [n, h] (row stride ldp) = sum_{row} gz1,
 * gz1 [e, h] in EDGE order (the caller's by-col segment sum gives g_q), gs [e] = w_d . gz1_e and, when
 * g_wd / g_b0 are given (both or neither), g_wd = sum_e s_e gz1_e and g_b0 = sum_e gz1_e.
 * workspace: hgb_egnn_edge_workspace_bytes.                                                            */
int hgb_egnn_edge_bwd_data(const float* g_out, const float* s, const float* wd, const float* w1,
                           const uint64_t* masks, const int32_t* rowptr, const int32_t* perm, int32_t n,
                           int32_t h, int32_t nodes_per_tile, float* g_p, int32_t ldp, float* gz1, float* gs,
                           float* g_wd, float* g_b0, void* workspace, hgb_stream_t stream);
/* g_w1 [h, h] = sum_e (mask2 * g_out[row]) y_e^T with y_e = relu(z1_e) (tangent == 0) or
 * mask1 * (P[row] + Q[col] + s_e w_d) (tangent != 0); g_b1 [h] (optional) = sum_e mask2 * g_out[row].   */
int hgb_egnn_edge_wgrad(const float* g_out, const float* pq, const float* s, const float* wd, const float* b0,
                        const uint64_t* masks, const int32_t* rowptr, const int32_t* perm, const int32_t* nbr,
                        int32_t n, int32_t h, int32_t nodes_per_tile, int32_t tangent, float* g_w1, float* g_b1,
                        void* workspace, hgb_stream_t stream);
/* out [h] = sum_e w[e] x[e, :]  (h divides 256) */
int hgb_weighted_colsum(const float* x, const float* w, int64_t e, int32_t h, float* out, void* workspace,
                        hgb_stream_t stream);
int64_t hgb_weighted_colsum_workspace_bytes(int32_t h);
/* Closed edge-length primitives for d_e = |pos[col] - pos[row] + shift_e| (operations.py:21-36; the length
 * itself is hgb_edge_geom_fwd).  bwd: gvec_e = gd_e vhat_e.  bwd2 (adjoint of bwd + scatter with respect to
 * gd and pos): w_e = ggpos[col] - ggpos[row]; g_gd_e = <vhat_e, w_e>; q_e = gd_e (w_e - vhat <vhat, w_e>) / d_e.
 * scatter: g_pos[i] = sum_{col(e)=i} gvec_e - sum_{row(e)=i} gvec_e (ordered).                           */
int hgb_edge_len_bwd(const float* pos, const int32_t* row, const int32_t* col, const float* shifts,
                     const float* gd, int64_t e, float* gvec, hgb_stream_t stream);
int hgb_edge_len_bwd2(const float* pos, const int32_t* row, const int32_t* col, const float* shifts,
                      const float* gd, const float* ggpos, int64_t e, float* g_gd, float* q,
                      hgb_stream_t stream);
int hgb_edge_vec_scatter(const float* gvec, const int32_t* col_rowptr, const int32_t* col_perm,
                         const int32_t* row_rowptr, const int32_t* row_perm, int32_t n, float* gpos,
                         hgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Loss / optimizer (hydragnn/train/train_validate_test.py:736-769, torch.optim.AdamW)
 * ------------------------------------------------------------------------------------------ */

/* loss[0] = mean((pred - target)^2) (mode 0) or mean(|pred - target|) (mode 1);
 * gpred = d loss / d pred * gscale.  Single-block deterministic reduction.
 * valid_rows (optional, device int32): capacity-padded batches -- only the first *valid_rows rows of
 * row_width entries are real: the mean runs over them and gpred is zero beyond.                      */
int hgb_loss_fwd_bwd(const float* pred, const float* target, int64_t count, int32_t mode, float gscale,
                     float* loss, float* gpred, const int32_t* valid_rows, int32_t row_width,
                     hgb_stream_t stream);
/* Fused AdamW over one flat parameter buffer: p, g, m, v [count]; `grad_scale` multiplies g first
 * (1/world_size after the flat all-reduce); step is 1-based and read from device (`step_dev`, fp32,
 * incremented by the kernel) so the launch is CUDA-graph capturable.  hyper_dev (optional, device,
 * 2 floats {lr, grad_scale}): when given it overrides the by-value lr / grad_scale, so a captured
 * step follows a learning-rate scheduler (train_validate_test.py:452-476 steps ReduceLROnPlateau). */
int hgb_adamw_step(float* p, const float* g, float* m, float* v, int64_t count, float lr, float beta1,
                   float beta2, float eps, float weight_decay, float grad_scale, float* step_dev,
                   const float* hyper_dev, hgb_stream_t stream);

/* PaiNN update block at node_size == 1 (the reference's first layer runs at width input_dim, quirk Q4): the whole block
 * (PAINNStack.py:298-328) per node in one kernel.  params16 / gparams16 (device, 16 floats): 0 uw, 1 ub, 2 vw, 3 vb,
 * 4 w1[|Vv|], 5 w1[s], 6 b1, 7..9 w2 rows, 10..12 b2 (rows = (a_vv, a_sv, a_ss), or (a_sv, a_ss) when last != 0).
 * s [n], v [n,3]; gv receives the complete gradient w.r.t. v (direct path included).                                     */
int64_t hgb_painn_update_scalar_workspace_bytes(void);
int hgb_painn_update_scalar_fwd(const float* s, const float* v, const float* params16, int32_t n, int32_t last, float* s_out,
                                float* v_out, hgb_stream_t stream);
int hgb_painn_update_scalar_bwd(const float* gs_out, const float* gv_out, const float* s, const float* v, const float* params16,
                                int32_t n, int32_t last, float* gs, float* gv, float* gparams16, void* workspace,
                                hgb_stream_t stream);

/* Linear(1,1) - act - Linear(1,out) with out <= 4 on one scalar per row (scalar_message_mlp of a width-1 PaiNN layer, quirk Q4):
 * params10 / gparams10 (device) = [w1, b1, w2[0..3], b2[0..3]].  x [n], y [n,out]; gx may be NULL.                        */
int64_t hgb_mlp2_scalar_workspace_bytes(void);
int hgb_mlp2_scalar_fwd(const float* x, const float* params10, int32_t n, int32_t out, int32_t act, float act_param, float* y,
                        hgb_stream_t stream);
int hgb_mlp2_scalar_bwd(const float* gy, const float* x, const float* params10, int32_t n, int32_t out, int32_t act,
                        float act_param, float* gx, float* gparams10, void* workspace, hgb_stream_t stream);

/* Device-side collate (SURVEY 8f-1; replaces the index bookkeeping of PyG Batch.from_data_list + move_batch_to_device,
 * hydragnn/preprocess/load_data.py:157-164, train_validate_test.py:74-84): ptr [g+1] = exclusive scan of the per-graph
 * node counts.  batch[i] = graph of node i;  edge_index[:, k] = edge_index_local[:, k] + node_ptr[graph of edge k].      */
int hgb_collate_batch_vector(const int32_t* ptr, int32_t g, int64_t n, int64_t* batch, hgb_stream_t stream);
int hgb_collate_offset_edges(const int64_t* edge_index_local, const int32_t* edge_ptr, const int32_t* node_ptr, int32_t g,
                             int64_t e, int64_t* edge_index, hgb_stream_t stream);

/* PNA aggregation (hydragnn/models/PNAEqStack.py:396-400; torch_geometric 2.6.1 DegreeScalerAggregation with aggregators
 * mean, min, max, std): one pass per CSR segment.  m [e,c] -> out [n,4c] = [mean | min | max | std]; argmin / argmax [n,c]
 * = edge id of the first extremum (-1: empty segment).  Backward: g_m [e,c] from g_out [n,4c]; idx [e] = segment of every edge. */
int hgb_pna_aggregate_fwd(const float* m, const int32_t* rowptr, const int32_t* perm, int32_t n, int32_t c, float* out,
                          int32_t* argmin, int32_t* argmax, hgb_stream_t stream);
int hgb_pna_aggregate_bwd(const float* g_out, const float* m, const float* out, const int32_t* idx, const int32_t* rowptr,
                          const int32_t* argmin, const int32_t* argmax, int64_t e, int32_t c, float* g_m, hgb_stream_t stream);

/* ---- MACE (hydragnn/utils/model/mace_utils/modules/blocks.py:369-402, symmetric_contraction.py:92-242) ------------------
 * Features are channel-last: [N, spherical index, F].  lmax_in <= 2, 1 <= lmax_sh <= 3, lmax_in <= lmax_sh, F % 32 == 0.
 * Path order / coupling constants = tp_out_irreps_with_instructions (irreps_tools.py:15-44) with e3nn's real Wigner 3j.   */

/* number of accumulator rows (sum over output degrees l3 of n_paths(l3) * (2 l3 + 1)); -1 if unsupported.               */
int hgb_mace_tp_num_acc(int32_t lmax_in, int32_t lmax_sh);

/* conv_tp (o3.TensorProduct "uvu", blocks.py:320-327,390) fused with scatter(..., receiver, "sum") (:393-395).
 * up [N,(lmax_in+1)^2,F], sh [E, sh_ld] (first (lmax_sh+1)^2 columns), tpw [E, n_paths*F]; (rowptr, perm, snd): CSR of the
 * receivers with the edge id and the sender of every slot.  out: packed, per output degree l3 a [N, 2l3+1, n_paths(l3)*F]
 * block starting at float offset N*F*acc_base(l3).                                                                      */
int hgb_mace_tp_scatter_fwd(const float* up, const float* sh, const float* tpw, const int32_t* rowptr, const int32_t* perm,
                            const int32_t* snd, int32_t n, int32_t f, int32_t lmax_in, int32_t lmax_sh, int32_t sh_ld, float* out,
                            hgb_stream_t stream);

/* backward: g_tpw [E, n_paths*F], g_up_edge [E,(lmax_in+1)^2,F] (per-edge sender gradients; reduce per sender with
 * hgb_segment_sum), g_sh [E, sh_ld] or NULL (must be zero-filled by the caller when F/64 > 1).                          */
int hgb_mace_tp_scatter_bwd(const float* g_out, const float* up, const float* sh, const float* tpw, const int32_t* rowptr,
                            const int32_t* perm, const int32_t* snd, int32_t n, int32_t f, int32_t lmax_in, int32_t lmax_sh,
                            int32_t sh_ld, float* g_tpw, float* g_up_edge, float* g_sh, hgb_stream_t stream);

/* SymmetricContraction with correlation 2 (symmetric_contraction.py:131-239): weight rows per output degree L are
 * [weights_max (P2(L)), weights.0 (P1(L))], concatenated over L: wall [118, KTOT, F]; z [N] element index (0-based);
 * x [N,(lmax_in+1)^2,F] -> out [N,(lmax_out+1)^2,F].                                                                    */
int hgb_mace_symcontract_num_weights(int32_t lmax_in, int32_t lmax_out);
int hgb_mace_symcontract_fwd(const float* x, const float* wall, const int32_t* z, int32_t n, int32_t f, int32_t lmax_in,
                             int32_t lmax_out, float* out, hgb_stream_t stream);
/* gx [N,(lmax_in+1)^2,F]; gw_node [N,KTOT,F] (per-node weight gradients; reduce per element with hgb_segment_sum).       */
int hgb_mace_symcontract_bwd(const float* g_out, const float* x, const float* wall, const int32_t* z, int32_t n, int32_t f,
                             int32_t lmax_in, int32_t lmax_out, float* gx, float* gw_node, hgb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* HGB_H */
