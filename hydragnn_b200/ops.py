"""torch-facing wrappers of the libhgb.so kernels.

Two layers:

* ``raw_*`` -- thin launchers: check tensors, allocate outputs with torch (device memory + current
  stream are the only things torch provides), call the C-ABI through ctypes.
* ``torch.autograd.Function`` classes.  Two families:
    - primitives that are closed under differentiation (``GatherRows`` <-> ``SegmentSum`` are each
      other's adjoint, ``MatMul``'s backward is ``MatMul``): any-order differentiable, used when the
      force loss needs ``create_graph=True`` (hydragnn/models/create.py:718-724);
    - fused blocks with hand-written first-order backward kernels (``LinearAct``, ``PainnMessageFn``,
      ``PainnUpdateFn``, ``PoolFn``, ``EdgeGeomFn`` ...): the fast path for ordinary training /
      inference.  They are ``once_differentiable``: asking for a second derivative raises.

Nothing here falls back to ATen/PyG scatter kernels; a missing library raises in ``_lib.lib()``.
"""
import os

import torch
from torch.autograd.function import once_differentiable

from . import _lib

ACT_CODES = {None: 0, "none": 0, "relu": 1, "silu": 2, "tanh": 3, "sigmoid": 4, "lrelu": 5, "elu": 6, "selu": 7}
POOL_CODES = {"add": 0, "sum": 0, "mean": 1, "max": 2}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _chk(t, dtype=torch.float32):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("hydragnn_b200 ops need CUDA tensors (no CPU fallback on the hot path)")
    if t.dtype != dtype:
        raise RuntimeError("expected %s, got %s" % (dtype, t.dtype))
    return t if t.is_contiguous() else t.contiguous()


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


# =====================================================================================================
# graph plan: int32 indices + CSR views of both rows of edge_index
# =====================================================================================================
class Csr:
    """CSR view of an index vector: the entries equal to k are ``perm[rowptr[k]:rowptr[k+1]]`` (ascending)."""
    __slots__ = ("idx", "rowptr", "perm", "n")

    def __init__(self, idx, rowptr, perm, n):
        self.idx, self.rowptr, self.perm, self.n = idx, rowptr, perm, n


def csr_build(index64, n):
    index64 = _chk(index64, torch.int64)
    e = index64.numel()
    dev = index64.device
    idx32 = torch.empty(e, dtype=torch.int32, device=dev)
    rowptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    perm = torch.empty(e, dtype=torch.int32, device=dev)
    ws = _ws(_lib.query("hgb_csr_workspace_bytes", e, n), dev)
    _lib.call("hgb_csr_build", _p(index64), e, n, _p(idx32), _p(rowptr), _p(perm), _p(guard_flag(dev)), _p(ws), _stream())
    return Csr(idx32, rowptr, perm, n)


def csr_build_grouped(index64, n, node_ptr, edge_ptr, g):
    """``csr_build`` for edges grouped by graph (radius-graph output): sort-free, see hgb_csr_build_grouped."""
    index64 = _chk(index64, torch.int64)
    e = index64.numel()
    dev = index64.device
    idx32 = torch.empty(e, dtype=torch.int32, device=dev)
    rowptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    perm = torch.empty(e, dtype=torch.int32, device=dev)
    ws = _ws(_lib.query("hgb_csr_grouped_workspace_bytes", e, n), dev)
    _lib.call("hgb_csr_build_grouped", _p(index64), e, n, _p(node_ptr), _p(edge_ptr), int(g), _p(idx32), _p(rowptr), _p(perm),
              _p(guard_flag(dev)), _p(ws), _stream())
    return Csr(idx32, rowptr, perm, n)


class EdgePlan:
    """Everything index-shaped a conv layer needs, built once per batch (SURVEY hard part H3: the
    stacks aggregate by ``edge_index[0]`` which is not the sorted row of a PyG radius graph)."""

    def __init__(self, edge_index, num_nodes, col_rowptr=None, graph_ptr=None):
        """``col_rowptr`` [N+1] int32 (optional): the edges are already grouped by ``edge_index[1]`` in ascending order with
        these segment offsets (what the engine's own radius-graph kernels emit) -- that CSR view then needs no build.  With
        ``graph_ptr`` [G+1] int32 as well, the by-source view is filled graph by graph without a sort."""
        ei = _chk(edge_index, torch.int64)
        self.num_nodes, self.num_edges = int(num_nodes), int(ei.shape[1])
        if col_rowptr is not None and graph_ptr is not None and GROUPED_CSR:
            self.by_row = csr_build_grouped(ei[0], self.num_nodes, graph_ptr, col_rowptr, graph_ptr.numel() - 1)
        else:
            self.by_row = csr_build(ei[0], self.num_nodes)
        if col_rowptr is not None:
            self.by_col = Csr(ei[1].to(torch.int32), col_rowptr, torch.arange(self.num_edges, dtype=torch.int32, device=ei.device),
                              self.num_nodes)
        else:
            self.by_col = csr_build(ei[1], self.num_nodes)
        self.row, self.col = self.by_row.idx, self.by_col.idx
        self._nbr = {}

    def nbr(self, which):
        """Neighbour node of every CSR slot: 'row' -> col[by_row.perm] (source of the message summed into row),
        'col' -> row[by_col.perm]."""
        if which not in self._nbr:
            idx, perm = (self.col, self.by_row.perm) if which == "row" else (self.row, self.by_col.perm)
            out = torch.empty_like(perm)
            _lib.call("hgb_gather_i32", _p(idx), _p(perm), perm.numel(), _p(out), _stream())
            self._nbr[which] = out
        return self._nbr[which]


def graph_ptr_from_batch(batch, num_graphs):
    """int32 [G+1] offsets of the (sorted) batch vector -- itself a CSR build with identity perm."""
    return csr_build(batch, num_graphs)


def exclusive_scan(x):
    x = _chk(x, torch.int32)
    out = torch.empty(x.numel() + 1, dtype=torch.int32, device=x.device)
    ws = _ws(_lib.query("hgb_exclusive_scan_workspace_bytes", x.numel()), x.device)
    _lib.call("hgb_exclusive_scan_i32", _p(x), _p(out), x.numel(), _p(ws), _stream())
    return out


# ---- device-side guards of captured steps ---------------------------------------------------------------
GUARD_EDGE_COUNT = 1        # a neighbour build produced a different number of edges / candidates than the captured size
GUARD_BAD_INDEX = 2         # an index vector handed to csr_build had entries outside [0, n)
_GUARD = {}


def guard_flag(device):
    """One int32 error word per device; kernels OR bits into it, ``check_guard`` reads it."""
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _GUARD:
        _GUARD[key] = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", key))
    return _GUARD[key]


def expect_count(value_i32, expected, bit=GUARD_EDGE_COUNT):
    _lib.call("hgb_expect_i32", _p(value_i32), int(expected), int(bit), _p(guard_flag(value_i32.device)), _stream())


def check_guard(device=None):
    """Host read (one sync) of the guard word; raises if a captured step saw a shape it was not captured for."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    word = int(guard_flag(dev).item())
    if word:
        guard_flag(dev).zero_()
        what = []
        if word & GUARD_EDGE_COUNT:
            what.append("a neighbour build produced a different edge count than the one the step was captured with")
        if word & GUARD_BAD_INDEX:
            what.append("an index vector had entries outside [0, n)")
        raise RuntimeError("hydragnn_b200 device guard tripped: " + "; ".join(what))


# =====================================================================================================
# raw launchers
# =====================================================================================================
def raw_gather(x, idx32):
    x = _chk(x)
    c = 1
    for d in x.shape[1:]:
        c *= d
    out = torch.empty((idx32.numel(),) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    _lib.call("hgb_gather_rows", _p(x), _p(idx32), idx32.numel(), c, _p(out), _stream())
    return out


def raw_segment_sum(m, rowptr, perm, n):
    m = _chk(m)
    c = 1
    for d in m.shape[1:]:
        c *= d
    out = torch.empty((n,) + tuple(m.shape[1:]), dtype=m.dtype, device=m.device)
    _lib.call("hgb_segment_sum", _p(m), _p(rowptr), _p(perm), n, c, _p(out), _stream())
    return out


def raw_gemm(a, b, ta, tb, out=None, beta_one=False):
    """op(a) @ op(b) for 2-D row-major (possibly row-strided) operands."""
    # unit inner stride (a one-column matrix may carry any inner stride: it is never used)
    assert a.dim() == 2 and b.dim() == 2 and (a.stride(1) == 1 or a.shape[1] == 1) and (b.stride(1) == 1 or b.shape[1] == 1)
    m, k = (a.shape[1], a.shape[0]) if ta else (a.shape[0], a.shape[1])
    k2, n = (b.shape[1], b.shape[0]) if tb else (b.shape[0], b.shape[1])
    assert k == k2, "gemm inner dimensions differ"
    if out is None:
        out = torch.empty(m, n, dtype=a.dtype, device=a.device)
    if gemm3_ok(a, b, out, m, n, k, ta, tb):
        # fp32-accurate tensor-core path (4xTF32 split products, fp32 register accumulation): csrc/hgb_gemm3.cu
        nbytes = _lib.query("hgb_gemm3_workspace_bytes", m, n, k, int(ta))
        ws = _ws(nbytes, a.device) if nbytes else None
        _lib.call("hgb_gemm3", _p(a), _p(b), _p(out), m, n, k, int(ta), int(tb), a.stride(0), b.stride(0), out.stride(0), int(beta_one),
                  None, 0, 0.0, None, _p(ws), _stream())
        return out
    nbytes = _lib.query("hgb_gemm_workspace_bytes", m, n, k, int(ta))
    ws = _ws(nbytes, a.device) if nbytes else None
    _lib.call("hgb_gemm", _p(a), _p(b), _p(out), m, n, k, int(ta), int(tb), a.stride(0), b.stride(0), out.stride(0),
              int(beta_one), _p(ws), nbytes, _stream())
    return out


GEMM3 = os.environ.get("HGB_GEMM3", "0") == "1"      # 1: exact-fp32 GEMMs on the 4xTF32 mma.sync kernels (csrc/hgb_gemm3.cu); off by
                                                     # default (four legacy-path MMAs per product)


def gemm3_ok(a, b, out, m, n, k, ta, tb):
    if not GEMM3 or a.dtype != torch.float32:
        return False
    if a.data_ptr() % 16 or out.data_ptr() % 16 or (ta and b.data_ptr() % 16):
        return False
    return bool(_lib.query("hgb_gemm3_supported", m, n, k, int(ta), int(tb), a.stride(0), b.stride(0), out.stride(0)))


def raw_colsum(x2d):
    m, n = x2d.shape
    out = torch.empty(n, dtype=x2d.dtype, device=x2d.device)
    ws = _ws(_lib.query("hgb_colsum_workspace_bytes", m, n), x2d.device)
    _lib.call("hgb_colsum", _p(x2d), m, n, _p(out), _p(ws), _stream())
    return out


# ---- tensor-core (wgmma / TF32) dense layers: enabled per model by precision="bf16" -----------------
_TC = {"enabled": False}
_DATA_ONLY = {"on": False}     # inside ``only_data_grads()``: the force pass of the MLIP loss


class tensor_cores:
    """Context manager: run the large-M Linear layers on the wgmma TF32 kernels (hgb_tc_*)."""

    def __init__(self, enabled=True):
        self.enabled, self.prev = bool(enabled), None

    def __enter__(self):
        self.prev = _TC["enabled"]
        _TC["enabled"] = self.enabled
        return self

    def __exit__(self, *exc):
        _TC["enabled"] = self.prev
        return False


EXACT_TC = os.environ.get("HGB_EXACT_TC", "1") == "1"     # fp32 mode: large-M Linears on wgmma with the 3xTF32 split (fp32-accurate)
EXACT_WGRAD = os.environ.get("HGB_EXACT_WGRAD", "1") == "1"   # ... and their weight gradients (0: SIMT fp32 GEMM)


def tc_wgrad_ok(m, n_out, k_out, *tensors):
    """dW = dZ^T X on the wgmma kernel: always in TF32 mode, in fp32 mode when the split variant is enabled"""
    if not (_TC["enabled"] or (EXACT_TC and EXACT_WGRAD)):
        return False
    return k_out + 16 <= 256 and tc_ok(m, n_out, k_out, *tensors)


def tc_ok(m, n_out, k_red, *tensors):
    if not (_TC["enabled"] or EXACT_TC):
        return False
    if not _lib.query("hgb_tc_linear_supported", m, n_out, k_red):
        return False
    for t in tensors:
        if t is not None and (t.data_ptr() % 16 != 0 or (t.dim() == 2 and t.stride(0) % 4 != 0)):
            return False
    return True


def raw_tc_linear(a2, w, trans_b, bias, n_out, k_red, code=0, param=0.0, want_z=False, addend=None, gsrc=None, gact=0):
    m = a2.shape[0]
    y = torch.empty(m, n_out, dtype=a2.dtype, device=a2.device)
    z = torch.empty_like(y) if want_z else None
    _lib.call("hgb_tc_linear", _p(a2), a2.stride(0), _p(w), w.stride(0), int(trans_b), _p(bias), m, n_out, k_red, code, float(param),
              _p(y), _p(z), _p(addend), _p(gsrc), int(gact), 0 if _TC["enabled"] else 1, _stream())
    return y, z


def raw_tc_wgrad(dz, x2, want_bias=True, dw=None, db=None, accumulate=False):
    m, n_out = dz.shape
    k_out = x2.shape[1]
    if dw is None:
        dw = torch.empty(n_out, k_out, dtype=dz.dtype, device=dz.device)
    if want_bias and db is None:
        db = torch.empty(n_out, dtype=dz.dtype, device=dz.device)
    exact = 0 if _TC["enabled"] else 1              # fp32 mode: 3xTF32 split inside the kernel
    piece = 256 if k_out <= 96 else 128             # the pipeline stages of (dz piece + x) must fit shared memory
    for c0 in range(0, n_out, piece):               # output-feature pieces (independent rows of dw)
        nc = min(piece, n_out - c0)
        nbytes = _lib.query("hgb_tc_wgrad_workspace_bytes", nc, k_out)
        ws = _ws(nbytes, dz.device)
        _lib.call("hgb_tc_wgrad", _p(dz[:, c0:]), dz.stride(0), _p(x2), x2.stride(0), m, nc, k_out, _p(dw[c0:]), dw.stride(0),
                  _p(db[c0:]) if want_bias else None, int(accumulate), exact, _p(ws), nbytes, _stream())
    return dw, db


def smallk_ok(n, k):
    return k <= 8 and bool(_lib.query("hgb_linear_smallk_supported", n, k))


def raw_smallk_fwd(x2, w, b, code=0, param=0.0, want_z=False):
    m, k = x2.shape
    n = w.shape[0]
    y = torch.empty(m, n, dtype=x2.dtype, device=x2.device)
    z = torch.empty_like(y) if want_z else None
    _lib.call("hgb_linear_smallk_fwd", _p(x2), x2.stride(0), _p(w), w.stride(0), _p(b), m, n, k, code, float(param), _p(y), _p(z), _stream())
    return y, z


def raw_smallk_bwd(dy, y, z, x2, w, code=0, param=0.0, need_x=True, need_w=True, need_b=True):
    """One pass: applies act' to dy, returns (dx, dw, db)."""
    m, n = dy.shape
    k = x2.shape[1]
    dx = torch.empty(m, k, dtype=dy.dtype, device=dy.device) if need_x else None
    dw = torch.empty(n, k, dtype=dy.dtype, device=dy.device) if need_w else None
    db = torch.empty(n, dtype=dy.dtype, device=dy.device) if need_b else None
    ws = _ws(_lib.query("hgb_linear_smallk_bwd_workspace_bytes", m, n, k), dy.device)
    _lib.call("hgb_linear_smallk_bwd", _p(dy), _p(y), _p(z), _p(x2), x2.stride(0), _p(w), w.stride(0), m, n, k, code, float(param),
              _p(dx), _p(dw), k, _p(db), _p(ws), _stream())
    return dx, dw, db


GROUPED_CSR = os.environ.get("HGB_GROUPED_CSR", "1") == "1"   # sort-free by-source CSR for radius-graph edges
COL_HINT = os.environ.get("HGB_COL_HINT", "1") == "1"   # reuse the radius graph's by-target offsets as the by_col CSR
ACT_DERIV = 100   # HGB_ACT_DERIV: "the tensor already holds act'(.)"


def linear_fwd_dispatch(x2, w, b, code=0, param=0.0, want_z=False):
    """y = act(x2 W^T + b) on the tensor-core kernel when the shape qualifies, else the exact-fp32 kernel."""
    return linear_fwd_dispatch_ex(x2, w, b, code, param, want_z)[:2]


def linear_fwd_dispatch_ex(x2, w, b, code=0, param=0.0, want_z=False, z_deriv=False):
    """-> (y, z, z_is_derivative).  With ``z_deriv`` a SiLU layer on the tensor-core path stores silu'(pre-activation) in z
    (computed next to the activation itself), so that its backward is a plain multiply."""
    m, k = x2.shape
    n = w.shape[0]
    if smallk_ok(n, k):
        return raw_smallk_fwd(x2, w, b, code, param, want_z) + (False,)
    if tc_ok(m, n, k, x2) and (k <= 256 or (code == 0 and not want_z)):     # a reduction cut into pieces needs a plain linear layer
        deriv = bool(z_deriv and want_z and code == ACT_CODES["silu"])
        return raw_tc_linear(x2, w, False, b, n, k, code, param, want_z, gact=ACT_DERIV if deriv else 0) + (deriv,)
    return raw_linear(x2, w, b, code, param, want_z) + (False,)


# ---- weight gradient next to the data gradient ---------------------------------------------------------------------------------
# The weight gradient and the data gradient of a layer read the same dZ and are independent of each other.  ``fork_join`` launches
# the weight-gradient kernels on a SIDE stream forked from the current one, lets the caller launch the data gradient on the main
# stream, and joins before either result is handed to autograd -- in a captured step the two become parallel branches of the CUDA
# graph.  Inside ``deferred_weight_gradients()`` (the engine's own step: FlatAdamW.backward) the join of a LEAF parameter that has
# not received a gradient in this backward pass moves to the end of the pass (an autograd-engine callback): nothing reads such a
# gradient on the main stream before the optimizer (AccumulateGrad takes the tensor over without a kernel), so the weight-gradient
# kernels overlap everything that follows.  The inputs of the deferred kernels are kept referenced until the join, which stops
# autograd from accumulating into them in place (it only does that to tensors nobody else holds).  Derived weights (scaled, sliced,
# concatenated: MACE, PNAEq) are read by their own backward nodes right away -- those join immediately; so does everything outside
# the context, where gradient hooks (torch DDP's reducer, user hooks) may read a gradient the moment it is accumulated.
WGRAD_OVERLAP = os.environ.get("HGB_WGRAD_OVERLAP", "1") == "1"
_SIDE = {}


def _side_stream(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _SIDE:
        _SIDE[key] = torch.cuda.Stream(device=key)
    return _SIDE[key]


class capture_graph:
    """``with capture_graph(g):`` = ``torch.cuda.graph(g)`` with Python's cyclic collector paused for the duration: a collection
    that runs mid-capture may destroy an older CUDAGraph (or free event-carrying blocks), and those driver calls are not
    permitted while a global-mode capture is open (seen as a flaky failed capture in a long test session)."""

    def __init__(self, graph, **kw):
        self.ctx = torch.cuda.graph(graph, **kw)

    def __enter__(self):
        import gc
        self.gc_was_on = gc.isenabled()
        gc.collect()
        gc.disable()
        try:
            return self.ctx.__enter__()
        except BaseException:
            if self.gc_was_on:
                gc.enable()
            raise

    def __exit__(self, *exc):
        import gc
        try:
            return self.ctx.__exit__(*exc)
        finally:
            if self.gc_was_on:
                gc.enable()


_PENDING = {"keys": set(), "leaves": set(), "hold": [], "bytes": 0}
_DEFER = {"on": False}
HOLD_LIMIT = 8 << 30          # bytes of deferred-kernel inputs kept alive before a join is forced


class deferred_weight_gradients:
    """Context manager around ``loss.backward()`` of a step whose gradients are first read by ``FlatAdamW.gather_grads``."""

    def __enter__(self):
        self.prev = _DEFER["on"]
        _DEFER["on"] = True
        return self

    def __exit__(self, *exc):
        _DEFER["on"] = self.prev
        join_side_streams()


def join_side_streams():
    """Join every side stream with deferred weight-gradient work (end of a backward pass; also called by FlatAdamW.gather_grads)."""
    for key in list(_PENDING["keys"]):
        torch.cuda.current_stream(key).wait_stream(_SIDE[key])
    _PENDING["keys"].clear()
    _PENDING["leaves"].clear()
    _PENDING["hold"].clear()
    _PENDING["bytes"] = 0


class fork_join:
    """``with fork_join(dz, x2) as fj: w = fj.side(lambda: wgrad(...)); dx = dgrad(...)`` -- ``w`` and ``dx`` are both ready (in stream
    order) when the block exits."""

    def __init__(self, *inputs, defer_for=None):
        """``defer_for``: the leaf parameters whose gradients the side work produces (or None): if every one is a leaf that has no
        gradient yet and was not served earlier in this backward pass, the join is deferred to the end of the pass."""
        self.inputs = [t for t in inputs if t is not None]
        self.on = bool(WGRAD_OVERLAP and self.inputs and self.inputs[0].is_cuda)
        self.defer = False
        if self.on and defer_for and _DEFER["on"]:
            ok = all(p is not None and p.is_leaf and p.requires_grad and p.grad is None and id(p) not in _PENDING["leaves"] for p in defer_for)
            if ok:
                try:
                    torch.autograd.Variable._execution_engine.queue_callback(join_side_streams)
                    self.defer = True
                    self.leaf_ids = [id(p) for p in defer_for]
                except RuntimeError:             # not inside a backward pass
                    self.defer = False

    def __enter__(self):
        if self.on:
            dev = self.inputs[0].device
            self.main = torch.cuda.current_stream(dev)
            self.sidestream = _side_stream(dev)
            self.sidestream.wait_stream(self.main)
            self.outs = []
        return self

    def side(self, fn):
        if not self.on:
            return fn()
        with torch.cuda.stream(self.sidestream):
            out = fn()
        self.outs.append(out)
        return out

    def __exit__(self, *exc):
        if self.on:
            if self.defer:
                key = self.inputs[0].device.index if self.inputs[0].device.index is not None else torch.cuda.current_device()
                _PENDING["keys"].add(key)
                _PENDING["leaves"].update(self.leaf_ids)
                _PENDING["hold"].append(self.inputs)           # referenced -> autograd will not accumulate into them in place
                _PENDING["bytes"] += sum(t.numel() * t.element_size() for t in self.inputs)
                if _PENDING["bytes"] > HOLD_LIMIT:
                    join_side_streams()
            else:
                self.main.wait_stream(self.sidestream)
            for t in self.inputs:
                t.record_stream(self.sidestream)
            for out in self.outs:
                for t in (out if isinstance(out, (tuple, list)) else (out,)):
                    if torch.is_tensor(t):
                        t.record_stream(self.main)
        return False


def linear_bwd_dispatch(dz, x2, w, need_x=True, need_w=True, need_b=True, dx_addend=None, dx_gsrc=None, dx_gact=0, dx_gparam=0.0,
                        leaves=None):
    """(dx, dw, db) of y = x2 W^T + b given dz.  ``dx_addend`` (same shape as dx) is accumulated into dx.  With ``dx_gsrc``
    the layer's input was act(.) and dx is returned already multiplied by act'(dx_gsrc) (SiLU: pre-activation, else output):
    on the tensor-core path that happens in the dgrad epilogue."""
    m, n = dz.shape
    k = x2.shape[1]

    def through_act(dx):
        if dx is None or dx_gsrc is None:
            return dx
        silu = dx_gact in (ACT_CODES["silu"], ACT_DERIV)
        return raw_act_bwd(dx, None if silu else dx_gsrc, dx_gsrc if silu else None, dx_gact, dx_gparam)

    if smallk_ok(n, k):
        dx, dw, db = raw_smallk_bwd(dz, None, None, x2, w, 0, 0.0, need_x, need_w, need_b)
        return through_act(dx + dx_addend if (dx is not None and dx_addend is not None) else dx), dw, db
    dx = dw = db = None
    with fork_join(dz, x2, defer_for=leaves) as fj:
        if need_w or need_b:                                                     # side stream: the weight gradient
            if tc_wgrad_ok(m, n, k, dz, x2):
                dw, db = fj.side(lambda: raw_tc_wgrad(dz, x2, want_bias=need_b))
            else:
                dw, db = fj.side(lambda: ((raw_gemm(dz, x2, True, False) if need_w else None), (raw_colsum(dz) if need_b else None)))
        if need_x:                                                               # main stream: the data gradient
            if tc_ok(m, k, n, dz, dx_addend, dx_gsrc) and (n <= 256 or dx_gsrc is None):
                dx = raw_tc_linear(dz, w, True, None, k, n, param=dx_gparam, addend=dx_addend, gsrc=dx_gsrc, gact=dx_gact)[0]
            elif dx_addend is not None:
                dx = through_act(raw_gemm(dz, w, False, False, out=dx_addend.clone(), beta_one=True))
            else:
                dx = through_act(raw_gemm(dz, w, False, False))
    return dx, dw, db


def _row_major_2d(t):
    """View an [..., k] tensor as [m, k] with unit inner stride (copying only if it has to)."""
    k = t.shape[-1]
    t2 = t.reshape(-1, k)
    if t2.stride(1) != 1 or (t2.shape[0] > 1 and t2.stride(0) < k):
        t2 = t2.contiguous()
    return t2


# =====================================================================================================
# any-order differentiable primitives
# =====================================================================================================
class GatherRows(torch.autograd.Function):
    """``x[idx]``; adjoint = SegmentSum over the CSR of ``idx``."""

    @staticmethod
    def forward(ctx, x, csr):
        ctx.csr = csr
        return raw_gather(x, csr.idx)

    @staticmethod
    def backward(ctx, g):
        return SegmentSum.apply(g, ctx.csr), None


class SegmentSum(torch.autograd.Function):
    """``zeros(n).index_add_(0, idx, m)`` as a deterministic segmented reduction; adjoint = GatherRows."""

    @staticmethod
    def forward(ctx, m, csr):
        ctx.csr = csr
        return raw_segment_sum(m, csr.rowptr, csr.perm, csr.n)

    @staticmethod
    def backward(ctx, g):
        return GatherRows.apply(g, ctx.csr), None


class MatMul(torch.autograd.Function):
    """``op(a) @ op(b)`` (2-D).  d/da and d/db are MatMuls again, so this is closed under autograd.  Under
    ``tensor_cores(True)`` (precision="bf16") the three shapes a training step produces -- x Wᵀ, g W and gᵀ x -- run on the
    wgmma TF32 kernels; the flag travels with the node so that (double) backward passes outside the context keep it."""

    @staticmethod
    def forward(ctx, a, b, ta, tb, b_is_weight=False):
        ctx.save_for_backward(a, b)
        ctx.ta, ctx.tb, ctx.tc = ta, tb, _TC["enabled"]
        ctx.b_is_weight = bool(b_is_weight)
        a2, b2 = _row_major_2d(a), _row_major_2d(b)
        if ctx.tc or EXACT_TC:      # precision "bf16": plain TF32; "fp32": the 3xTF32 split inside the same kernel (exact flag)
            if not ta and tb and tc_ok(a2.shape[0], b2.shape[0], a2.shape[1], a2):             # [m,k] x [n,k]^T  (the small operand is staged
                                                                                                 #  by plain loads: any row stride, e.g. a column slice)
                return raw_tc_linear(a2, b2, False, None, b2.shape[0], a2.shape[1])[0]
            if not ta and not tb and tc_ok(a2.shape[0], b2.shape[1], a2.shape[1], a2):         # [m,n] x [n,k]
                return raw_tc_linear(a2, b2, True, None, b2.shape[1], a2.shape[1])[0]
            if ta and not tb and tc_wgrad_ok(a2.shape[0], a2.shape[1], b2.shape[1], a2, b2):
                return raw_tc_wgrad(a2, b2, want_bias=False)[0]                                    # [m,n]^T x [m,k]
        return raw_gemm(a2, b2, ta, tb)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        ta, tb = ctx.ta, ctx.tb
        ga = gb = None
        with tensor_cores(ctx.tc):
            if ctx.needs_input_grad[0]:
                #  C = A B     : gA = G B^T      C = A^T B   : gA = B G^T
                #  C = A B^T   : gA = G B        C = A^T B^T : gA = B^T G^T
                ga = MatMul.apply(b, g, tb, True) if ta else MatMul.apply(g, b, False, not tb)
            # the force pass of the MLIP loss (only_data_grads) differentiates w.r.t. positions only: weight gradients computed
            # there would be thrown away by autograd (a custom Function cannot see which outputs the engine needs)
            if ctx.needs_input_grad[1] and not (ctx.b_is_weight and _DATA_ONLY["on"]):
                #  C = A B     : gB = A^T G      C = A B^T   : gB = G^T A
                #  C = A^T B   : gB = A G        C = A^T B^T : gB = G^T A^T
                gb = MatMul.apply(g, a, True, ta) if tb else MatMul.apply(a, g, not ta, False)
        return ga, gb, None, None, None


class ColSum(torch.autograd.Function):
    """``x.sum(0)`` of a 2-D tensor with the two-stage column-sum kernel; adjoint = row broadcast (closed with BiasAdd)."""

    @staticmethod
    def forward(ctx, x):
        ctx.rows = x.shape[0]
        return raw_colsum(_chk(x if x.is_contiguous() else x.contiguous()))

    @staticmethod
    def backward(ctx, g):
        return g.unsqueeze(0).expand(ctx.rows, g.shape[0])


class BiasAdd(torch.autograd.Function):
    """``y + b`` (b broadcast over rows); the bias gradient is a ColSum, so any order of differentiation stays closed."""

    @staticmethod
    def forward(ctx, y, b):
        return y + b

    @staticmethod
    def backward(ctx, g):
        return g, (ColSum.apply(g) if (ctx.needs_input_grad[1] and not _DATA_ONLY["on"]) else None)


def linear_any_order(x, weight, bias=None):
    """``x @ W^T + b`` built from the closed primitives (MatMul, BiasAdd / ColSum)."""
    shp = x.shape
    y = MatMul.apply(x.reshape(-1, shp[-1]), weight, False, True, True)
    if bias is not None:
        y = BiasAdd.apply(y, bias)
    return y.reshape(shp[:-1] + (weight.shape[0],))


# =====================================================================================================
# fused first-order blocks
# =====================================================================================================
class LinearAct(torch.autograd.Function):
    """``act(x W^T + b)`` in one kernel; backward = act' kernel + two GEMMs + a column sum."""

    @staticmethod
    def forward(ctx, x, weight, bias, act, act_param):
        shp = x.shape
        x2 = _row_major_2d(x)
        w = weight if weight.stride(1) == 1 else weight.contiguous()
        m, k = x2.shape
        n = w.shape[0]
        code = ACT_CODES[act]
        y, z = linear_fwd_dispatch(x2, w, _chk(bias), code, act_param, want_z=(code == ACT_CODES["silu"]))
        ctx.save_for_backward(x2, w, y if code not in (0, ACT_CODES["silu"]) else None, z)
        ctx.code, ctx.param, ctx.shp, ctx.has_bias = code, float(act_param), shp, bias is not None
        ctx.tc = _TC["enabled"]                      # the backward runs outside the forward's precision context
        ctx.leaves = [weight] + ([bias] if bias is not None else [])     # who receives the weight gradient (leaf parameters?)
        return y.reshape(shp[:-1] + (n,))

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x2, w, y, z = ctx.saved_tensors
        m, k = x2.shape
        n = w.shape[0]
        gy2 = _chk(gy.reshape(m, n))
        if smallk_ok(n, k):
            gx, gw, gb = raw_smallk_bwd(gy2, y, z, x2, w, ctx.code, ctx.param, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                        ctx.has_bias and ctx.needs_input_grad[2])
            return (gx.reshape(ctx.shp) if gx is not None else None), gw, gb, None, None
        if ctx.code != 0:
            dz = torch.empty_like(gy2)
            _lib.call("hgb_act_bwd", _p(gy2), _p(y), _p(z), gy2.numel(), ctx.code, ctx.param, _p(dz), _stream())
        else:
            dz = gy2
        with tensor_cores(ctx.tc):
            gx, gw, gb = linear_bwd_dispatch(dz, x2, w, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                             ctx.has_bias and ctx.needs_input_grad[2], leaves=ctx.leaves)
        if gx is not None:
            gx = gx.reshape(ctx.shp)
        return gx, gw, gb, None, None


def linear_act(x, weight, bias=None, act=None, act_param=0.0):
    return LinearAct.apply(x, weight, bias, act, act_param)


class Mlp2Fn(torch.autograd.Function):
    """``act2(act1(x W1^T + b1) W2^T + b2)`` as one node: in the backward the gradient through act1 is applied in the epilogue of
    the second layer's data-gradient GEMM (no separate activation-backward pass over the hidden tensor)."""

    @staticmethod
    def forward(ctx, x, w1, b1, act1, p1, w2, b2, act2, p2):
        shp = x.shape
        x2 = _row_major_2d(x)
        w1_in, w2_in = w1, w2
        w1 = w1 if w1.stride(1) == 1 else w1.contiguous()
        w2 = w2 if w2.stride(1) == 1 else w2.contiguous()
        c1, c2 = ACT_CODES[act1], ACT_CODES[act2]
        silu = ACT_CODES["silu"]
        h, z1, deriv = linear_fwd_dispatch_ex(x2, w1, _chk(b1), c1, p1, want_z=(c1 == silu), z_deriv=True)
        y, z2 = linear_fwd_dispatch(h, w2, _chk(b2), c2, p2, want_z=(c2 == silu))
        ctx.save_for_backward(x2, w1, w2, h, z1, y if c2 not in (0, silu) else None, z2)
        ctx.cfg = (ACT_DERIV if deriv else c1, float(p1), c2, float(p2), shp, b1 is not None, b2 is not None)
        ctx.tc = _TC["enabled"]
        ctx.leaves1 = [w1_in] + ([b1] if b1 is not None else [])
        ctx.leaves2 = [w2_in] + ([b2] if b2 is not None else [])
        return y.reshape(shp[:-1] + (w2.shape[0],))

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x2, w1, w2, h, z1, y, z2 = ctx.saved_tensors
        c1, p1, c2, p2, shp, has_b1, has_b2 = ctx.cfg
        m = x2.shape[0]
        gy2 = _chk(gy.reshape(m, w2.shape[0]))
        dz2 = raw_act_bwd(gy2, y, z2, c2, p2) if c2 != 0 else gy2
        with tensor_cores(ctx.tc):
            dz1, gw2, gb2 = linear_bwd_dispatch(dz2, h, w2, True, ctx.needs_input_grad[5], has_b2 and ctx.needs_input_grad[6],
                                                dx_gsrc=(z1 if c1 in (ACT_CODES["silu"], ACT_DERIV) else h), dx_gact=c1, dx_gparam=p1,
                                                leaves=ctx.leaves2)
            gx, gw1, gb1 = linear_bwd_dispatch(dz1, x2, w1, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                               has_b1 and ctx.needs_input_grad[2], leaves=ctx.leaves1)
        return (gx.reshape(shp) if gx is not None else None), gw1, gb1, None, None, gw2, gb2, None, None


class Mlp2ScalarFn(torch.autograd.Function):
    """Linear(1,1) - act - Linear(1,out<=4): one kernel forward, one kernel + a 10-value reduce backward."""

    @staticmethod
    def forward(ctx, x, w1, b1, act1, p1, w2, b2):
        n, out = x.shape[0], w2.shape[0]
        pad = x.new_zeros(4 - out)
        pk = torch.cat([w1.reshape(1), b1.reshape(1), w2.reshape(out), pad, b2.reshape(out), pad]).contiguous()
        x1 = _chk(x.reshape(n).contiguous())
        y = torch.empty(n, out, dtype=x.dtype, device=x.device)
        _lib.call("hgb_mlp2_scalar_fwd", _p(x1), _p(pk), n, out, ACT_CODES[act1], float(p1), _p(y), _stream())
        ctx.save_for_backward(x1, pk)
        ctx.cfg = (ACT_CODES[act1], float(p1), out)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x1, pk = ctx.saved_tensors
        code, p1, out = ctx.cfg
        n = x1.shape[0]
        gx = torch.empty_like(x1) if ctx.needs_input_grad[0] else None
        gp = torch.empty(10, dtype=x1.dtype, device=x1.device)
        ws = _ws(_lib.query("hgb_mlp2_scalar_workspace_bytes"), x1.device)
        _lib.call("hgb_mlp2_scalar_bwd", _p(_chk(gy.contiguous())), _p(x1), _p(pk), n, out, code, p1, _p(gx), _p(gp), _p(ws), _stream())
        return (gx.reshape(n, 1) if gx is not None else None), gp[0:1].reshape(1, 1), gp[1:2], None, None, gp[2:2 + out].reshape(out, 1), gp[6:6 + out]


def mlp2(x, w1, b1, act1, p1, w2, b2, act2=None, p2=0.0):
    if (SCALAR_UPDATE and act2 is None and b1 is not None and b2 is not None and x.dim() == 2 and x.shape[1] == 1
            and w1.shape == (1, 1) and w2.shape[1] == 1 and w2.shape[0] <= 4):
        return Mlp2ScalarFn.apply(x, w1, b1, act1, p1, w2, b2)          # width-1 layer (quirk Q4)
    return Mlp2Fn.apply(x, w1, b1, act1, p1, w2, b2, act2, p2)


class EdgeGeomFn(torch.autograd.Function):
    """(vec, len, unit) of hydragnn/utils/model/operations.py:21-36 in one pass; the backward turns the
    three edge gradients into one [E,3] vector and scatters it to both endpoints with segment sums."""

    @staticmethod
    def forward(ctx, pos, shifts, plan, eps):
        pos = _chk(pos)
        e = plan.num_edges
        vec = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        ln = torch.empty(e, 1, dtype=pos.dtype, device=pos.device)
        unit = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        _lib.call("hgb_edge_geom_fwd", _p(pos), _p(plan.row), _p(plan.col), _p(_chk(shifts)), e, float(eps), _p(vec), _p(ln),
                  _p(unit), _stream())
        ctx.save_for_backward(vec, ln)
        ctx.plan, ctx.eps = plan, float(eps)
        return vec, ln, unit

    @staticmethod
    @once_differentiable
    def backward(ctx, g_vec, g_len, g_unit):
        vec, ln = ctx.saved_tensors
        plan = ctx.plan
        gv = torch.empty_like(vec)
        _lib.call("hgb_edge_geom_bwd", _p(vec), _p(ln), ctx.eps, _p(_chk(g_vec)), _p(_chk(g_len)), _p(_chk(g_unit)),
                  plan.num_edges, _p(gv), _stream())
        g_pos = g_shift = None
        if ctx.needs_input_grad[0]:
            # vec = pos[col] - pos[row] + shift
            g_pos = raw_segment_sum(gv, plan.by_col.rowptr, plan.by_col.perm, plan.num_nodes) - \
                raw_segment_sum(gv, plan.by_row.rowptr, plan.by_row.perm, plan.num_nodes)
        if ctx.needs_input_grad[1]:
            g_shift = gv
        return g_pos, g_shift, None, None


class PainnEdgeEmbedFn(torch.autograd.Function):
    """len/unit -> one 12-float record per edge {rbf*cutoff (8, zero padded), cutoff, dir = unit/len [quirk Q2]}
    (hydragnn/models/PAINNStack.py:239-242,257)."""

    @staticmethod
    def forward(ctx, unit, ln, num_radial, cutoff):
        e = unit.shape[0]
        epack = torch.empty(e, 12, dtype=unit.dtype, device=unit.device)
        _lib.call("hgb_painn_edge_embed_fwd", _p(unit), _p(ln), e, num_radial, float(cutoff), _p(epack), _stream())
        ctx.save_for_backward(unit, ln)
        ctx.r, ctx.cutoff = num_radial, float(cutoff)
        return epack

    @staticmethod
    @once_differentiable
    def backward(ctx, g_epack):
        unit, ln = ctx.saved_tensors
        e = unit.shape[0]
        g_unit = torch.empty_like(unit)
        g_len = torch.empty_like(ln)
        _lib.call("hgb_painn_edge_embed_bwd", _p(unit), _p(ln), _p(_chk(g_epack)), e, ctx.r, ctx.cutoff, _p(g_unit), _p(g_len), _stream())
        return g_unit, g_len, None, None


class PainnMessageFn(torch.autograd.Function):
    """Fused PaiNN message (hydragnn/models/PAINNStack.py:239-270): returns (s + ds, v + dv)."""

    @staticmethod
    def forward(ctx, phi, s, v, epack, wf, bf, efilt, plan, rec_row=None):
        n, f = s.shape
        r = wf.shape[1]
        phi, s, v = _chk(phi), _chk(s), _chk(v)
        s_out, v_out = torch.empty_like(s), torch.empty_like(v)
        agg = plan.by_row     # messages are summed into edge[:,0] = edge_index[0]
        _lib.call("hgb_painn_message_fwd", _p(phi), _p(s), _p(v), _p(agg.rowptr), _p(agg.perm), _p(plan.nbr("row")), _p(epack),
                  _p(rec_row), _p(_chk(wf)), _p(_chk(bf)), _p(_chk(efilt)), n, f, r, _p(s_out), _p(v_out), _stream())
        ctx.save_for_backward(phi, v, epack, wf, bf, efilt)
        ctx.plan, ctx.use_rec = plan, rec_row is not None
        return s_out, v_out

    @staticmethod
    @once_differentiable
    def backward(ctx, gs_out, gv_out):
        phi, v, epack, wf, bf, efilt = ctx.saved_tensors
        plan = ctx.plan
        n, f = gs_out.shape
        r = wf.shape[1]
        gs_out, gv_out = _chk(gs_out), _chk(gv_out)
        need_edge = ctx.needs_input_grad[3]
        gphi, gv = torch.empty_like(phi), torch.empty_like(v)
        gwf, gbf = torch.empty_like(wf), torch.empty_like(bf)
        cpl = 2 if (f >= 64 and f % 2 == 0) else 1          # mirrors painn_cpl / painn_group in csrc/hgb_painn.cu
        multi = f > 32 * cpl                                # several channel blocks accumulate into g_epack
        g_epack = (torch.zeros_like(epack) if multi else torch.empty_like(epack)) if need_edge else None
        g_ef = torch.empty_like(efilt) if efilt is not None else None
        nbytes = _lib.query("hgb_painn_message_bwd_workspace_bytes", n, f, r)
        ws = _ws(nbytes, phi.device)
        src = plan.by_col     # the gather side: edge[:,1] = edge_index[1]
        rec_col = None
        if ctx.use_rec:       # by-col records: built once per batch (cached on the plan, keyed by the epack buffer)
            cache = plan.__dict__.setdefault("_rec_col", {})
            key = epack.data_ptr()
            if key not in cache:
                cache.clear()
                cache[key] = painn_edge_records(epack, plan, "col")
            rec_col = cache[key]
        _lib.call("hgb_painn_message_bwd", _p(gs_out), _p(gv_out), _p(phi), _p(v), _p(src.rowptr), _p(src.perm), _p(plan.nbr("col")),
                  _p(epack), _p(rec_col), _p(wf), _p(bf), _p(efilt), n, f, r, _p(gphi), _p(gv), _p(gwf), _p(gbf), _p(g_epack), _p(g_ef),
                  _p(ws), nbytes, _stream())
        return gphi, gs_out, gv, g_epack, gwf, gbf, g_ef, None, None


def painn_edge_records(epack, plan, which):
    """CSR-ordered 64-byte edge records for the tiled message kernels (built once per batch, shared by all layers)."""
    csr = plan.by_row if which == "row" else plan.by_col
    rec = torch.empty(plan.num_edges, 16, dtype=epack.dtype, device=epack.device)
    _lib.call("hgb_painn_edge_records", _p(epack.detach()), _p(csr.perm), _p(plan.nbr(which)), plan.num_edges, _p(rec), _stream())
    return rec


def raw_linear(x2, w, b, code=0, param=0.0, want_z=False):
    m, k = x2.shape
    n = w.shape[0]
    y = torch.empty(m, n, dtype=x2.dtype, device=x2.device)
    z = torch.empty_like(y) if want_z else None
    if gemm3_ok(x2, w, y, m, n, k, False, True):
        _lib.call("hgb_gemm3", _p(x2), _p(w), _p(y), m, n, k, 0, 1, x2.stride(0), w.stride(0), n, 0, _p(b), code, float(param), _p(z), None,
                  _stream())
        return y, z
    _lib.call("hgb_linear_fwd", _p(x2), _p(w), _p(b), m, n, k, x2.stride(0), w.stride(0), code, float(param), _p(y), _p(z), _stream())
    return y, z


def raw_act_bwd(dy, y, z, code, param=0.0):
    dz = torch.empty_like(dy)
    _lib.call("hgb_act_bwd", _p(dy), _p(y), _p(z), dy.numel(), code, float(param), _p(dz), _stream())
    return dz


class PainnUpdateFn(torch.autograd.Function):
    """The whole PaiNN update block (hydragnn/models/PAINNStack.py:298-328) with one hand-written
    backward: U/V linears, |Vv|, update_mlp (Linear-SiLU-Linear) and the gated residuals.
    update_U and update_V read the same input, so they run as ONE GEMM against the stacked weights [U; V]
    (output [3n, 2f]: uv = left half, vv = right half); the backward is one dgrad and one wgrad for both."""

    @staticmethod
    def forward(ctx, s, v, uw, ub, vw, vb, w1, b1, w2, b2, last):
        n, f = s.shape
        s, v = _chk(s), _chk(v)
        w1, b1, w2, b2 = [_chk(t) for t in (w1, b1, w2, b2)]
        v2 = v.reshape(3 * n, f)
        wuv, buv = torch.cat([uw, vw], dim=0).contiguous(), torch.cat([ub, vb], dim=0).contiguous()
        y_uv, _ = linear_fwd_dispatch(v2, wuv, buv)                                  # [3n, 2f]
        uv, vv, ld = y_uv, y_uv[:, f:], 2 * f
        mlp_in = torch.empty(n, 2 * f, dtype=s.dtype, device=s.device)
        _lib.call("hgb_painn_update_pre_fwd", _p(vv), ld, _p(s), n, f, _p(mlp_in), _stream())
        h, z1, deriv = linear_fwd_dispatch_ex(mlp_in, w1, b1, ACT_CODES["silu"], 0.0, want_z=True, z_deriv=True)
        a, _ = linear_fwd_dispatch(h, w2, b2)
        ctx.z1_code = ACT_DERIV if deriv else ACT_CODES["silu"]
        s_out = torch.empty_like(s)
        v_out = None if last else torch.empty_like(v)
        _lib.call("hgb_painn_update_post_fwd", _p(a), _p(uv), _p(vv), ld, _p(s), _p(v), n, f, int(last), _p(s_out), _p(v_out), _stream())
        ctx.save_for_backward(v2, y_uv, mlp_in, z1, h, a, wuv, w1, w2)
        ctx.last = bool(last)
        ctx.tc = _TC["enabled"]
        ctx.leaves = ([uw, ub, vw, vb], [w1, b1], [w2, b2])
        if last:
            return s_out, s_out.new_zeros(0)
        return s_out, v_out

    @staticmethod
    @once_differentiable
    def backward(ctx, gs_out, gv_out):
        v2, y_uv, mlp_in, z1, h, a, wuv, w1, w2 = ctx.saved_tensors
        last = ctx.last
        n, f = gs_out.shape
        ld = 2 * f
        uv, vv = y_uv, y_uv[:, f:]
        gs_out = _chk(gs_out)
        gv_out = None if last else _chk(gv_out.contiguous())
        ga = torch.empty_like(a)
        _lib.call("hgb_painn_update_post_bwd_a", _p(gs_out), _p(gv_out), _p(uv), _p(vv), ld, n, f, int(last), _p(ga), _stream())
        with tensor_cores(ctx.tc):
            gz1, gw2, gb2 = linear_bwd_dispatch(ga, h, w2, dx_gsrc=z1, dx_gact=ctx.z1_code, leaves=ctx.leaves[2])     # dgrad through the SiLU
            g_mlp_in, gw1, gb1 = linear_bwd_dispatch(gz1, mlp_in, w1, leaves=ctx.leaves[1])
        g_uv = torch.empty_like(y_uv)                                                # [3n, 2f] = [guv | gvv]
        gs = torch.empty_like(gs_out)
        _lib.call("hgb_painn_update_bwd", _p(gs_out), _p(gv_out), _p(g_mlp_in), _p(a), _p(uv), _p(vv), ld, _p(mlp_in), n, f,
                  int(last), _p(g_uv), _p(g_uv[:, f:]), _p(gs), None, _stream())
        with tensor_cores(ctx.tc):
            # gv = gv_out (direct path, added in the dgrad epilogue) + [guv | gvv] [U; V]
            gv, gwuv, gbuv = linear_bwd_dispatch(g_uv, v2, wuv, dx_addend=None if last else gv_out.reshape(3 * n, f), leaves=ctx.leaves[0])
        return gs, gv.reshape(n, 3, f), gwuv[:f], gbuv[:f], gwuv[f:], gbuv[f:], gw1, gb1, gw2, gb2, None


SCALAR_UPDATE = os.environ.get("HGB_SCALAR", "1") == "1"   # PaiNN update block at node_size == 1 through the one-kernel path


class PainnUpdateScalarFn(torch.autograd.Function):
    """PaiNN update block at node_size == 1 (the first layer of the reference runs at width input_dim, quirk Q4): the whole
    block in one kernel forward, one kernel + a 16-value reduce backward (everything is recomputed from s, v)."""

    @staticmethod
    def forward(ctx, s, v, uw, ub, vw, vb, w1, b1, w2, b2, last):
        n = s.shape[0]
        na = 2 if last else 3
        pad = s.new_zeros(3 - na)
        pk = torch.cat([uw.reshape(1), ub.reshape(1), vw.reshape(1), vb.reshape(1), w1.reshape(2), b1.reshape(1), w2.reshape(na), pad,
                        b2.reshape(na), pad, s.new_zeros(3)]).contiguous()
        s2, v2 = _chk(s.reshape(n).contiguous()), _chk(v.reshape(n, 3).contiguous())
        s_out = torch.empty_like(s2)
        v_out = None if last else torch.empty_like(v2)
        _lib.call("hgb_painn_update_scalar_fwd", _p(s2), _p(v2), _p(pk), n, int(last), _p(s_out), _p(v_out), _stream())
        ctx.save_for_backward(s2, v2, pk)
        ctx.last = bool(last)
        if last:
            return s_out.reshape(n, 1), s_out.new_zeros(0)
        return s_out.reshape(n, 1), v_out.reshape(n, 3, 1)

    @staticmethod
    @once_differentiable
    def backward(ctx, gs_out, gv_out):
        s2, v2, pk = ctx.saved_tensors
        n, last = s2.shape[0], ctx.last
        na = 2 if last else 3
        gs_out = _chk(gs_out.reshape(n).contiguous())
        gv_out = None if last else _chk(gv_out.reshape(n, 3).contiguous())
        gs, gv, gp = torch.empty_like(s2), torch.empty_like(v2), torch.empty(16, dtype=s2.dtype, device=s2.device)
        nbytes = _lib.query("hgb_painn_update_scalar_workspace_bytes")
        ws = _ws(nbytes, s2.device)
        _lib.call("hgb_painn_update_scalar_bwd", _p(gs_out), _p(gv_out), _p(s2), _p(v2), _p(pk), n, int(last), _p(gs), _p(gv), _p(gp),
                  _p(ws), _stream())
        return (gs.reshape(n, 1), gv.reshape(n, 3, 1), gp[0:1].reshape(1, 1), gp[1:2], gp[2:3].reshape(1, 1), gp[3:4],
                gp[4:6].reshape(1, 2), gp[6:7], gp[7:7 + na].reshape(na, 1), gp[10:10 + na], None)


class PoolFn(torch.autograd.Function):
    """global_{add,mean,max}_pool over a sorted batch vector (hydragnn/models/Base.py:147-170)."""

    @staticmethod
    def forward(ctx, x, gcsr, mode):
        x = _chk(x)
        g, c = gcsr.n, x.shape[1]
        out = torch.empty(g, c, dtype=x.dtype, device=x.device)
        code = POOL_CODES[mode]
        arg = torch.empty(g, c, dtype=torch.int32, device=x.device) if code == 2 else None
        _lib.call("hgb_pool_fwd", _p(x), _p(gcsr.rowptr), g, c, code, _p(out), _p(arg), _stream())
        ctx.gcsr, ctx.code, ctx.n, ctx.arg = gcsr, code, x.shape[0], arg
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        g = _chk(g)
        gx = torch.empty(ctx.n, g.shape[1], dtype=g.dtype, device=g.device)
        _lib.call("hgb_pool_bwd", _p(g), _p(ctx.gcsr.rowptr), _p(ctx.arg), ctx.n, ctx.gcsr.n, g.shape[1], ctx.code, _p(gx), _stream())
        return gx, None, None


class LossFn(torch.autograd.Function):
    """mean squared / absolute error with its gradient produced in the same pass."""

    @staticmethod
    def forward(ctx, pred, target, mode, valid_rows=None, row_width=1):
        pred, target = _chk(pred), _chk(target)
        loss = torch.empty(1, dtype=pred.dtype, device=pred.device)
        gpred = torch.empty_like(pred)
        _lib.call("hgb_loss_fwd_bwd", _p(pred), _p(target), pred.numel(), mode, 1.0, _p(loss), _p(gpred), _p(valid_rows), int(row_width),
                  _stream())
        ctx.save_for_backward(gpred)
        return loss.reshape(())

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (gpred,) = ctx.saved_tensors
        return gpred * g, None, None, None, None


class PnaAggregateFn(torch.autograd.Function):
    """[mean | min | max | std] of every CSR segment in one pass (the four PNA aggregators of PNAEqStack.py:396-400)."""

    @staticmethod
    def forward(ctx, m, csr):
        m = _chk(m.contiguous())
        n, c = csr.n, m.shape[1]
        out = torch.empty(n, 4 * c, dtype=m.dtype, device=m.device)
        amin = torch.empty(n, c, dtype=torch.int32, device=m.device)
        amax = torch.empty_like(amin)
        _lib.call("hgb_pna_aggregate_fwd", _p(m), _p(csr.rowptr), _p(csr.perm), n, c, _p(out), _p(amin), _p(amax), _stream())
        ctx.save_for_backward(m, out, amin, amax)
        ctx.csr = csr
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        m, out, amin, amax = ctx.saved_tensors
        csr = ctx.csr
        gm = torch.empty_like(m)
        _lib.call("hgb_pna_aggregate_bwd", _p(_chk(g.contiguous())), _p(m), _p(out), _p(csr.idx), _p(csr.rowptr), _p(amin), _p(amax),
                  m.shape[0], m.shape[1], _p(gm), _stream())
        return gm, None


# =====================================================================================================
# grouped dense layers (multi-branch decoding)
# =====================================================================================================
class GroupedLinearFn(torch.autograd.Function):
    """``y[r] = act(x[r] W_g^T + b_g)`` for rows sorted by group (``rowptr`` [groups + 1] on the device): the per-dataset branch
    heads of hydragnn/models/Base.py:770-780,816-840 as ONE launch per layer, no host read of the group sizes."""

    @staticmethod
    def forward(ctx, x, w, b, rowptr, act, act_param):
        x, w = _chk(x.contiguous()), _chk(w.contiguous())
        b = _chk(b.contiguous()) if b is not None else None
        groups, n, k = w.shape
        m = x.shape[0]
        code = ACT_CODES[act]
        y = torch.empty(m, n, dtype=x.dtype, device=x.device)
        z = torch.empty_like(y) if code == ACT_CODES["silu"] else None
        _lib.call("hgb_grouped_linear", _p(x), k, _p(w), _p(b), _p(rowptr), groups, m, n, k, 0, code, float(act_param), _p(y), _p(z), _stream())
        ctx.save_for_backward(x, w, y if code not in (0, ACT_CODES["silu"]) else None, z, rowptr)
        ctx.cfg = (code, float(act_param), b is not None)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, w, y, z, rowptr = ctx.saved_tensors
        code, param, has_b = ctx.cfg
        groups, n, k = w.shape
        m = x.shape[0]
        gy = _chk(gy.contiguous())
        dz = raw_act_bwd(gy, y, z, code, param) if code != 0 else gy
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = torch.empty(m, k, dtype=x.dtype, device=x.device)
            _lib.call("hgb_grouped_linear", _p(dz), n, _p(w), None, _p(rowptr), groups, m, k, n, 1, 0, 0.0, _p(gx), None, _stream())
        if ctx.needs_input_grad[1] or (has_b and ctx.needs_input_grad[2]):
            gw = torch.empty_like(w)
            gb = torch.empty(groups, n, dtype=x.dtype, device=x.device) if has_b else None
            _lib.call("hgb_grouped_wgrad", _p(dz), _p(x), k, _p(rowptr), groups, m, n, k, _p(gw), _p(gb), _stream())
        return gx, gw, gb, None, None, None


def grouped_mlp(seq_by_group, x, rowptr):
    """Run structurally identical ``nn.Sequential`` MLPs (one per group) on rows sorted by group.  Returns None when the
    branches do not share one architecture (the caller then falls back to per-branch launches)."""
    from torch import nn
    from .stacks import _act_code
    mods = [list(s) for s in seq_by_group]
    if any(len(m) != len(mods[0]) for m in mods):
        return None
    i = 0
    while i < len(mods[0]):
        layer = [m[i] for m in mods]
        if not all(isinstance(l, nn.Linear) for l in layer) or len({tuple(l.weight.shape) for l in layer}) != 1:
            return None
        code = _act_code(mods[0][i + 1]) if i + 1 < len(mods[0]) else None
        if i + 1 < len(mods[0]) and code is None:
            return None
        w = torch.stack([l.weight for l in layer])
        b = torch.stack([l.bias for l in layer]) if layer[0].bias is not None else None
        x = GroupedLinearFn.apply(x, w, b, rowptr, code[0] if code else None, code[1] if code else 0.0)
        i += 2 if code else 1
    return x


# =====================================================================================================
# fused EGNN edge block + closed edge-length primitives (any order of differentiation the MLIP loss needs)
# =====================================================================================================
FUSED_EGNN = os.environ.get("HGB_FUSED_EGNN", "1") == "1"     # 0: the round-1 composed path (gather / Linear / segment-sum)


class only_data_grads:
    """Context manager for the FORCE pass of the MLIP loss (``torch.autograd.grad(E, pos, create_graph=True)``,
    hydragnn/models/create.py:718-724): fused blocks skip their parameter gradients there -- autograd would compute and drop
    them (custom Functions cannot see which of their outputs the engine needs)."""

    def __enter__(self):
        self.prev = _DATA_ONLY["on"]
        _DATA_ONLY["on"] = True
        return self

    def __exit__(self, *exc):
        _DATA_ONLY["on"] = self.prev
        return False


def egnn_nodes_per_tile(plan):
    deg = max(1.0, plan.num_edges / max(plan.num_nodes, 1))
    return int(max(1, min(32, 120 // deg)))


def egnn_edge_supported(h):
    return bool(_lib.query("hgb_egnn_edge_supported", int(h)))


def _egnn_ws(n, h, npt, dev):
    return _ws(_lib.query("hgb_egnn_edge_workspace_bytes", n, h, npt), dev)


def _raw_egnn_fwd(pq, s, wd, b0, w1, b1, plan, npt, masks, tangent):
    n, h = pq.shape[0], pq.shape[1] // 2
    out = torch.empty(n, h, dtype=pq.dtype, device=pq.device)
    csr = plan.by_row
    _lib.call("hgb_egnn_edge_fwd", _p(pq), _p(s), _p(wd), _p(b0), _p(w1), _p(b1), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("row")), n, h,
              npt, int(tangent), _p(masks), _p(out), _stream())
    return out


def _raw_egnn_bwd_data(g_out, s, wd, w1, masks, plan, npt, want_params):
    """-> (g_pq [n, 2h], gz1 [e, h], gs [e], g_wd, g_b0)"""
    n, h = g_out.shape
    e = plan.num_edges
    dev = g_out.device
    g_pq = torch.empty(n, 2 * h, dtype=g_out.dtype, device=dev)
    gz1 = torch.empty(e, h, dtype=g_out.dtype, device=dev)
    gs = torch.empty(e, dtype=g_out.dtype, device=dev)
    g_wd = torch.empty(h, dtype=g_out.dtype, device=dev) if want_params else None
    g_b0 = torch.empty(h, dtype=g_out.dtype, device=dev) if want_params else None
    ws = _egnn_ws(n, h, npt, dev) if want_params else None
    csr = plan.by_row
    _lib.call("hgb_egnn_edge_bwd_data", _p(g_out), _p(s), _p(wd), _p(w1), _p(masks), _p(csr.rowptr), _p(csr.perm), n, h, npt, _p(g_pq), 2 * h,
              _p(gz1), _p(gs), _p(g_wd), _p(g_b0), _p(ws), _stream())
    # g_q = by-col segment sum of gz1, written into the right half of g_pq
    col = plan.by_col
    gq = g_pq[:, h:]
    _lib.call("hgb_segment_sum_strided", _p(gz1), _p(col.rowptr), _p(col.perm), n, h, _p(gq), 2 * h, _stream())
    return g_pq, gz1, gs, g_wd, g_b0


def _raw_egnn_wgrad(g_out, pq, s, wd, b0, masks, plan, npt, tangent, want_b1):
    n, h = g_out.shape
    dev = g_out.device
    g_w1 = torch.empty(h, h, dtype=g_out.dtype, device=dev)
    g_b1 = torch.empty(h, dtype=g_out.dtype, device=dev) if want_b1 else None
    ws = _egnn_ws(n, h, npt, dev)
    csr = plan.by_row
    _lib.call("hgb_egnn_edge_wgrad", _p(g_out), _p(pq), _p(s), _p(wd), _p(b0), _p(masks), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("row")),
              n, h, npt, int(tangent), _p(g_w1), _p(g_b1), _p(ws), _stream())
    return g_w1, g_b1


class EgnnEdgeFn(torch.autograd.Function):
    """agg = sum_row relu(W1 relu(P[row] + Q[col] + s w_d + b0) + b1)  -- the edge model and the scatter of E_GCL
    (hydragnn/models/EGCLStack.py:245-258) in one kernel.  Differentiable to the order the MLIP loss needs: its backward is
    ``EgnnEdgeBwdFn`` (itself differentiable); parameter gradients come from the fused weight-gradient kernel."""

    @staticmethod
    def forward(ctx, pq, s, wd, b0, w1, b1, plan):
        npt = egnn_nodes_per_tile(plan)
        masks = torch.empty(plan.num_edges, 2, dtype=torch.int64, device=pq.device)
        out = _raw_egnn_fwd(_chk(pq), _chk(s), _chk(wd), _chk(b0), _chk(w1), _chk(b1), plan, npt, masks, False)
        # save the INPUTS themselves (w_d is a column view of edge_mlp[0].weight): the differentiable backward below must see
        # tensors that are connected to the graph, not contiguous copies made for the kernel
        ctx.save_for_backward(pq, s, wd, b0, w1, masks)
        ctx.plan, ctx.npt = plan, npt
        return out

    @staticmethod
    def backward(ctx, g_out):
        pq, s, wd, b0, w1, masks = ctx.saved_tensors
        plan, npt = ctx.plan, ctx.npt
        g_out = _chk(g_out.contiguous())
        params = not _DATA_ONLY["on"]
        if torch.is_grad_enabled():                       # create_graph=True: the force pass, differentiated again later
            g_pq, gs, g_wd, g_b0 = EgnnEdgeBwdFn.apply(g_out, s, wd, w1, masks, plan, npt, params)
        else:
            g_pq, _, gs, g_wd, g_b0 = _raw_egnn_bwd_data(g_out, _chk(s), _chk(wd), _chk(w1), masks, plan, npt, params)
        g_w1 = g_b1 = None
        if params and (ctx.needs_input_grad[4] or ctx.needs_input_grad[5]):
            with torch.no_grad():
                g_w1, g_b1 = _raw_egnn_wgrad(g_out.detach(), _chk(pq), _chk(s), _chk(wd), _chk(b0), masks, plan, npt, False, True)
        return g_pq, gs, g_wd, g_b0, g_w1, g_b1, None


class EgnnEdgeBwdFn(torch.autograd.Function):
    """(g_out, s, w_d, W1) -> (g_pq, gs[, g_wd, g_b0]): the data side of the block's backward as a differentiable op.  Its own
    backward (the second backward pass of the force loss) is the block's TANGENT kernel plus two small parameter reductions:
    with u_e = ggP[row] + ggQ[col] + ggs_e w_d,  d/d g_out = sum_row mask2 (W1 (mask1 u_e)),  d/d W1 = sum_e gz2_e (mask1 u_e)^T,
    d/d w_d = sum_e ggs_e gz1_e.  (The masks make z1 / s enter only through constants: no gradient to s or P, Q here.)"""

    @staticmethod
    def forward(ctx, g_out, s, wd, w1, masks, plan, npt, params):
        wd, w1 = _chk(wd), _chk(w1)
        g_pq, gz1, gs, g_wd, g_b0 = _raw_egnn_bwd_data(_chk(g_out), _chk(s), wd, w1, masks, plan, npt, params)
        ctx.save_for_backward(g_out, wd, w1, masks, gz1)
        ctx.plan, ctx.npt, ctx.params = plan, npt, params
        ctx.mark_non_differentiable(*[t for t in (g_wd, g_b0) if t is not None])
        return g_pq, gs, g_wd, g_b0

    @staticmethod
    @once_differentiable
    def backward(ctx, gg_pq, gg_s, _gwd, _gb0):
        g_out, wd, w1, masks, gz1 = ctx.saved_tensors
        plan, npt = ctx.plan, ctx.npt
        n, h = g_out.shape
        if gg_pq is None:
            gg_pq = torch.zeros(n, 2 * h, dtype=g_out.dtype, device=g_out.device)
        if gg_s is None:
            gg_s = torch.zeros(plan.num_edges, dtype=g_out.dtype, device=g_out.device)
        gg_pq, gg_s = _chk(gg_pq.contiguous()), _chk(gg_s.contiguous())
        g_gout = _raw_egnn_fwd(gg_pq, gg_s, wd, None, w1, None, plan, npt, masks, True)
        g_w1 = g_wd = None
        if not _DATA_ONLY["on"]:
            g_w1, _ = _raw_egnn_wgrad(g_out, gg_pq, gg_s, wd, None, masks, plan, npt, True, False)
            g_wd = torch.empty(h, dtype=g_out.dtype, device=g_out.device)
            ws = _ws(_lib.query("hgb_weighted_colsum_workspace_bytes", h), g_out.device)
            _lib.call("hgb_weighted_colsum", _p(gz1), _p(gg_s), plan.num_edges, h, _p(g_wd), _p(ws), _stream())
        return g_gout, None, g_wd, g_w1, None, None, None, None


class EdgeLenFn(torch.autograd.Function):
    """d_e = |pos[col] - pos[row] + shift_e| (hydragnn/utils/model/operations.py:21-36, the ``radial`` of E_GCL).  Backward =
    ``EdgeLenBwdFn`` (differentiable once more: forces are differentiated by the MLIP loss)."""

    @staticmethod
    def forward(ctx, pos, shifts, plan):
        posc = _chk(pos)
        e = plan.num_edges
        ln = torch.empty(e, dtype=pos.dtype, device=pos.device)
        _lib.call("hgb_edge_geom_fwd", _p(posc), _p(plan.row), _p(plan.col), _p(_chk(shifts)), e, 0.0, None, _p(ln), None, _stream())
        ctx.save_for_backward(pos, shifts)              # the input itself: the differentiable backward must stay connected to it
        ctx.plan = plan
        return ln

    @staticmethod
    def backward(ctx, gd):
        pos, shifts = ctx.saved_tensors
        gd = _chk(gd.contiguous())
        if torch.is_grad_enabled():
            return EdgeLenBwdFn.apply(gd, pos, shifts, ctx.plan), None, None
        return _raw_edge_len_bwd(gd, _chk(pos), _chk(shifts), ctx.plan), None, None


def _edge_vec_scatter(gvec, plan):
    gpos = torch.empty(plan.num_nodes, 3, dtype=gvec.dtype, device=gvec.device)
    _lib.call("hgb_edge_vec_scatter", _p(gvec), _p(plan.by_col.rowptr), _p(plan.by_col.perm), _p(plan.by_row.rowptr), _p(plan.by_row.perm),
              plan.num_nodes, _p(gpos), _stream())
    return gpos


def _raw_edge_len_bwd(gd, pos, shifts, plan):
    gvec = torch.empty(plan.num_edges, 3, dtype=pos.dtype, device=pos.device)
    _lib.call("hgb_edge_len_bwd", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), _p(gd), plan.num_edges, _p(gvec), _stream())
    return _edge_vec_scatter(gvec, plan)


class EdgeLenBwdFn(torch.autograd.Function):
    """(gd, pos) -> g_pos = scatter(gd_e * vhat_e); its backward yields d/d gd = <vhat_e, ggpos[col] - ggpos[row]> and the
    curvature term d/d pos = scatter(gd_e (w_e - vhat <vhat, w_e>) / d_e)."""

    @staticmethod
    def forward(ctx, gd, pos, shifts, plan):
        gd, pos, shifts = _chk(gd), _chk(pos), _chk(shifts)
        ctx.save_for_backward(gd, pos, shifts)
        ctx.plan = plan
        return _raw_edge_len_bwd(gd, pos, shifts, plan)

    @staticmethod
    @once_differentiable
    def backward(ctx, ggpos):
        gd, pos, shifts = ctx.saved_tensors
        plan = ctx.plan
        e = plan.num_edges
        ggpos = _chk(ggpos.contiguous())
        g_gd = torch.empty(e, dtype=pos.dtype, device=pos.device)
        q = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        _lib.call("hgb_edge_len_bwd2", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), _p(gd), _p(ggpos), e, _p(g_gd), _p(q), _stream())
        g_pos = _edge_vec_scatter(q, plan) if ctx.needs_input_grad[1] else None
        return g_gd, g_pos, None, None


# =====================================================================================================
# MACE: fused tensor-product + scatter, symmetric contraction (first-order blocks)
# =====================================================================================================
def mace_tp_supported(lin, lsh, f):
    return 0 <= lin <= 2 and 1 <= lsh <= 3 and lin <= lsh and f % 32 == 0


class MaceTpScatterFn(torch.autograd.Function):
    """conv_tp + scatter-sum over receivers in one kernel (blocks.py:390-395).  up [N, S_in, F], sh [E, S_sh], tpw [E, P F];
    returns the packed message buffer (per output degree l3 a [N, 2l3+1, n_paths(l3) F] block)."""

    @staticmethod
    def forward(ctx, up, sh, tpw, plan, lin, lsh):
        up, sh, tpw = _chk(up.contiguous()), _chk(sh.contiguous()), _chk(tpw.contiguous())
        n, f = up.shape[0], up.shape[2]
        nacc = _lib.query("hgb_mace_tp_num_acc", lin, lsh)
        out = torch.empty(nacc * n * f, dtype=up.dtype, device=up.device)
        csr = plan.by_col
        _lib.call("hgb_mace_tp_scatter_fwd", _p(up), _p(sh), _p(tpw), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("col")), n, f, lin, lsh,
                  sh.shape[1], _p(out), _stream())
        ctx.save_for_backward(up, sh, tpw)
        ctx.plan, ctx.cfg = plan, (lin, lsh)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        up, sh, tpw = ctx.saved_tensors
        plan, (lin, lsh) = ctx.plan, ctx.cfg
        n, s_in, f = up.shape
        e = tpw.shape[0]
        g = _chk(g.contiguous())
        g_tpw = torch.empty_like(tpw)
        g_up_e = torch.empty(e, s_in * f, dtype=up.dtype, device=up.device)
        g_sh = torch.zeros_like(sh) if ctx.needs_input_grad[1] else None
        csr = plan.by_col
        _lib.call("hgb_mace_tp_scatter_bwd", _p(g), _p(up), _p(sh), _p(tpw), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("col")), n, f, lin,
                  lsh, sh.shape[1], _p(g_tpw), _p(g_up_e), _p(g_sh), _stream())
        g_up = raw_segment_sum(g_up_e, plan.by_row.rowptr, plan.by_row.perm, n).reshape(n, s_in, f) if ctx.needs_input_grad[0] else None
        return g_up, g_sh, g_tpw, None, None, None


def mace_sc_supported(lin, lout, correlation):
    return correlation == 2 and 1 <= lin <= 3 and 0 <= lout <= 2 and lout <= lin


class MaceSymContractFn(torch.autograd.Function):
    """SymmetricContraction, correlation 2, all output degrees at once.  x [N, S, F], wall [118, KTOT, F], zcsr: CSR of the
    element index."""

    @staticmethod
    def forward(ctx, x, wall, zcsr, lin, lout):
        x, wall = _chk(x.contiguous()), _chk(wall.contiguous())
        n, _, f = x.shape
        assert wall.shape[1] == _lib.query("hgb_mace_symcontract_num_weights", lin, lout)
        out = torch.empty(n, (lout + 1) ** 2, f, dtype=x.dtype, device=x.device)
        _lib.call("hgb_mace_symcontract_fwd", _p(x), _p(wall), _p(zcsr.idx), n, f, lin, lout, _p(out), _stream())
        ctx.save_for_backward(x, wall)
        ctx.zcsr, ctx.cfg = zcsr, (lin, lout)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, wall = ctx.saved_tensors
        zcsr, (lin, lout) = ctx.zcsr, ctx.cfg
        n, _, f = x.shape
        gx = torch.empty_like(x)
        gw_node = torch.empty(n, wall.shape[1] * f, dtype=x.dtype, device=x.device)
        _lib.call("hgb_mace_symcontract_bwd", _p(_chk(g.contiguous())), _p(x), _p(wall), _p(zcsr.idx), n, f, lin, lout, _p(gx), _p(gw_node),
                  _stream())
        gwall = raw_segment_sum(gw_node, zcsr.rowptr, zcsr.perm, zcsr.n).reshape(wall.shape)
        return gx, gwall, None, None, None


# ---- closed MACE primitives (any order of differentiation): csrc/hgb_mace_any.cu -----------------------------------------
def _tp_call(mode, p0, p1, p2, cg, out_shape):
    p0, p1, p2, cg = _chk(p0.contiguous()), _chk(p1.contiguous()), _chk(p2.contiguous()), _chk(cg.contiguous())
    ni, nj, nk = cg.shape
    e, f = p0.shape[0], p0.shape[2]
    out = torch.empty(out_shape, dtype=p0.dtype, device=p0.device)
    _lib.call("hgb_mace_tp_path", mode, _p(p0), _p(p1), _p(p2), _p(cg), e, f, ni, nj, nk, _p(out), _stream())
    return out


class TpOut(torch.autograd.Function):
    """o[e, k, f] = w[e, f] sum_ij C[i, j, k] a[e, i, f] y[e, j]: one tensor-product path on per-edge operands (blocks.py:386-392).
    Derivatives are TpOut (C permuted), TpY and TpW again: closed under autograd."""

    @staticmethod
    def forward(ctx, a, y, w, cg):
        ctx.save_for_backward(a, y, w, cg)
        return _tp_call(0, a, y, w, cg, (a.shape[0], cg.shape[2], a.shape[2]))

    @staticmethod
    def backward(ctx, g):
        a, y, w, cg = ctx.saved_tensors
        ga = TpOut.apply(g, y, w, cg.permute(2, 1, 0)) if ctx.needs_input_grad[0] else None
        gy = TpY.apply(a, g, w, cg) if ctx.needs_input_grad[1] else None
        gw = TpW.apply(a, y, g, cg) if ctx.needs_input_grad[2] else None
        return ga, gy, gw, None


class TpY(torch.autograd.Function):
    """o[e, j] = sum_f w[e, f] sum_ik C[i, j, k] a[e, i, f] g[e, k, f]"""

    @staticmethod
    def forward(ctx, a, g, w, cg):
        ctx.save_for_backward(a, g, w, cg)
        return _tp_call(1, a, g, w, cg, (a.shape[0], cg.shape[1]))

    @staticmethod
    def backward(ctx, gy):
        a, g, w, cg = ctx.saved_tensors
        ga = TpOut.apply(g, gy, w, cg.permute(2, 1, 0)) if ctx.needs_input_grad[0] else None
        gg = TpOut.apply(a, gy, w, cg) if ctx.needs_input_grad[1] else None
        gw = TpW.apply(a, gy, g, cg) if ctx.needs_input_grad[2] else None
        return ga, gg, gw, None


class TpW(torch.autograd.Function):
    """o[e, f] = sum_ijk C[i, j, k] a[e, i, f] y[e, j] g[e, k, f]"""

    @staticmethod
    def forward(ctx, a, y, g, cg):
        ctx.save_for_backward(a, y, g, cg)
        return _tp_call(2, a, y, g, cg, (a.shape[0], a.shape[2]))

    @staticmethod
    def backward(ctx, gw):
        a, y, g, cg = ctx.saved_tensors
        ga = TpOut.apply(g, y, gw, cg.permute(2, 1, 0)) if ctx.needs_input_grad[0] else None
        gy = TpY.apply(a, g, gw, cg) if ctx.needs_input_grad[1] else None
        gg = TpOut.apply(a, y, gw, cg) if ctx.needs_input_grad[2] else None
        return ga, gy, gg, None


def _chan_call(mode, p0, p1, n, f, p, ni, out_shape):
    p0, p1 = _chk(p0.contiguous()), _chk(p1.contiguous())
    out = torch.empty(out_shape, dtype=p0.dtype, device=p0.device)
    _lib.call("hgb_mace_chan_contract", mode, _p(p0), _p(p1), n, f, p, ni, _p(out), _stream())
    return out


class ChanCL(torch.autograd.Function):
    """o[b, c, p] = sum_i t[b, c, p, i] x[b, i, c] (one contraction step of symmetric_contraction.py:228-239)"""

    @staticmethod
    def forward(ctx, t, x):
        ctx.save_for_backward(t, x)
        n, f, p, ni = t.shape
        return _chan_call(0, t, x, n, f, p, ni, (n, f, p))

    @staticmethod
    def backward(ctx, g):
        t, x = ctx.saved_tensors
        return (ChanOU.apply(g, x) if ctx.needs_input_grad[0] else None), (ChanRP.apply(g, t) if ctx.needs_input_grad[1] else None)


class ChanOU(torch.autograd.Function):
    """o[b, c, p, i] = g[b, c, p] x[b, i, c]"""

    @staticmethod
    def forward(ctx, g, x):
        ctx.save_for_backward(g, x)
        n, f, p = g.shape
        ni = x.shape[1]
        return _chan_call(1, g, x, n, f, p, ni, (n, f, p, ni))

    @staticmethod
    def backward(ctx, go):
        g, x = ctx.saved_tensors
        return (ChanCL.apply(go, x) if ctx.needs_input_grad[0] else None), (ChanRP.apply(g, go) if ctx.needs_input_grad[1] else None)


class ChanRP(torch.autograd.Function):
    """o[b, i, c] = sum_p g[b, c, p] t[b, c, p, i]"""

    @staticmethod
    def forward(ctx, g, t):
        ctx.save_for_backward(g, t)
        n, f, p, ni = t.shape
        return _chan_call(2, g, t, n, f, p, ni, (n, ni, f))

    @staticmethod
    def backward(ctx, gx):
        g, t = ctx.saved_tensors
        return (ChanCL.apply(t, gx) if ctx.needs_input_grad[0] else None), (ChanOU.apply(g, gx) if ctx.needs_input_grad[1] else None)


class MaceEdgeEmbedFn(torch.autograd.Function):
    """(pos, shifts) -> (sh [E, (L+1)^2], radial [E, R]): spherical harmonics and Bessel x polynomial-cutoff basis of every edge in
    one kernel (first-order path; MACEStack.py:455-466, blocks.py:164-177), analytic d/dpos in the backward."""

    @staticmethod
    def forward(ctx, pos, shifts, plan, lmax, num_bessel, r_max, p):
        pos, shifts = _chk(pos), _chk(shifts)
        e = plan.num_edges
        ns = (lmax + 1) ** 2
        sh = torch.empty(e, ns, dtype=pos.dtype, device=pos.device)
        radial = torch.empty(e, num_bessel, dtype=pos.dtype, device=pos.device)
        _lib.call("hgb_mace_edge_embed_fwd", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), e, int(lmax), int(num_bessel), float(r_max),
                  float(p), _p(sh), _p(radial), _stream())
        ctx.save_for_backward(pos, shifts)
        ctx.plan, ctx.cfg = plan, (int(lmax), int(num_bessel), float(r_max), float(p))
        return sh, radial

    @staticmethod
    @once_differentiable
    def backward(ctx, g_sh, g_radial):
        pos, shifts = ctx.saved_tensors
        plan, (lmax, nb, rc, p) = ctx.plan, ctx.cfg
        e = plan.num_edges
        gvec = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        _lib.call("hgb_mace_edge_embed_bwd", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), _p(_chk(g_sh.contiguous())),
                  _p(_chk(g_radial.contiguous())), e, lmax, nb, rc, p, _p(gvec), _stream())
        return _edge_vec_scatter(gvec, plan), None, None, None, None, None, None


def adamw_step(p, g, m, v, step_dev, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_adamw_step", _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2), float(eps),
              float(weight_decay), float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())
