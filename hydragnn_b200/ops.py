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
from typing import NamedTuple

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
        if col_rowptr is not None and graph_ptr is not None:
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
            self._nbr[which] = gather_i32(idx, perm)
        return self._nbr[which]


def gather_i32(idx, perm):
    """``idx[perm]`` of two int32 vectors."""
    out = torch.empty_like(perm)
    _lib.call("hgb_gather_i32", _p(idx), _p(perm), perm.numel(), _p(out), _stream())
    return out


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
    nbytes = _lib.query("hgb_gemm_workspace_bytes", m, n, k, int(ta))
    ws = _ws(nbytes, a.device) if nbytes else None
    _lib.call("hgb_gemm", _p(a), _p(b), _p(out), m, n, k, int(ta), int(tb), a.stride(0), b.stride(0), out.stride(0),
              int(beta_one), _p(ws), nbytes, _stream())
    return out


def raw_colsum(x2d):
    m, n = x2d.shape
    out = torch.empty(n, dtype=x2d.dtype, device=x2d.device)
    ws = _ws(_lib.query("hgb_colsum_workspace_bytes", m, n), x2d.device)
    _lib.call("hgb_colsum", _p(x2d), m, n, _p(out), _p(ws), _stream())
    return out


# ---- tensor-core (wgmma) dense layers: plain TF32 under precision="bf16", the fp32-accurate 3xTF32 split otherwise -----
_TC = {"enabled": False}
_DATA_ONLY = {"on": False}     # inside ``only_data_grads()``: the force pass of the MLIP loss


class tensor_cores:
    """Context manager: run the large-M Linear layers of the wgmma kernels (hgb_tc_*) in plain TF32, not the 3xTF32 split."""

    def __init__(self, enabled=True):
        self.enabled, self.prev = bool(enabled), None

    def __enter__(self):
        self.prev = _TC["enabled"]
        _TC["enabled"] = self.enabled
        return self

    def __exit__(self, *exc):
        _TC["enabled"] = self.prev
        return False


def tc_wgrad_ok(m, n_out, k_out, *tensors):
    """dW = dZ^T X on the wgmma kernel (TF32 mode, or the 3xTF32 split in fp32 mode)"""
    return k_out + 16 <= 256 and tc_ok(m, n_out, k_out, *tensors)


def tc_ok(m, n_out, k_red, *tensors):
    if not _lib.query("hgb_tc_linear_supported", m, n_out, k_red):
        return False
    for t in tensors:
        if t is not None and (t.data_ptr() % 16 != 0 or (t.dim() == 2 and t.stride(0) % 4 != 0)):
            return False
    return True


def raw_tc_linear(a2, w, trans_b, bias, n_out, k_red, code=0, param=0.0, want_z=False, addend=None, gsrc=None, gact=0):
    m = a2.shape[0]
    for t in (addend, gsrc):             # the epilogue reads them with y's row stride n_out
        if t is not None and (tuple(t.shape) != (m, n_out) or not t.is_contiguous()):
            raise RuntimeError("raw_tc_linear: addend / gsrc must be dense row-major [%d, %d] tensors, got shape %s stride %s"
                               % (m, n_out, tuple(t.shape), t.stride()))
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


ACT_DERIV = 100   # HGB_ACT_DERIV: "the tensor already holds act'(.)"
RELU_SELECT = 101  # HGB_ACT_RELU_SELECT: the gradient through a ReLU as threshold_backward's select


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
# graph.  Inside ``deferred_weight_gradients()`` (the engine's step: FlatOptimizer.backward) the join of a LEAF parameter that has
# not received a gradient in this backward pass moves to the end of the pass (an autograd-engine callback): nothing reads such a
# gradient on the main stream before the optimizer (AccumulateGrad takes the tensor over without a kernel), so the weight-gradient
# kernels overlap everything that follows.  The inputs of the deferred kernels are kept referenced until the join, which stops
# autograd from accumulating into them in place (it only does that to tensors nobody else holds).  Derived weights (scaled, sliced,
# concatenated: MACE, PNAEq) are read by their own backward nodes right away -- those join immediately; so does everything outside
# the context, where gradient hooks (torch DDP's reducer, user hooks) may read a gradient the moment it is accumulated.
WGRAD_OVERLAP = True          # False: everything on the current stream (a profiler pass that attributes kernels to calls)
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
    """Context manager around ``loss.backward()`` of a step whose gradients are first read by ``FlatOptimizer.gather_grads``."""

    def __enter__(self):
        self.prev = _DEFER["on"]
        _DEFER["on"] = True
        return self

    def __exit__(self, *exc):
        _DEFER["on"] = self.prev
        join_side_streams()


def join_side_streams():
    """Join every side stream with deferred weight-gradient work (end of a backward pass; also called by FlatOptimizer.gather_grads)."""
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
    # the tensor-core epilogue reads dx_addend / dx_gsrc with dx's row stride k and hgb_act_bwd reads dx_gsrc as a flat array:
    # a column block of a wider tensor is copied to a dense [m, k] first
    dx_addend, dx_gsrc = _dense_2d(dx_addend, m, k), _dense_2d(dx_gsrc, m, k)

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


def _dense_2d(t, m, k):
    """``t`` (a [m, k] tensor or None) as a dense row-major [m, k] tensor, copying only if it is strided."""
    if t is None:
        return None
    if tuple(t.shape) != (m, k):
        raise RuntimeError("expected a [%d, %d] tensor, got %s" % (m, k, tuple(t.shape)))
    return _chk(t)


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
        # precision "bf16": plain TF32; "fp32": the 3xTF32 split inside the same kernel (exact flag)
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
    """``act(x W^T + b)``; for ``act = "prelu"`` ``act_param`` is the slope tensor (``LinearPReluFn``)."""
    if act == "prelu":
        return LinearPReluFn.apply(x, weight, bias, act_param)
    return LinearAct.apply(x, weight, bias, act, act_param)


def _prelu_bwd(g, z, slope, need_slope):
    """(dz, dslope) of y = prelu(z) in one ``hgb_prelu_bwd`` launch; dslope None when not needed or under ``only_data_grads``."""
    n = z.numel()
    need = need_slope and not _DATA_ONLY["on"]
    dz = torch.empty_like(z)
    if n == 0:
        return dz, (torch.zeros_like(slope) if need else None)
    dw = torch.empty_like(slope) if need else None
    ws = _ws(_lib.query("hgb_prelu_workspace_bytes", n), z.device) if need else None
    _lib.call("hgb_prelu_bwd", _p(_chk(g)), _p(z), n, _p(slope), _p(dz), _p(dw), _p(ws), 0 if need else 1, _stream())
    return dz, dw


class LinearPReluFn(torch.autograd.Function):
    """``prelu(x W^T + b)`` with one learnable slope (``nn.PReLU()``), the PReLU in the Linear's forward epilogue: the small-k and
    exact-fp32 kernels (``hgb_linear_smallk_fwd_prelu``, ``hgb_linear_fwd_prelu``) read the slope from device memory and store z
    next to y.  Where the tensor-core Linear takes the shape, the layer runs there without an activation and ``hgb_prelu_fwd``
    follows.  Backward: ``hgb_prelu_bwd`` (dz and the slope gradient, one launch), then the layer's plain backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, slope):
        if slope.numel() != 1:
            raise ValueError("LinearPReluFn: one shared slope (nn.PReLU()) expected, got %d" % slope.numel())
        shp = x.shape
        x2 = _row_major_2d(x)
        w = weight if weight.stride(1) == 1 else weight.contiguous()
        sl = _chk(slope)
        b = _chk(bias)
        m, k = x2.shape
        n = w.shape[0]
        if smallk_ok(n, k):
            y, z = torch.empty(m, n, dtype=x2.dtype, device=x2.device), torch.empty(m, n, dtype=x2.dtype, device=x2.device)
            _lib.call("hgb_linear_smallk_fwd_prelu", _p(x2), x2.stride(0), _p(w), w.stride(0), _p(b), m, n, k, _p(sl), _p(y), _p(z),
                      _stream())
        elif tc_ok(m, n, k, x2) and k <= 256:
            z, _ = raw_tc_linear(x2, w, False, b, n, k)
            y = torch.empty_like(z)
            if z.numel():
                _lib.call("hgb_prelu_fwd", _p(z), z.numel(), _p(sl), _p(y), _stream())
        else:
            y, z = torch.empty(m, n, dtype=x2.dtype, device=x2.device), torch.empty(m, n, dtype=x2.dtype, device=x2.device)
            _lib.call("hgb_linear_fwd_prelu", _p(x2), _p(w), _p(b), m, n, k, x2.stride(0), w.stride(0), _p(sl), _p(y), _p(z),
                      _stream())
        ctx.save_for_backward(x2, w, z, sl)
        ctx.shp, ctx.has_bias, ctx.tc = shp, bias is not None, _TC["enabled"]
        ctx.leaves = [weight] + ([bias] if bias is not None else [])
        return y.reshape(shp[:-1] + (n,))

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x2, w, z, sl = ctx.saved_tensors
        m, k = x2.shape
        n = w.shape[0]
        dz, dslope = _prelu_bwd(gy.reshape(m, n), z, sl, ctx.needs_input_grad[3])
        need = ctx.needs_input_grad
        if smallk_ok(n, k):
            gx, gw, gb = raw_smallk_bwd(dz, None, None, x2, w, 0, 0.0, need[0], need[1], ctx.has_bias and need[2])
        else:
            with tensor_cores(ctx.tc):
                gx, gw, gb = linear_bwd_dispatch(dz, x2, w, need[0], need[1], ctx.has_bias and need[2], leaves=ctx.leaves)
        if gx is not None:
            gx = gx.reshape(ctx.shp)
        return gx, gw, gb, (dslope.reshape(ctx.saved_tensors[3].shape) if dslope is not None else None)


class PReluFn(torch.autograd.Function):
    """``torch.nn.functional.prelu(x, weight)`` with one learnable slope (``nn.PReLU()``, the reference's "prelu").  The kernels
    read the slope from device memory (``hgb_prelu_fwd`` / ``hgb_prelu_bwd``), so no host synchronisation, and a captured step
    follows the optimiser's in-place updates.  The backward writes dx and the slope gradient in one launch, the latter a
    fixed-order sum (the same bits on every run); under ``only_data_grads`` it is skipped."""

    @staticmethod
    def forward(ctx, x, weight):
        if weight.numel() != 1:
            raise ValueError("PReluFn: one shared slope (nn.PReLU()) expected, got %d" % weight.numel())
        x, w = _chk(x), _chk(weight)
        y = torch.empty_like(x)
        if x.numel():
            _lib.call("hgb_prelu_fwd", _p(x), x.numel(), _p(w), _p(y), _stream())
        ctx.save_for_backward(x, w)
        ctx.wshape = weight.shape
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        n = x.numel()
        need_w = ctx.needs_input_grad[1] and not _DATA_ONLY["on"]
        if n == 0:
            return torch.zeros_like(x), (torch.zeros(ctx.wshape, dtype=w.dtype, device=w.device) if need_w else None)
        g = _chk(g)
        dx = torch.empty_like(x)
        dw = torch.empty(ctx.wshape, dtype=w.dtype, device=w.device) if need_w else None
        ws = _ws(_lib.query("hgb_prelu_workspace_bytes", n), x.device) if need_w else None
        _lib.call("hgb_prelu_bwd", _p(g), _p(x), n, _p(w), _p(dx), _p(dw), _p(ws), 0 if need_w else 1, _stream())
        return dx, dw


def prelu(x, weight, higher_order=False):
    """PReLU on the engine: ``PReluFn`` for first-order CUDA use, ATen's ``F.prelu`` (differentiable to any order) for the
    force-training path and CPU tensors."""
    if higher_order or not x.is_cuda:
        return torch.nn.functional.prelu(x, weight)
    return PReluFn.apply(x, weight)


def _mlp2_fwd(x2, w1, b1, c1, p1, w2, b2, c2, p2):
    """act2(act1(x2 W1^T + b1) W2^T + b2) -> (y, tensors to save, act1 config), the forward of Mlp2Fn and of the nodes that fold an
    activation next to it."""
    w1 = w1 if w1.stride(1) == 1 else w1.contiguous()
    w2 = w2 if w2.stride(1) == 1 else w2.contiguous()
    silu = ACT_CODES["silu"]
    h, z1, deriv = linear_fwd_dispatch_ex(x2, w1, _chk(b1), c1, p1, want_z=(c1 == silu), z_deriv=True)
    y, z2 = linear_fwd_dispatch(h, w2, _chk(b2), c2, p2, want_z=(c2 == silu))
    return y, [x2, w1, w2, h, z1, y if c2 not in (0, silu) else None, z2], (ACT_DERIV if deriv else c1, float(p1))


def _mlp2_bwd(dz2, saved, act1, need, leaves1, leaves2, dx_addend=None, dx_gsrc=None, dx_gact=0):
    """Backward of ``_mlp2_fwd`` from dz2 (the gradient at the second layer's pre-activation) -> (gx, gw1, gb1, gw2, gb2); the
    gradient through act1 runs in the epilogue of the second layer's data gradient.  need = (x, w1, b1, w2, b2); dx_*: as in
    linear_bwd_dispatch, for gx."""
    x2, w1, w2, h, z1 = saved[:5]
    c1, p1 = act1
    dz1, gw2, gb2 = linear_bwd_dispatch(dz2, h, w2, True, need[3], need[4], dx_gsrc=(z1 if c1 in (ACT_CODES["silu"], ACT_DERIV) else h),
                                        dx_gact=c1, dx_gparam=p1, leaves=leaves2)
    gx, gw1, gb1 = linear_bwd_dispatch(dz1, x2, w1, need[0], need[1], need[2], dx_addend=dx_addend, dx_gsrc=dx_gsrc, dx_gact=dx_gact,
                                       leaves=leaves1)
    return gx, gw1, gb1, gw2, gb2


def _leaves(w, b):
    return [w] + ([b] if b is not None else [])


class Mlp2Fn(torch.autograd.Function):
    """``act2(act1(x W1^T + b1) W2^T + b2)`` as one node: in the backward the gradient through act1 is applied in the epilogue of
    the second layer's data-gradient GEMM (no separate activation-backward pass over the hidden tensor)."""

    @staticmethod
    def forward(ctx, x, w1, b1, act1, p1, w2, b2, act2, p2):
        shp = x.shape
        c2 = ACT_CODES[act2]
        y, saved, ctx.act1 = _mlp2_fwd(_row_major_2d(x), w1, b1, ACT_CODES[act1], p1, w2, b2, c2, p2)
        ctx.save_for_backward(*saved)
        ctx.cfg = (c2, float(p2), shp, b1 is not None, b2 is not None)
        ctx.tc = _TC["enabled"]
        ctx.leaves1, ctx.leaves2 = _leaves(w1, b1), _leaves(w2, b2)
        return y.reshape(shp[:-1] + (w2.shape[0],))

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        saved = ctx.saved_tensors
        x2, w2, y, z2 = saved[0], saved[2], saved[5], saved[6]
        c2, p2, shp, has_b1, has_b2 = ctx.cfg
        gy2 = _chk(gy.reshape(x2.shape[0], w2.shape[0]))
        dz2 = raw_act_bwd(gy2, y, z2, c2, p2) if c2 != 0 else gy2
        nig = ctx.needs_input_grad
        with tensor_cores(ctx.tc):
            gx, gw1, gb1, gw2, gb2 = _mlp2_bwd(dz2, saved, ctx.act1, (nig[0], nig[1], has_b1 and nig[2], nig[5], has_b2 and nig[6]),
                                               ctx.leaves1, ctx.leaves2)
        return (gx.reshape(shp) if gx is not None else None), gw1, gb1, None, None, gw2, gb2, None, None


# ---- a PaiNN layer's closing ReLU folded into the passes next to it (C2: node_embed_out - ReLU - {next message | mean pool}) ----
def relu_embed_fold_ok(x, w1, w2):
    """True when relu(Linear - act - Linear) of x can run with the ReLU in the second Linear's tensor-core epilogue (TF32 mode),
    which gives torch.relu's bits."""
    m, k = x.shape
    return (_TC["enabled"] and x.is_cuda and x.dtype == torch.float32 and not smallk_ok(w2.shape[0], w1.shape[0])
            and tc_ok(m, w2.shape[0], w1.shape[0]) and w1.shape[0] <= 256)


class ReluMlp2PhiFn(torch.autograd.Function):
    """(s, phi) with s = relu(act1a(x W1a^T + b1a) W2a^T + b2a) -- a PaiNN layer's node_embed_out and the encoder's ReLU -- and
    phi = act1b(s W1b^T + b1b) W2b^T + b2b, the next layer's scalar-message MLP, as one node.  The ReLU runs in the epilogue of
    the Linear that writes s; in the backward the data gradient of phi's first Linear adds g_s (the message's passthrough
    gradient of s) and applies the ReLU's select in its epilogue, which is the gradient at s's pre-activation.  Every value has
    the bits of Mlp2Fn - torch.relu - Mlp2Fn with autograd's sum of the two gradients of s."""

    @staticmethod
    def forward(ctx, x, w1a, b1a, act1a, p1a, w2a, b2a, w1b, b1b, act1b, p1b, w2b, b2b):
        x2 = _row_major_2d(x)
        s, saved_a, ctx.act_a = _mlp2_fwd(x2, w1a, b1a, ACT_CODES[act1a], p1a, w2a, b2a, ACT_CODES["relu"], 0.0)
        phi, saved_b, ctx.act_b = _mlp2_fwd(s, w1b, b1b, ACT_CODES[act1b], p1b, w2b, b2b, 0, 0.0)
        ctx.save_for_backward(*saved_a, *saved_b)
        ctx.cfg = (x.shape, b1a is not None, b2a is not None, b1b is not None, b2b is not None)
        ctx.tc = _TC["enabled"]
        ctx.leaves = (_leaves(w1a, b1a), _leaves(w2a, b2a), _leaves(w1b, b1b), _leaves(w2b, b2b))
        return s, phi

    @staticmethod
    @once_differentiable
    def backward(ctx, g_s, g_phi):
        saved = ctx.saved_tensors
        saved_a, saved_b = saved[:7], saved[7:]
        s = saved_a[5]
        shp, hb1a, hb2a, hb1b, hb2b = ctx.cfg
        nig = ctx.needs_input_grad
        la1, la2, lb1, lb2 = ctx.leaves
        with tensor_cores(ctx.tc):
            dz2a, gw1b, gb1b, gw2b, gb2b = _mlp2_bwd(_chk(g_phi), saved_b, ctx.act_b, (True, nig[7], hb1b and nig[8], nig[11], hb2b and nig[12]),
                                                     lb1, lb2, dx_addend=_chk(g_s), dx_gsrc=s, dx_gact=RELU_SELECT)
            gx, gw1a, gb1a, gw2a, gb2a = _mlp2_bwd(dz2a, saved_a, ctx.act_a, (nig[0], nig[1], hb1a and nig[2], nig[5], hb2a and nig[6]),
                                                   la1, la2)
        return ((gx.reshape(shp) if gx is not None else None), gw1a, gb1a, None, None, gw2a, gb2a, gw1b, gb1b, None, None, gw2b, gb2b)


class ReluMlp2MeanPoolFn(torch.autograd.Function):
    """mean_pool(relu(act1(x W1^T + b1) W2^T + b2)) over the graphs of a sorted batch as one node: the ReLU runs in the second
    Linear's epilogue, and the pool's backward applies the ReLU's select while it broadcasts, which is the gradient at the second
    Linear's pre-activation; from there the backward is Mlp2Fn's.  Bits of Mlp2Fn - torch.relu - PoolFn."""

    @staticmethod
    def forward(ctx, x, w1, b1, act1, p1, w2, b2, gcsr):
        x2 = _row_major_2d(x)
        y, saved, ctx.act1 = _mlp2_fwd(x2, w1, b1, ACT_CODES[act1], p1, w2, b2, ACT_CODES["relu"], 0.0)
        g, c = gcsr.n, y.shape[1]
        out = torch.empty(g, c, dtype=y.dtype, device=y.device)
        _lib.call("hgb_pool_fwd", _p(y), _p(gcsr.rowptr), g, c, POOL_CODES["mean"], _p(out), None, _stream())
        ctx.save_for_backward(*saved)
        ctx.gcsr, ctx.cfg, ctx.tc = gcsr, (x.shape, b1 is not None, b2 is not None), _TC["enabled"]
        ctx.leaves1, ctx.leaves2 = _leaves(w1, b1), _leaves(w2, b2)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        saved = ctx.saved_tensors
        y = saved[5]
        shp, has_b1, has_b2 = ctx.cfg
        g = _chk(g)
        dz2 = torch.empty_like(y)
        _lib.call("hgb_pool_bwd", _p(g), _p(ctx.gcsr.rowptr), None, _p(y), y.shape[0], ctx.gcsr.n, y.shape[1], POOL_CODES["mean"],
                  _p(dz2), _stream())
        nig = ctx.needs_input_grad
        with tensor_cores(ctx.tc):
            gx, gw1, gb1, gw2, gb2 = _mlp2_bwd(dz2, saved, ctx.act1, (nig[0], nig[1], has_b1 and nig[2], nig[5], has_b2 and nig[6]),
                                               ctx.leaves1, ctx.leaves2)
        return (gx.reshape(shp) if gx is not None else None), gw1, gb1, None, None, gw2, gb2, None


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
    if (act2 is None and b1 is not None and b2 is not None and x.dim() == 2 and x.shape[1] == 1
            and w1.shape == (1, 1) and w2.shape[1] == 1 and w2.shape[0] <= 4):
        return Mlp2ScalarFn.apply(x, w1, b1, act1, p1, w2, b2)          # width-1 layer (quirk Q4)
    return Mlp2Fn.apply(x, w1, b1, act1, p1, w2, b2, act2, p2)


class EdgeGeomFn(torch.autograd.Function):
    """(vec, len, unit) of hydragnn/utils/model/operations.py:21-36 in one pass; the backward turns the
    three edge gradients into one [E,3] vector and scatters it to both endpoints with segment sums.  Without edges no
    kernel runs."""

    @staticmethod
    def forward(ctx, pos, shifts, plan, eps):
        pos = _chk(pos)
        e = plan.num_edges
        vec = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        ln = torch.empty(e, 1, dtype=pos.dtype, device=pos.device)
        unit = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        if e > 0:
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
        g_pos = g_shift = None
        if plan.num_edges == 0:
            return (vec.new_zeros(plan.num_nodes, 3) if ctx.needs_input_grad[0] else None), \
                (gv if ctx.needs_input_grad[1] else None), None, None
        _lib.call("hgb_edge_geom_bwd", _p(vec), _p(ln), ctx.eps, _p(_chk(g_vec)), _p(_chk(g_len)), _p(_chk(g_unit)),
                  plan.num_edges, _p(gv), _stream())
        if ctx.needs_input_grad[0]:
            # vec = pos[col] - pos[row] + shift
            g_pos = raw_segment_sum(gv, plan.by_col.rowptr, plan.by_col.perm, plan.num_nodes) - \
                raw_segment_sum(gv, plan.by_row.rowptr, plan.by_row.perm, plan.num_nodes)
        if ctx.needs_input_grad[1]:
            g_shift = gv
        return g_pos, g_shift, None, None


class PainnEdgeEmbedFn(torch.autograd.Function):
    """len/unit -> one 12-float record per edge {rbf*cutoff (8, zero padded), cutoff, dir = unit/len [quirk Q2]}
    (hydragnn/models/PAINNStack.py:239-242,257).  Without edges no kernel runs."""

    @staticmethod
    def forward(ctx, unit, ln, num_radial, cutoff):
        e = unit.shape[0]
        epack = torch.empty(e, 12, dtype=unit.dtype, device=unit.device)
        if e > 0:
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
        if e > 0:
            _lib.call("hgb_painn_edge_embed_bwd", _p(unit), _p(ln), _p(_chk(g_epack)), e, ctx.r, ctx.cutoff, _p(g_unit), _p(g_len), _stream())
        return g_unit, g_len, None, None


class AffineV(NamedTuple):
    """The layer input v[n, k, c] = v0[n, k, 0] * weight[c, 0] + bias[c] (a Linear(1, F) of a [N, 3, 1] tensor: PaiNN's first
    vec_embed_out), kept unevaluated so that the message kernels can form it on chip."""
    v0: torch.Tensor
    weight: torch.Tensor
    bias: torch.Tensor

    def materialize(self, higher_order=False):
        return linear_any_order(self.v0, self.weight, self.bias) if higher_order else linear_act(self.v0, self.weight, self.bias)


def painn_affine_v_ok(v, s, rec_row):
    """True when the tiled message kernels can take ``v`` as its AffineV record."""
    n, f = s.shape
    return (isinstance(v, AffineV) and rec_row is not None and s.is_cuda and v.v0.is_contiguous() and v.v0.data_ptr() % 16 == 0
            and bool(_lib.query("hgb_painn_message_affine_v_supported", n, f)))


class PainnMessageFn(torch.autograd.Function):
    """Fused PaiNN message (hydragnn/models/PAINNStack.py:239-270): returns (s + ds, v + dv).  The input v is either a
    [n, 3, f] tensor (``v0 = vw = vb = None``) or, with ``v = None``, the affine v0 [n, 3, 1], vw [f, 1], vb [f] of an
    ``AffineV`` (``painn_affine_v_ok``).  Without nodes or edges no kernel runs: s and v pass through unchanged."""

    @staticmethod
    def forward(ctx, phi, s, v, epack, wf, bf, efilt, plan, rec_row=None, v0=None, vw=None, vb=None):
        n, f = s.shape
        r = wf.shape[1]
        phi, s = _chk(phi), _chk(s)
        av = v0 is not None
        if av:
            v, v0, vw, vb = None, _chk(v0), _chk(vw), _chk(vb)
        else:
            v = _chk(v)
        agg = plan.by_row     # messages are summed into edge[:,0] = edge_index[0]
        if n == 0 or plan.num_edges == 0:
            s_out = s.clone()
            v_out = linear_act(v0, vw, vb) if av else v.clone()
        else:
            s_out = torch.empty_like(s)
            v_out = torch.empty(n, 3, f, dtype=s.dtype, device=s.device)
            _lib.call("hgb_painn_message_fwd", _p(phi), _p(s), _p(v), _p(v0), _p(vw), _p(vb), _p(agg.rowptr), _p(agg.perm),
                      _p(plan.nbr("row")), _p(epack), _p(rec_row), _p(_chk(wf)), _p(_chk(bf)), _p(_chk(efilt)), n, f, r, _p(s_out),
                      _p(v_out), _stream())
        ctx.save_for_backward(phi, v, epack, wf, bf, efilt, v0, vw, vb)
        ctx.plan, ctx.use_rec = plan, rec_row is not None
        return s_out, v_out

    @staticmethod
    @once_differentiable
    def backward(ctx, gs_out, gv_out):
        phi, v, epack, wf, bf, efilt, v0, vw, vb = ctx.saved_tensors
        plan = ctx.plan
        n, f = gs_out.shape
        r = wf.shape[1]
        gs_out, gv_out = _chk(gs_out), _chk(gv_out)
        need_edge = ctx.needs_input_grad[3]
        e = plan.num_edges
        if n == 0 or e == 0:
            g_epack = torch.zeros_like(epack) if need_edge else None
            g_ef = torch.zeros_like(efilt) if efilt is not None else None
            return PainnMessageFn._grads(ctx, torch.zeros_like(phi), gs_out, gv_out, g_epack, torch.zeros_like(wf),
                                         torch.zeros_like(bf), g_ef, v0, vw)
        gphi = torch.empty_like(phi)
        gv = torch.empty(n, 3, f, dtype=phi.dtype, device=phi.device)
        gwf, gbf = torch.empty_like(wf), torch.empty_like(bf)
        g_epack = torch.empty_like(epack) if need_edge else None
        g_ef = torch.empty_like(efilt) if efilt is not None else None
        nbytes = _lib.query("hgb_painn_message_bwd_workspace_bytes", n, f, r, e)
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
        _lib.call("hgb_painn_message_bwd", _p(gs_out), _p(gv_out), _p(phi), _p(v), _p(v0), _p(vw), _p(vb), _p(src.rowptr),
                  _p(src.perm), _p(plan.nbr("col")), _p(epack), _p(rec_col), _p(wf), _p(bf), _p(efilt), n, f, r, e, _p(gphi),
                  _p(gv), _p(gwf), _p(gbf), _p(g_epack), _p(g_ef), _p(ws), nbytes, _stream())
        return PainnMessageFn._grads(ctx, gphi, gs_out, gv, g_epack, gwf, gbf, g_ef, v0, vw)

    @staticmethod
    def _grads(ctx, gphi, gs_out, gv, g_epack, gwf, gbf, g_ef, v0, vw):
        n, f = gs_out.shape
        if v0 is None:
            return gphi, gs_out, gv, g_epack, gwf, gbf, g_ef, None, None, None, None, None
        # v = Linear(1, f)(v0): the same small-k backward LinearAct runs on a stored v, so all three gradients keep its bits
        g_v0, g_vw, g_vb = raw_smallk_bwd(gv.reshape(3 * n, f), None, None, v0.reshape(3 * n, 1), vw, 0, 0.0,
                                          ctx.needs_input_grad[9], ctx.needs_input_grad[10], ctx.needs_input_grad[11])
        return gphi, gs_out, None, g_epack, gwf, gbf, g_ef, None, None, (g_v0.reshape(v0.shape) if g_v0 is not None else None), g_vw, g_vb


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


def painn_update_tc_ok(s, v):
    """``PainnUpdateTcFn`` runs the block: TF32 mode, f = 64, as many rows as the tensor-core Linears take, dense 16-byte aligned
    fp32 CUDA tensors."""
    n, f = s.shape
    return (_TC["enabled"] and f == 64 and tuple(v.shape) == (n, 3, f) and s.is_cuda and v.is_cuda
            and s.dtype == torch.float32 and v.dtype == torch.float32 and s.is_contiguous() and v.is_contiguous()
            and s.data_ptr() % 16 == 0 and v.data_ptr() % 16 == 0 and bool(_lib.query("hgb_tc_linear_supported", n, f, 2 * f)))


def _aligned(t):
    """dense and 16-byte aligned (a view at an odd offset is copied)"""
    t = _chk(t)
    return t if t.data_ptr() % 16 == 0 else t.clone()


class PainnUpdateTcFn(torch.autograd.Function):
    """``PainnUpdateFn`` at f = 64 in TF32 mode without the [3n, 2f] U/V product in memory (csrc/hgb_painn_tc.cu): each step of the
    block recomputes [uv | vv] from v on the tensor cores for its 64-node tiles and reduces over the three spatial rows in registers.
    Forward: [|vv|, s] -> update_mlp (tc_linear) -> s_out (v_out).  Backward: ga -> the update_mlp backward -> [guv | gvv] and gv, the
    U/V data gradient, in one kernel; the U/V weight gradient still reads [guv | gvv] on the side stream.  Same bits as
    ``PainnUpdateFn``."""

    @staticmethod
    def forward(ctx, s, v, uw, ub, vw, vb, w1, b1, w2, b2, last):
        n, f = s.shape
        w1, b1, w2, b2 = [_chk(t) for t in (w1, b1, w2, b2)]
        wuv, buv = torch.cat([uw, vw], dim=0).contiguous(), torch.cat([ub, vb], dim=0).contiguous()
        mlp_in = torch.empty(n, 2 * f, dtype=s.dtype, device=s.device)
        inner = torch.empty_like(s) if last else None       # a last layer's post and ga read it instead of recomputing [uv | vv]
        _lib.call("hgb_painn_update_tc_fwd", _p(v), _p(s), _p(wuv), _p(buv), n, _p(mlp_in), _p(inner), _stream())
        h, z1, deriv = linear_fwd_dispatch_ex(mlp_in, w1, b1, ACT_CODES["silu"], 0.0, want_z=True, z_deriv=True)
        a, _ = linear_fwd_dispatch(h, w2, b2)
        ctx.z1_code = ACT_DERIV if deriv else ACT_CODES["silu"]
        s_out = torch.empty_like(s)
        v_out = None if last else torch.empty_like(v)
        _lib.call("hgb_painn_update_tc_post", _p(v), _p(s), _p(a), _p(inner), _p(wuv), _p(buv), n, int(last), _p(s_out), _p(v_out),
                  _stream())
        ctx.save_for_backward(v, mlp_in, z1, h, a, wuv, buv, w1, w2, inner)
        ctx.last = bool(last)
        ctx.leaves = ([uw, ub, vw, vb], [w1, b1], [w2, b2])
        if last:
            return s_out, s_out.new_zeros(0)
        return s_out, v_out

    @staticmethod
    @once_differentiable
    def backward(ctx, gs_out, gv_out):
        v, mlp_in, z1, h, a, wuv, buv, w1, w2, inner = ctx.saved_tensors
        last = ctx.last
        n, f = mlp_in.shape[0], v.shape[2]
        gs_out = _aligned(gs_out)
        gv_out = None if last else _aligned(gv_out)
        ga = torch.empty_like(a)
        _lib.call("hgb_painn_update_tc_bwd_a", _p(v), _p(gs_out), _p(gv_out), _p(inner), _p(wuv), _p(buv), n, int(last), _p(ga), _stream())
        with tensor_cores(True):
            gz1, gw2, gb2 = linear_bwd_dispatch(ga, h, w2, dx_gsrc=z1, dx_gact=ctx.z1_code, leaves=ctx.leaves[2])     # dgrad through the SiLU
            g_mlp_in, gw1, gb1 = linear_bwd_dispatch(gz1, mlp_in, w1, leaves=ctx.leaves[1])
        g_uv = torch.empty(3 * n, 2 * f, dtype=v.dtype, device=v.device)            # [guv | gvv]
        gs, gv = torch.empty_like(gs_out), torch.empty_like(v)
        _lib.call("hgb_painn_update_tc_bwd", _p(v), _p(gs_out), _p(gv_out), _p(g_mlp_in), _p(a), _p(mlp_in), _p(wuv), _p(buv), n, int(last),
                  _p(g_uv), _p(gs), _p(gv), _stream())
        with tensor_cores(True):
            _, gwuv, gbuv = linear_bwd_dispatch(g_uv, v.reshape(3 * n, f), wuv, need_x=False, leaves=ctx.leaves[0])
        return gs, gv, gwuv[:f], gbuv[:f], gwuv[f:], gbuv[f:], gw1, gb1, gw2, gb2, None


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
        _lib.call("hgb_pool_bwd", _p(g), _p(ctx.gcsr.rowptr), _p(ctx.arg), None, ctx.n, ctx.gcsr.n, g.shape[1], ctx.code, _p(gx),
                  _stream())
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


GNLL_EPS = 1e-6          # torch.nn.GaussianNLLLoss's default, the one the reference's loss_function_selection builds


class GaussianNLLFn(torch.autograd.Function):
    """``torch.nn.GaussianNLLLoss()(mean, target, var)`` (full=False, eps=1e-6, mean) with the gradients with respect to mean and
    var produced in the same pass (``hgb_gnll_fwd_bwd``).  ``valid_rows`` / ``row_width``: mean over the real prefix rows of a
    capacity-padded batch, as ``LossFn``."""

    @staticmethod
    def forward(ctx, mean, var, target, valid_rows=None, row_width=1):
        mean, var, target = _chk(mean), _chk(var), _chk(target)
        n = mean.numel()
        if var.numel() != n or target.numel() != n:
            raise ValueError("GaussianNLLFn: mean, var and target need the same number of elements (%d, %d, %d)"
                             % (n, var.numel(), target.numel()))
        loss = torch.empty(1, dtype=mean.dtype, device=mean.device)
        gmean, gvar = torch.empty_like(mean), torch.empty_like(var)
        ws = torch.empty(int(_lib.query("hgb_gnll_workspace_bytes", n)), dtype=torch.uint8, device=mean.device)
        _lib.call("hgb_gnll_fwd_bwd", _p(mean), _p(var), _p(target), n, GNLL_EPS, _p(loss), _p(gmean), _p(gvar), _p(ws),
                  _p(valid_rows), int(row_width), _stream())
        ctx.save_for_backward(gmean, gvar)
        return loss.reshape(())

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        gmean, gvar = ctx.saved_tensors
        return gmean * g, gvar * g, None, None, None


def gaussian_nll_any_order(mean, var, target, mask=None, count=None):
    """The same loss composed from ATen, differentiable to any order, on any device: ``var`` clamped to ``GNLL_EPS`` in value
    while its gradient passes through unchanged (torch clamps a copy under no_grad).  With ``mask`` (0/1 per element) the sum
    of the masked terms is divided by ``count`` instead of taking the mean."""
    vc = torch.where(var >= GNLL_EPS, var, var - var.detach() + GNLL_EPS)
    d = mean - target
    term = 0.5 * (torch.log(vc) + d * d / vc)
    return term.mean() if mask is None else (term * mask).sum() / count


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


PNA_CONV_MAX_EDGE_DIM = 16


def raw_pna_conv_fwd(pq, eattr, mt, cvec, plan):
    """-> (agg [n, 4f], argmin, argmax [n, f] int32): hgb_pna_conv_fwd over the by-target CSR of ``plan``."""
    n, f = pq.shape[0], pq.shape[1] // 2
    d = 0 if eattr is None else eattr.shape[1]
    col = plan.by_col
    agg = torch.empty(n, 4 * f, dtype=pq.dtype, device=pq.device)
    amin = torch.empty(n, f, dtype=torch.int32, device=pq.device)
    amax = torch.empty_like(amin)
    _lib.call("hgb_pna_conv_fwd", _p(pq), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d, _p(mt), _p(cvec), n, f,
              _p(agg), _p(amin), _p(amax), _stream())
    return agg, amin, amax


def raw_pna_conv_bwd(g_agg, pq, eattr, mt, cvec, agg, amin, amax, plan):
    """-> (g_pq [n, 2f], g_h [e, f], g_cm [1 + d, f] = [g_c ; g_M^T])."""
    n, f = pq.shape[0], pq.shape[1] // 2
    d = 0 if eattr is None else eattr.shape[1]
    dev = pq.device
    g_pq = torch.empty(n, 2 * f, dtype=pq.dtype, device=dev)
    g_h = torch.empty(plan.num_edges, f, dtype=pq.dtype, device=dev)
    g_cm = torch.empty(1 + d, f, dtype=pq.dtype, device=dev)
    ws = _ws(_lib.query("hgb_pna_conv_workspace_bytes", f, d), dev)
    col = plan.by_col
    _lib.call("hgb_pna_conv_bwd", _p(g_agg), _p(pq), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d, _p(mt), _p(cvec),
              _p(agg), _p(amin), _p(amax), n, f, _p(g_pq), 2 * f, _p(g_h), _p(g_cm), _p(ws), _stream())
    # g_Q: Q was gathered by the source of every edge, so its gradient is the by-source segment sum of g_h
    row = plan.by_row
    _lib.call("hgb_segment_sum_strided", _p(g_h), _p(row.rowptr), _p(row.perm), n, f, _p(g_pq[:, f:]), 2 * f, _stream())
    return g_pq, g_h, g_cm


class PnaConvFn(torch.autograd.Function):
    """agg = [mean | min | max | std] over the targets i = edge_index[1] of h_e = P[i] + Q[j] + M a_e + c, with
    [P | Q] = ``pq`` [n, 2f], M = ``mt``ᵀ [f, d] and c = ``cvec`` [f] -- PNAConv's pre_nn Linear and its four aggregators
    (torch_geometric 2.6.1 PNAConv.message / DegreeScalerAggregation) in one kernel; the [E, f] messages never reach memory.
    ``eattr`` [e, d] with d <= 16, or None."""

    @staticmethod
    def forward(ctx, pq, eattr, mt, cvec, plan):
        pq, cvec = _chk(pq), _chk(cvec)
        eattr = _chk(eattr) if eattr is not None else None
        mt = _chk(mt) if eattr is not None else None
        agg, amin, amax = raw_pna_conv_fwd(pq, eattr, mt, cvec, plan)
        ctx.save_for_backward(pq, eattr, mt, cvec, agg, amin, amax)
        ctx.plan = plan
        return agg

    @staticmethod
    @once_differentiable
    def backward(ctx, g_agg):
        pq, eattr, mt, cvec, agg, amin, amax = ctx.saved_tensors
        g_pq, g_h, g_cm = raw_pna_conv_bwd(_chk(g_agg.contiguous()), pq, eattr, mt, cvec, agg, amin, amax, ctx.plan)
        g_eattr = g_mt = None
        if eattr is not None:
            g_mt = g_cm[1:]
            if ctx.needs_input_grad[1]:
                g_eattr = raw_gemm(g_h, mt, False, True)                           # [e, f] x [d, f]^T
        return g_pq, g_eattr, g_mt, g_cm[0], None


def pnaplus_conv_supported(f, r, d):
    """Shapes ``PnaPlusConvFn`` takes: 1 <= f <= 64, 1 <= num_radial <= 16, edge input width d <= 16."""
    return bool(_lib.query("hgb_pnaplus_conv_supported", int(f), int(r), int(d)))


def raw_pnaplus_conv_fwd(pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, radius, expo, plan):
    """-> (agg [n, 4f], argmin, argmax [n, f] int32): hgb_pnaplus_conv_fwd over the by-target CSR of ``plan``."""
    n, f = pq.shape[0], pq.shape[1] // 2
    d, r = (0 if eattr is None else eattr.shape[1]), freq.numel()
    col = plan.by_col
    agg = torch.empty(n, 4 * f, dtype=pq.dtype, device=pq.device)
    amin = torch.empty(n, f, dtype=torch.int32, device=pq.device)
    amax = torch.empty_like(amin)
    _lib.call("hgb_pnaplus_conv_fwd", _p(pq), _p(dist), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d, _p(freq), r,
              float(radius), int(expo), _p(wr), _p(br), _p(wl), _p(mr), _p(mat), _p(cvec), n, f, _p(agg), _p(amin), _p(amax), _stream())
    return agg, amin, amax


def raw_pnaplus_conv_bwd(g_agg, pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, radius, expo, agg, amin, amax, plan,
                         need_dist=True, need_eattr=True, need_params=True):
    """-> (g_pq [n, 2f], g_dist [e] or None, g_eattr [e, d] or None, g_params or None); g_params is laid out as
    [c f | mat d*f | mr f*f | wr^T r*f | br f | wl^T r*f | freq r] (include/hgb.h)."""
    n, f = pq.shape[0], pq.shape[1] // 2
    d, r, e = (0 if eattr is None else eattr.shape[1]), freq.numel(), plan.num_edges
    dev = pq.device
    g_pq = torch.empty(n, 2 * f, dtype=pq.dtype, device=dev)
    g_h = torch.empty(e, f, dtype=pq.dtype, device=dev)
    g_dist = torch.empty(e, dtype=pq.dtype, device=dev) if need_dist else None
    g_eattr = torch.empty(e, d, dtype=pq.dtype, device=dev) if (need_eattr and d > 0) else None
    g_params = torch.empty(f + d * f + f * f + 2 * r * f + f + r, dtype=pq.dtype, device=dev) if need_params else None
    ws = _ws(_lib.query("hgb_pnaplus_conv_workspace_bytes", f, r, d), dev) if need_params else None
    col = plan.by_col
    _lib.call("hgb_pnaplus_conv_bwd", _p(g_agg), _p(pq), _p(dist), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d,
              _p(freq), r, float(radius), int(expo), _p(wr), _p(br), _p(wl), _p(mr), _p(mat), _p(cvec), _p(agg), _p(amin), _p(amax),
              n, f, _p(g_pq), 2 * f, _p(g_h), _p(g_dist), _p(g_eattr), _p(g_params), _p(ws), _stream())
    row = plan.by_row          # Q was gathered by the source of every edge: g_Q is the by-source segment sum of g_h
    _lib.call("hgb_segment_sum_strided", _p(g_h), _p(row.rowptr), _p(row.perm), n, f, _p(g_pq[:, f:]), 2 * f, _stream())
    return g_pq, g_dist, g_eattr, g_params


class PnaPlusConvFn(torch.autograd.Function):
    """agg = [mean | min | max | std] over the targets i = edge_index[1] of PNAPlus's message (hydragnn/models/PNAPlusStack.py
    :233-263) m_e = (P[i] + Q[j] + M_r relu(W_r rbf_e + b_r) + M_a a_e + c) * (W_l rbf_e), with rbf_e the Bessel basis of the
    edge length ``dist`` [e] (torch_geometric 2.6.1 BesselBasisLayer: ``freq`` [r], ``radius``, envelope exponent ``expo``).
    [P | Q] = ``pq`` [n, 2f]; ``wr`` / ``wl`` [f, r], ``br`` [f], ``mr`` [f, f], ``mat`` = M_a^T [d, f] (None without edge
    input), ``cvec`` [f].  One kernel each way; neither the basis, the embedding nor the message reaches memory."""

    @staticmethod
    def forward(ctx, pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, radius, expo, plan):
        pq, dist, freq, wr, br, wl, mr, cvec = (_chk(t) for t in (pq, dist, freq, wr, br, wl, mr, cvec))
        eattr = _chk(eattr) if eattr is not None else None
        mat = _chk(mat) if eattr is not None else None
        agg, amin, amax = raw_pnaplus_conv_fwd(pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, radius, expo, plan)
        ctx.save_for_backward(pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, agg, amin, amax)
        ctx.radius, ctx.expo, ctx.plan = float(radius), int(expo), plan
        return agg

    @staticmethod
    @once_differentiable
    def backward(ctx, g_agg):
        pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec, agg, amin, amax = ctx.saved_tensors
        need = ctx.needs_input_grad
        need_params = any(need[3:10]) and not _DATA_ONLY["on"]
        g_pq, g_dist, g_eattr, gp = raw_pnaplus_conv_bwd(_chk(g_agg.contiguous()), pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec,
                                                         ctx.radius, ctx.expo, agg, amin, amax, ctx.plan, need_dist=need[1],
                                                         need_eattr=eattr is not None and need[2], need_params=need_params)
        if gp is None:
            return g_pq, g_dist, g_eattr, None, None, None, None, None, None, None, None, None, None
        f, r = pq.shape[1] // 2, freq.numel()
        d = 0 if eattr is None else eattr.shape[1]
        sizes = [f, d * f, f * f, r * f, f, r * f, r]
        g_c, g_mat, g_mr, g_wrt, g_br, g_wlt, g_freq = torch.split(gp, sizes)
        return (g_pq, g_dist, g_eattr, g_freq, g_wrt.view(r, f).t(), g_br, g_wlt.view(r, f).t(), g_mr.view(f, f),
                g_mat.view(d, f) if eattr is not None else None, g_c, None, None, None)


def cgconv_supported(f, d):
    """Shapes ``CgConvFn`` takes: 1 <= f <= 128 channels, edge input width 0 <= d <= 16."""
    return bool(_lib.query("hgb_cgconv_supported", int(f), int(d)))


def raw_cgconv_fwd(pq, eattr, mt, cvec, x, plan):
    """-> out [n, f] = x + sum over the targets of sigmoid(f_e) * softplus(s_e): hgb_cgconv_fwd over the by-target CSR."""
    n, f = x.shape
    d = 0 if eattr is None else eattr.shape[1]
    col = plan.by_col
    out = torch.empty_like(x)
    _lib.call("hgb_cgconv_fwd", _p(pq), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d, _p(mt), _p(cvec), _p(x),
              n, plan.num_edges, f, _p(out), _stream())
    return out


def raw_cgconv_bwd(g_out, pq, eattr, mt, cvec, plan, need_eattr=True, need_params=True):
    """-> (g_pq [n, 4f], g_eattr [e, d] or None, g_params [1 + d, 2f] = [g_cvec ; g_mt] or None)."""
    n, f = g_out.shape
    d, e = (0 if eattr is None else eattr.shape[1]), plan.num_edges
    dev = g_out.device
    g_pq = torch.empty(n, 4 * f, dtype=g_out.dtype, device=dev)
    g_h = torch.empty(e, 2 * f, dtype=g_out.dtype, device=dev)
    g_eattr = torch.empty(e, d, dtype=g_out.dtype, device=dev) if (need_eattr and d > 0) else None
    g_params = torch.empty(1 + d, 2 * f, dtype=g_out.dtype, device=dev) if need_params else None
    ws = _ws(_lib.query("hgb_cgconv_workspace_bytes", f, d), dev) if need_params else None
    col = plan.by_col
    _lib.call("hgb_cgconv_bwd", _p(g_out), _p(pq), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col")), _p(eattr), d, _p(mt), _p(cvec),
              n, e, f, _p(g_pq), 4 * f, _p(g_h), _p(g_eattr), _p(g_params), _p(ws), _stream())
    row = plan.by_row          # Q was gathered by the source of every edge: g_Q is the by-source segment sum of g_h
    _lib.call("hgb_segment_sum_strided", _p(g_h), _p(row.rowptr), _p(row.perm), n, 2 * f, _p(g_pq[:, 2 * f:]), 4 * f, _stream())
    return g_pq, g_eattr, g_params


class CgConvFn(torch.autograd.Function):
    """out = x + sum over the targets i = edge_index[1] of m_e = sigmoid(f_e) * softplus(s_e) -- torch_geometric 2.6.1 CGConv
    (aggr "add", batch_norm=False; hydragnn/models/CGCNNStack.py:60-80) with f_e = P_f[i] + Q_f[j] + C_f a_e + b_f and s_e
    alike.  ``pq`` [n, 4f] = [P_f | P_s | Q_f | Q_s], ``mt`` [d, 2f] = [C_f | C_s]^T (None without edge input), ``cvec`` [2f]
    = [b_f | b_s], ``x`` [n, f] the residual.  One kernel each way; neither z, the pre-activations nor the message reach
    memory.  Without nodes or edges no kernel runs."""

    @staticmethod
    def forward(ctx, pq, eattr, mt, cvec, x, plan):
        pq, cvec, x = _chk(pq), _chk(cvec), _chk(x)
        eattr = _chk(eattr) if eattr is not None else None
        mt = _chk(mt) if eattr is not None else None
        ctx.save_for_backward(pq, eattr, mt, cvec)
        ctx.plan = plan
        if x.shape[0] == 0 or plan.num_edges == 0:
            return x.clone()
        return raw_cgconv_fwd(pq, eattr, mt, cvec, x, plan)

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        pq, eattr, mt, cvec = ctx.saved_tensors
        plan = ctx.plan
        need = ctx.needs_input_grad
        need_params = (need[2] or need[3]) and not _DATA_ONLY["on"]
        g_out = _chk(g_out.contiguous())
        n, f = g_out.shape
        d = 0 if eattr is None else eattr.shape[1]
        if n == 0 or plan.num_edges == 0:
            g_pq = torch.zeros_like(pq)
            g_eattr = torch.zeros_like(eattr) if (eattr is not None and need[1]) else None
            g_params = torch.zeros(1 + d, 2 * f, dtype=g_out.dtype, device=g_out.device) if need_params else None
        else:
            g_pq, g_eattr, g_params = raw_cgconv_bwd(g_out, pq, eattr, mt, cvec, plan, need_eattr=eattr is not None and need[1],
                                                     need_params=need_params)
        if g_params is None:
            return g_pq, g_eattr, None, None, g_out, None
        return g_pq, g_eattr, (g_params[1:] if eattr is not None else None), g_params[0], g_out, None


def gat_supported(heads, c, d):
    """Shapes ``GatConvFn`` takes: 1 <= heads <= 8, heads * c <= 512 (<= 256 when c is not a multiple of 4), 0 <= d <= 16."""
    return bool(_lib.query("hgb_gat_supported", int(heads), int(c), int(d)))


def gat_dropout_seed(device):
    """The attention-dropout seed of one training forward: one int64 drawn on the device from torch's CUDA generator, so
    ``torch.manual_seed`` reproduces the mask and a captured step draws a new one at every replay."""
    return torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=device)


def raw_gat_dropout_keep(n, e, heads, p, seed):
    """-> uint8 [e + n, heads], 1 where attention coefficient (edge id, head) is kept (self-loop of node i: edge id e + i)."""
    keep = torch.empty(e + n, heads, dtype=torch.uint8, device=seed.device)
    _lib.call("hgb_gat_dropout_keep", int(n), int(e), int(heads), float(p), _p(seed), _p(keep), _stream())
    return keep


def _al16(t):
    return t if t is None or t.data_ptr() % 16 == 0 else t.clone()


def raw_gat_fwd(xlr, eattr, mt, att, bias, plan, heads, c, concat, slope, p=0.0, seed=None):
    """-> (out [n, heads c] (concat) or [n, c], lse [n, heads]): hgb_gat_fwd over the by-target CSR."""
    n, e = xlr.shape[0], plan.num_edges
    d = 0 if eattr is None else eattr.shape[1]
    col = plan.by_col
    out = torch.empty(n, heads * c if concat else c, dtype=xlr.dtype, device=xlr.device)
    lse = torch.empty(n, heads, dtype=xlr.dtype, device=xlr.device)
    _lib.call("hgb_gat_fwd", _p(xlr), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col") if e else None), _p(eattr), d, _p(mt),
              _p(att), _p(bias), n, e, heads, c, int(bool(concat)), float(slope), float(p), _p(seed), _p(out), _p(lse), _stream())
    return out, lse


def raw_gat_bwd(g_out, xlr, eattr, mt, att, lse, plan, heads, c, concat, slope, p=0.0, seed=None, need_eattr=True,
                need_params=True):
    """-> (g_xlr [n, 2 heads c], g_eattr [e, d] or None, g_params [1 + d, heads c] = [g_att ; g_mt] or None)."""
    n, e = xlr.shape[0], plan.num_edges
    d = 0 if eattr is None else eattr.shape[1]
    dev = xlr.device
    g_xlr = torch.empty_like(xlr)
    g_eattr = torch.empty(e, d, dtype=xlr.dtype, device=dev) if (need_eattr and d > 0) else None
    g_params = torch.empty(1 + d, heads * c, dtype=xlr.dtype, device=dev) if need_params else None
    ws = _ws(_lib.query("hgb_gat_workspace_bytes", n, e, heads, c, d), dev)
    col, row = plan.by_col, plan.by_row
    _lib.call("hgb_gat_bwd", _p(g_out), _p(xlr), _p(col.rowptr), _p(col.perm), _p(plan.nbr("col") if e else None), _p(row.rowptr),
              _p(row.perm), _p(plan.nbr("row") if e else None), _p(eattr), d, _p(mt), _p(att), _p(lse), n, e, heads, c,
              int(bool(concat)), float(slope), float(p), _p(seed), _p(g_xlr), _p(g_eattr), _p(g_params), _p(ws), _stream())
    return g_xlr, g_eattr, g_params


class GatConvFn(torch.autograd.Function):
    """torch_geometric 2.6.1 GATv2Conv (add_self_loops=True, fill_value="mean", share_weights=False; hydragnn/models/
    GATStack.py:175-205) after its two Linears: ``xlr`` [n, 2 heads c] = [x_l | x_r], ``eattr`` [e, d] the edge input (None
    without one) and ``mt`` [d, heads c] the (folded) lin_edge weight transposed, ``att`` [heads c], ``bias`` [heads c] (concat)
    or [c] (mean over the heads).  Attention dropout with probability ``p`` keyed by the device ``seed``.  One kernel forward
    writes only out and the per-head log-sum-exp; the backward is two kernels (by target, by source) and no atomics."""

    @staticmethod
    def forward(ctx, xlr, eattr, mt, att, bias, plan, heads, c, concat, slope, p, seed):
        xlr, att, bias = _al16(_chk(xlr)), _chk(att), _chk(bias)
        eattr = _chk(eattr) if eattr is not None else None
        mt = _chk(mt) if eattr is not None else None
        n = xlr.shape[0]
        if n == 0:
            out = xlr.new_empty(0, heads * c if concat else c)
            lse = xlr.new_empty(0, heads)
        else:
            out, lse = raw_gat_fwd(xlr, eattr, mt, att, bias, plan, heads, c, concat, slope, p, seed)
        ctx.save_for_backward(xlr, eattr, mt, att, lse, seed)
        ctx.plan, ctx.cfg = plan, (heads, c, bool(concat), float(slope), float(p))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        xlr, eattr, mt, att, lse, seed = ctx.saved_tensors
        heads, c, concat, slope, p = ctx.cfg
        need = ctx.needs_input_grad
        data_only = _DATA_ONLY["on"]
        need_params = (need[2] or need[3]) and not data_only
        g_out = _al16(_chk(g_out.contiguous()))
        n = xlr.shape[0]
        d = 0 if eattr is None else eattr.shape[1]
        if n == 0:
            g_xlr = torch.zeros_like(xlr)
            g_eattr = torch.zeros_like(eattr) if (eattr is not None and need[1]) else None
            g_params = torch.zeros(1 + d, heads * c, dtype=xlr.dtype, device=xlr.device) if need_params else None
            g_bias = torch.zeros(g_out.shape[1], dtype=xlr.dtype, device=xlr.device)
        else:
            g_xlr, g_eattr, g_params = raw_gat_bwd(g_out, xlr, eattr, mt, att, lse, ctx.plan, heads, c, concat, slope, p, seed,
                                                   need_eattr=eattr is not None and need[1], need_params=need_params)
            g_bias = raw_colsum(g_out) if (need[4] and not data_only) else None
        g_att = g_params[0] if g_params is not None else None
        g_mt = g_params[1:] if (g_params is not None and eattr is not None) else None
        return (g_xlr, g_eattr, g_mt, g_att, None if data_only else g_bias) + (None,) * 7


def cfconv_supported(g, nf, d):
    """Shapes ``CfConvFn`` takes: 1 <= num_gaussians <= 64, 1 <= num_filters <= 128, raw edge input width <= 16."""
    return bool(_lib.query("hgb_cfconv_supported", int(g), int(nf), int(d)))


class CfConvFn(torch.autograd.Function):
    """SchNet's CFConv message and sum over the targets i = edge_index[1] (hgb_cfconv_fwd): out_i = sum_e xl[j] * W_e with the
    filter W_e = (ssp([rbf(d_e) | r_e] A + b1) W2^T + b2) * C(d_e) formed per edge on chip, d_e = |pos[i] - pos[j]|.
    ``a1t`` [G + d, nf] = [W1[:, :G]^T ; Mt], ``r`` [e, d] or None, ``mu`` the Gaussian centres.  With ``want_we`` the
    filter W_e [e, nf] is returned as a second output (the equivariant coordinate MLP reads it), else None."""

    @staticmethod
    def forward(ctx, xl, pos, r, a1t, b1, w2, b2, mu, coeff, cutoff, plan, want_we):
        xl, pos, a1t, b1, w2, b2, mu = (_chk(t) for t in (xl, pos, a1t, b1, w2, b2, mu))
        r = _chk(r) if r is not None else None
        n, nf = xl.shape
        g, d, e = mu.numel(), (0 if r is None else r.shape[1]), plan.num_edges
        out = torch.empty(n, nf, dtype=xl.dtype, device=xl.device)
        w_e = torch.empty(e, nf, dtype=xl.dtype, device=xl.device) if want_we else None
        col = plan.by_col
        _lib.call("hgb_cfconv_fwd", _p(xl), _p(pos), _p(plan.row), _p(col.rowptr), _p(col.perm), _p(r), d, _p(mu), float(coeff),
                  float(cutoff), _p(a1t), _p(b1), _p(w2), _p(b2), n, e, g, nf, _p(out), _p(w_e), _stream())
        ctx.save_for_backward(xl, pos, r, a1t, b1, w2, b2, mu)
        ctx.coeff, ctx.cutoff, ctx.plan = float(coeff), float(cutoff), plan
        if w_e is not None:
            return out, w_e
        return out, None

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_we):
        xl, pos, r, a1t, b1, w2, b2, mu = ctx.saved_tensors
        plan = ctx.plan
        n, nf = xl.shape
        g, d, e = mu.numel(), (0 if r is None else r.shape[1]), plan.num_edges
        dev = xl.device
        need_xl, need_pos, need_r = ctx.needs_input_grad[0], ctx.needs_input_grad[1], r is not None and ctx.needs_input_grad[2]
        g_xle = torch.empty(e, nf, dtype=xl.dtype, device=dev) if need_xl else None
        g_dist = torch.empty(e, dtype=xl.dtype, device=dev) if need_pos else None
        g_r = torch.empty(e, d, dtype=xl.dtype, device=dev) if need_r else None
        need_params = any(ctx.needs_input_grad[3:7])
        g_params = torch.empty((g + d) * nf + nf + nf * nf + nf, dtype=xl.dtype, device=dev) if need_params else None
        ws = _ws(_lib.query("hgb_cfconv_workspace_bytes", g, nf, d), dev) if need_params else None
        g_out = _chk(g_out.contiguous())
        g_we = _chk(g_we.contiguous()) if g_we is not None else None
        _lib.call("hgb_cfconv_bwd", _p(g_out), _p(g_we), _p(xl), _p(pos), _p(plan.row), _p(plan.col), _p(r), d, _p(mu), ctx.coeff,
                  ctx.cutoff, _p(a1t), _p(b1), _p(w2), _p(b2), n, e, g, nf, _p(g_xle), _p(g_dist), _p(g_r), _p(g_params), _p(ws),
                  _stream())
        g_xl = raw_segment_sum(g_xle, plan.by_row.rowptr, plan.by_row.perm, n) if need_xl else None     # xl was gathered by source
        g_pos = _raw_edge_len_bwd(g_dist, pos, None, plan) if need_pos else None
        if not need_params:
            return g_xl, g_pos, g_r, None, None, None, None, None, None, None, None, None
        k = (g + d) * nf
        g_a1t = g_params[:k].view(g + d, nf)
        g_b1 = g_params[k:k + nf]
        g_w2 = g_params[k + nf:k + nf + nf * nf].view(nf, nf)
        g_b2 = g_params[k + nf + nf * nf:]
        return g_xl, g_pos, g_r, g_a1t, g_b1, g_w2, g_b2, None, None, None, None, None


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


class GroupedLinearPReluFn(torch.autograd.Function):
    """``GroupedLinearFn`` with PReLU in the epilogue (``hgb_grouped_linear_prelu``: the slope read from device memory, z stored);
    backward: ``hgb_prelu_bwd``, then the grouped data and weight gradients without an activation."""

    @staticmethod
    def forward(ctx, x, w, b, rowptr, slope):
        x, w, sl = _chk(x.contiguous()), _chk(w.contiguous()), _chk(slope)
        b = _chk(b.contiguous()) if b is not None else None
        groups, n, k = w.shape
        m = x.shape[0]
        y = torch.empty(m, n, dtype=x.dtype, device=x.device)
        z = torch.empty_like(y)
        _lib.call("hgb_grouped_linear_prelu", _p(x), k, _p(w), _p(b), _p(rowptr), groups, m, n, k, _p(sl), _p(y), _p(z), _stream())
        ctx.save_for_backward(x, w, z, rowptr, sl)
        ctx.has_b = b is not None
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, w, z, rowptr, sl = ctx.saved_tensors
        groups, n, k = w.shape
        m = x.shape[0]
        dz, dslope = _prelu_bwd(gy.contiguous(), z, sl, ctx.needs_input_grad[4])
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = torch.empty(m, k, dtype=x.dtype, device=x.device)
            _lib.call("hgb_grouped_linear", _p(dz), n, _p(w), None, _p(rowptr), groups, m, k, n, 1, 0, 0.0, _p(gx), None, _stream())
        if ctx.needs_input_grad[1] or (ctx.has_b and ctx.needs_input_grad[2]):
            gw = torch.empty_like(w)
            gb = torch.empty(groups, n, dtype=x.dtype, device=x.device) if ctx.has_b else None
            _lib.call("hgb_grouped_wgrad", _p(dz), _p(x), k, _p(rowptr), groups, m, n, k, _p(gw), _p(gb), _stream())
        return gx, gw, gb, None, dslope


class GroupedMatMul(torch.autograd.Function):
    """``y[r] = x[r] W_g^T`` (``trans_w`` 0, w [groups, n, k]) or ``y[r] = x[r] W_g`` (``trans_w`` 1, w [groups, k, n]) for rows
    sorted by group (``rowptr`` [groups + 1] on the device), on ``hgb_grouped_linear``.  The data gradient is the same product
    with ``trans_w`` flipped and the weight gradient a ``GroupedWgrad``, whose own derivatives are grouped products again: closed
    under autograd, as ``MatMul`` is.  ``w_is_weight``: ``w`` is built from parameters, so its gradient is skipped under
    ``only_data_grads``."""

    @staticmethod
    def forward(ctx, x, w, rowptr, trans_w, w_is_weight=False):
        x, w = _chk(x.contiguous()), _chk(w.contiguous())
        groups = w.shape[0]
        m, k = x.shape
        n = w.shape[2] if trans_w else w.shape[1]
        y = torch.empty(m, n, dtype=x.dtype, device=x.device)
        _lib.call("hgb_grouped_linear", _p(x), k, _p(w), None, _p(rowptr), groups, m, n, k, int(trans_w), 0, 0.0, _p(y), None,
                  _stream())
        ctx.save_for_backward(x, w, rowptr)
        ctx.trans_w, ctx.w_is_weight = int(trans_w), bool(w_is_weight)
        return y

    @staticmethod
    def backward(ctx, g):
        x, w, rowptr = ctx.saved_tensors
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = GroupedMatMul.apply(g, w, rowptr, 1 - ctx.trans_w, ctx.w_is_weight)
        if ctx.needs_input_grad[1] and not (ctx.w_is_weight and _DATA_ONLY["on"]):
            #  y = x W_g^T: dW_g = g^T x          y = x W_g: dW_g = x^T g
            gw = GroupedWgrad.apply(x, g, rowptr) if ctx.trans_w else GroupedWgrad.apply(g, x, rowptr)
        return gx, gw, None, None, None


class GroupedWgrad(torch.autograd.Function):
    """``H_g = sum_{r in g} a[r]^T b[r]``: [groups, n, k] from a [m, n] and b [m, k] (``hgb_grouped_wgrad``; an empty group gives
    zeros).  d/da = b H^T and d/db = a H, both ``GroupedMatMul``s."""

    @staticmethod
    def forward(ctx, a, b, rowptr):
        a, b = _chk(a.contiguous()), _chk(b.contiguous())
        groups = rowptr.numel() - 1
        m, n = a.shape
        k = b.shape[1]
        h = torch.empty(groups, n, k, dtype=a.dtype, device=a.device)
        _lib.call("hgb_grouped_wgrad", _p(a), _p(b), k, _p(rowptr), groups, m, n, k, _p(h), None, _stream())
        ctx.save_for_backward(a, b, rowptr)
        return h

    @staticmethod
    def backward(ctx, h):
        a, b, rowptr = ctx.saved_tensors
        ga = GroupedMatMul.apply(b, h, rowptr, 0) if ctx.needs_input_grad[0] else None
        gb = GroupedMatMul.apply(a, h, rowptr, 1) if ctx.needs_input_grad[1] else None
        return ga, gb, None


class GroupedBiasAdd(torch.autograd.Function):
    """``y[r] + b[group of r]``: ``GatherRows`` of the per-group bias [groups, n] by the group of every row; the bias gradient is
    its adjoint ``SegmentSum`` (closed), skipped under ``only_data_grads``.  ``rows``: Csr of the group of every (sorted) row."""

    @staticmethod
    def forward(ctx, y, b, rows):
        ctx.rows = rows
        return y + raw_gather(_chk(b.contiguous()), rows.idx)

    @staticmethod
    def backward(ctx, g):
        gb = SegmentSum.apply(g, ctx.rows) if (ctx.needs_input_grad[1] and not _DATA_ONLY["on"]) else None
        return g, gb, None


def grouped_mlp_ok(layers_by_group):
    """Do the per-group MLPs share one architecture, so that ``grouped_mlp`` can run them?  ``layers_by_group``: one list per
    group of ``(weight [out, in], bias or None)`` pairs for the Linears and activation modules between them."""
    from torch import nn
    from .stacks import _act_code
    first = layers_by_group[0]
    if any(len(g) != len(first) for g in layers_by_group):
        return False
    for i, a in enumerate(first):
        layer = [g[i] for g in layers_by_group]
        if isinstance(a, tuple):
            if not all(isinstance(l, tuple) for l in layer) or len({tuple(l[0].shape) for l in layer}) != 1:
                return False
            if len({l[1] is None for l in layer}) != 1:
                return False
            if i + 1 < len(first) and not isinstance(first[i + 1], nn.Module):
                return False
        elif (not isinstance(a, nn.Module) or i == 0 or _act_code(a) is None or not isinstance(first[i - 1], tuple)
              or any(_act_code(l) is None or _act_code(l)[0] != _act_code(a)[0] for l in layer)):
            return False
        elif isinstance(a, nn.PReLU) and any(l is not a for l in layer):
            return False                                     # branches with slopes of their own: not the reference's layout
    return isinstance(first[-1], tuple) if first else False


def grouped_mlp(layers_by_group, x, rowptr, higher_order=False, rows=None):
    """Run per-group MLPs that ``grouped_mlp_ok`` accepts on rows sorted by group (``rowptr`` [groups + 1] on the device): one
    launch per Linear.  First order: ``GroupedLinearFn`` / ``GroupedLinearPReluFn`` with the activation in the epilogue.  Any
    order (``higher_order``): ``GroupedMatMul`` + ``GroupedBiasAdd`` (``rows``: the group of every row) with the activations as
    ATen glue, as ``linear_any_order`` does."""
    from .stacks import _act_code, apply_act
    first = layers_by_group[0]
    i = 0
    while i < len(first):
        w = torch.stack([g[i][0] for g in layers_by_group])
        b = torch.stack([g[i][1] for g in layers_by_group]) if first[i][1] is not None else None
        act = first[i + 1] if i + 1 < len(first) else None
        if higher_order:
            x = GroupedMatMul.apply(x, w, rowptr, 0, True)
            if b is not None:
                x = GroupedBiasAdd.apply(x, b, rows)
            if act is not None:
                x = apply_act(act, x, True)
        else:
            code = _act_code(act) if act is not None else None
            if code is not None and code[0] == "prelu":
                x = GroupedLinearPReluFn.apply(x, w, b, rowptr, code[1])
            else:
                x = GroupedLinearFn.apply(x, w, b, rowptr, code[0] if code else None, code[1] if code else 0.0)
        i += 2 if act is not None else 1
    return x


class BranchMixFn(torch.autograd.Function):
    """E [G] = sum_b w[g, b] E_gb from every branch's output e [R, B] (``hgb_branch_mix_fwd``): E_gb is e itself for a graph
    head (``gcsr`` None, R = G) or the sum of e over the atoms of graph g for a node head (``gcsr``: the graph CSR), written to
    ``eb`` [G, B].  The backward seeds the heads with w[g(r), b] dE_g (``hgb_branch_mix_bwd``).  ``w`` is data: no gradient."""

    @staticmethod
    def forward(ctx, e, w, gcsr, eb):
        e, w = _chk(e.contiguous()), _chk(w.contiguous())
        r, b = e.shape
        g = w.shape[0]
        gptr = None if gcsr is None else gcsr.rowptr
        out = torch.empty(g, dtype=e.dtype, device=e.device)
        _lib.call("hgb_branch_mix_fwd", _p(e), _p(gptr), _p(w), g, r, b, _p(eb), _p(out), _stream())
        ctx.save_for_backward(w)
        ctx.gptr, ctx.r = gptr, r
        return out

    @staticmethod
    def backward(ctx, dout):
        w, = ctx.saved_tensors
        g, b = w.shape
        seeds = torch.empty(ctx.r, b, dtype=w.dtype, device=w.device)
        _lib.call("hgb_branch_mix_bwd", _p(_chk(dout.contiguous())), _p(ctx.gptr), _p(w), g, ctx.r, b, _p(seeds), _stream())
        return seeds, None, None, None


def branch_mix(e, w, gcsr=None):
    """(E [G], E_gb [G, B]) of ``BranchMixFn``; E_gb is ``e`` itself (detached) for a graph head."""
    if e.dim() != 2 or w.dim() != 2 or e.shape[1] != w.shape[1]:
        raise ValueError("branch_mix: e [R, B] and w [G, B] must have the same B, got %s and %s" % (tuple(e.shape), tuple(w.shape)))
    graphs = e.shape[0] if gcsr is None else gcsr.n
    if graphs != w.shape[0]:
        raise ValueError("branch_mix: %d graphs but %d weight rows" % (graphs, w.shape[0]))
    if gcsr is None:
        return BranchMixFn.apply(e, w, None, None), e.detach()
    eb = torch.empty(w.shape, dtype=e.dtype, device=e.device)
    return BranchMixFn.apply(e, w, gcsr, eb), eb


# =====================================================================================================
# SAGEConv / MFConv: neighbour aggregation gathered into a degree-grouped wgmma Linear (hgb_nbr.cu)
# =====================================================================================================
class DegreePlan:
    """Nodes grouped by clamped in-degree (MFConv's weight index): ``order`` [n] row -> node (None: identity, one group),
    ``grp_ptr`` [groups + 1], ``tiles`` the fused kernel's tile table (None when the kernel does not take this many groups), and
    ``perm``, the CSR of ``order`` as a gather / scatter pair, built when the composed path first asks for it."""
    __slots__ = ("order", "grp_ptr", "tiles", "groups", "n", "_perm")

    def __init__(self, order, grp_ptr, tiles, groups, n):
        self.order, self.grp_ptr, self.tiles, self.groups, self.n, self._perm = order, grp_ptr, tiles, groups, n, None

    @property
    def perm(self):
        if self._perm is None:
            self._perm = csr_build(self.order.to(torch.int64), self.n)
        return self._perm


NBR_MAX_GROUPS = 128        # the largest group count hgb_nbr_tiles and the fused kernels take


def degree_plan(plan, groups):
    """Counting sort of the nodes by min(in-degree, groups - 1), stable by node id, on the device: a CSR build over the clamped
    degrees (no host read).  One group needs no sort: the order is the identity."""
    col = plan.by_col
    n = plan.num_nodes
    dev = col.rowptr.device
    if groups == 1:
        order, grp_ptr = None, torch.full((2,), n, dtype=torch.int32, device=dev)
        grp_ptr[0] = 0
    else:
        deg = (col.rowptr[1:] - col.rowptr[:-1]).clamp(max=groups - 1).to(torch.int64)
        csr = csr_build(deg, groups)
        order, grp_ptr = csr.perm, csr.rowptr
    tiles = None
    if groups <= NBR_MAX_GROUPS:
        tiles = torch.empty(((n + 63) // 64 + groups) * 2, dtype=torch.int32, device=dev)
        _lib.call("hgb_nbr_tiles", _p(grp_ptr), groups, n, _p(tiles), _stream())
    return DegreePlan(order, grp_ptr, tiles, groups, n)


def nbr_linear_supported(k, n_out, groups):
    """Shapes ``NbrLinearFn`` takes: 1 <= k <= 128, 1 <= n_out <= 256, groups <= 128."""
    return bool(_lib.query("hgb_nbr_linear_supported", int(k), int(n_out), int(groups)))


def _r32(v):
    return (v + 31) // 32 * 32


class NbrLinearFn(torch.autograd.Function):
    """out[i] = lin_l,g(h_i) + lin_r,g(x_i) with h_i the sum (``mean``: the mean, 0 without in-edges) of x_j over the in-edges
    j -> i (i = edge_index[1]) and g the node's group in ``dp`` -- SAGEConv with one group and the mean, MFConv with a group per
    clamped in-degree and the sum.  ``wl`` / ``wr`` [groups, n_out, k], ``bl`` [groups, n_out].  Forward: one hgb_nbr_linear_fwd
    launch; h never reaches memory unless the weight gradient needs it (as part of the [h | x] operand).  Backward: the grouped
    wgmma with the transposed weights gives [g_h | g_x root]; g_x = g_x root + the by-source segment sum of g_h; the weight
    gradient is hgb_tc_wgrad (one group) or hgb_grouped_wgrad (rows in degree order), skipped under ``only_data_grads``."""

    @staticmethod
    def forward(ctx, x, wl, bl, wr, dp, plan, mean):
        x = _chk(x.contiguous())
        n, k = x.shape
        groups, n_out, _ = wl.shape
        kp = _r32(k)
        w = x.new_zeros(groups, _r32(n_out), 2 * kp)                    # [W_l | 0 | W_r | 0], zero rows past n_out
        w[:, :n_out, :k] = wl
        w[:, :n_out, kp:kp + k] = wr
        need_w = any(ctx.needs_input_grad[1:4])
        hx = torch.empty(n, 2 * kp, dtype=x.dtype, device=x.device) if need_w else None
        out = torch.empty(n, n_out, dtype=x.dtype, device=x.device)
        ctx.tc, ctx.mean, ctx.dp, ctx.plan, ctx.k = _TC["enabled"], bool(mean), dp, plan, k
        ctx.save_for_backward(w, hx)
        col = plan.by_col
        _lib.call("hgb_nbr_linear_fwd", _p(x), n, k, _p(col.rowptr), _p(plan.nbr("col")), plan.num_edges, int(mean), _p(dp.order),
                  _p(dp.grp_ptr), _p(dp.tiles), groups, _p(w), _p(_chk(bl.contiguous())), n_out, _p(out), _p(hx),
                  0 if ctx.tc else 1, _stream())
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        w, hx = ctx.saved_tensors
        dp, plan, k = ctx.dp, ctx.plan, ctx.k
        g = _chk(g_out.contiguous())
        n, n_out = g.shape
        groups, kp = w.shape[0], w.shape[2] // 2
        exact = 0 if ctx.tc else 1
        need = ctx.needs_input_grad
        g_x = g_wl = g_bl = g_wr = None
        if need[0]:
            g_h = torch.empty(n, k, dtype=g.dtype, device=g.device)
            g_xr = torch.empty_like(g_h)
            _lib.call("hgb_nbr_linear_bwd_data", _p(g), n, n_out, _p(plan.by_col.rowptr), int(ctx.mean), _p(dp.order), _p(dp.grp_ptr),
                      _p(dp.tiles), groups, _p(w.transpose(1, 2).contiguous()), k, _p(g_h), _p(g_xr), exact, _stream())
            # every node j receives g_h of the targets of its out-edges: the by-source CSR, gathering target rows
            g_x = raw_segment_sum(g_h, plan.by_row.rowptr, plan.nbr("row"), n).add_(g_xr)
        if any(need[1:4]) and not _DATA_ONLY["on"]:
            if n == 0:
                dw = g.new_zeros(groups, n_out, 2 * kp)
                db = g.new_zeros(groups, n_out)
            elif groups == 1:
                with tensor_cores(ctx.tc):
                    _, dw, db = linear_bwd_dispatch(g, hx, w[0, :n_out], need_x=False)
                dw, db = dw[None], db[None]
            else:
                gs = raw_gather(g, dp.order)                               # g_out in degree order, as hx
                dw = torch.empty(groups, n_out, 2 * kp, dtype=g.dtype, device=g.device)
                db = torch.empty(groups, n_out, dtype=g.dtype, device=g.device)
                _lib.call("hgb_grouped_wgrad", _p(gs), _p(hx), 2 * kp, _p(dp.grp_ptr), groups, n, n_out, 2 * kp, _p(dw), _p(db),
                          _stream())
            g_wl, g_bl, g_wr = dw[:, :, :k], db, dw[:, :, kp:kp + k]
        return g_x, g_wl, g_bl, g_wr, None, None, None


def nbr_linear_composed(x, wl, bl, wr, dp, plan, mean, higher_order=False):
    """The same layer composed from GatherRows / SegmentSum, Linear and the grouped Linear over degree-sorted rows: the path of
    higher-order passes and unsupported shapes, and the reference the fused path is tested against.  With more than one group
    the grouped Linear is first-order only."""
    h = SegmentSum.apply(GatherRows.apply(x, plan.by_row), plan.by_col)             # sum of x[edge_index[0]] at edge_index[1]
    if mean:
        col = plan.by_col
        h = h / (col.rowptr[1:] - col.rowptr[:-1]).clamp(min=1).to(h.dtype)[:, None]
    if dp.groups == 1:
        lin = linear_any_order if higher_order else linear_act
        return lin(h, wl[0], bl[0]) + lin(x, wr[0], None)
    hx = GatherRows.apply(torch.cat([h, x], dim=1), dp.perm)                        # rows in degree order
    y = GroupedLinearFn.apply(hx, torch.cat([wl, wr], dim=2), bl, dp.grp_ptr, None, 0.0)
    return SegmentSum.apply(y, dp.perm)


# =====================================================================================================
# fused EGNN edge block + closed edge-length primitives (any order of differentiation the MLIP loss needs)
# =====================================================================================================
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
    if plan.num_edges == 0:         # hgb_edge_vec_scatter takes no edge count: it cannot tell no edges from NULL arrays
        return gvec.new_zeros(plan.num_nodes, 3)
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
MACE_TP_MAX_EDGE_DIM = 16       # MACE_TP_MAX_D of hgb_mace.cu: the largest edge_dim whose per-edge stage fits in shared memory


def mace_tp_supported(lin, lsh, f, edge_dim=0):
    return 0 <= lin <= 2 and 1 <= lsh <= 3 and lin <= lsh and f % 32 == 0 and 0 <= edge_dim <= MACE_TP_MAX_EDGE_DIM


class MaceTpScatterFn(torch.autograd.Function):
    """conv_tp + scatter-sum over receivers in one kernel (blocks.py:390-395).  up [N, S_in, F], sh [E, S_sh], tpw [E, W];
    returns the packed message buffer (per output degree l3 a [N, 2l3+1, n_paths(l3) F] block).  eattr: None (W = P F) or the
    edge attributes [E, D]; then W = (P + D (lin + 1)) F, the 0e paths' [F, D+1] blocks in the reference's layout."""

    @staticmethod
    def forward(ctx, up, sh, tpw, plan, lin, lsh, eattr=None):
        up, sh, tpw = _chk(up.contiguous()), _chk(sh.contiguous()), _chk(tpw.contiguous())
        eattr = None if eattr is None else _chk(eattr.contiguous())
        d = 0 if eattr is None else eattr.shape[1]
        n, f = up.shape[0], up.shape[2]
        nacc = _lib.query("hgb_mace_tp_num_acc", lin, lsh)
        if n == 0 or tpw.shape[0] == 0:
            # no edge: every sum is empty, and an empty per-edge array has no address to hand to the kernel
            out = torch.zeros(nacc * n * f, dtype=up.dtype, device=up.device)
        else:
            out = torch.empty(nacc * n * f, dtype=up.dtype, device=up.device)
            csr = plan.by_col
            _lib.call("hgb_mace_tp_scatter_fwd", _p(up), _p(sh), _p(tpw), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("col")), n, f, lin,
                      lsh, sh.shape[1], _p(eattr), d, _p(out), _stream())
        ctx.save_for_backward(up, sh, tpw, eattr)
        ctx.plan, ctx.cfg = plan, (lin, lsh)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        up, sh, tpw, eattr = ctx.saved_tensors
        plan, (lin, lsh) = ctx.plan, ctx.cfg
        d = 0 if eattr is None else eattr.shape[1]
        n, s_in, f = up.shape
        e = tpw.shape[0]
        if n == 0 or e == 0:
            return (torch.zeros_like(up) if ctx.needs_input_grad[0] else None, torch.zeros_like(sh) if ctx.needs_input_grad[1] else None,
                    torch.zeros_like(tpw), None, None, None, None)
        g = _chk(g.contiguous())
        g_tpw = torch.empty_like(tpw)
        g_up_e = torch.empty(e, s_in * f, dtype=up.dtype, device=up.device)
        g_sh = torch.zeros_like(sh) if ctx.needs_input_grad[1] else None
        csr = plan.by_col
        _lib.call("hgb_mace_tp_scatter_bwd", _p(g), _p(up), _p(sh), _p(tpw), _p(csr.rowptr), _p(csr.perm), _p(plan.nbr("col")), n, f, lin,
                  lsh, sh.shape[1], _p(eattr), d, _p(g_tpw), _p(g_up_e), _p(g_sh), _stream())
        g_up = raw_segment_sum(g_up_e, plan.by_row.rowptr, plan.by_row.perm, n).reshape(n, s_in, f) if ctx.needs_input_grad[0] else None
        return g_up, g_sh, g_tpw, None, None, None, None


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
        if n:
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
        if n == 0:
            return torch.empty_like(x), torch.zeros_like(wall), None, None, None
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
    if e:                    # an empty operand has no address
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


def _edge_mix_call(mode, src, eattr, c, f):
    """mode 0: src = w, rows [.., F (D+1) ..] of stride src.stride(0) -> [E, F];  mode 1: src = g [E, F] -> [E, F (D+1)]."""
    if not src.is_cuda or src.dtype != torch.float32:
        raise RuntimeError("mace_edge_mix: expected a float32 CUDA tensor, got %s on %s" % (src.dtype, src.device))
    if src.stride(1) != 1:                       # rows may be strided (a column block of tpw); columns must be dense
        src = src.contiguous()
    e, d = eattr.shape
    out = torch.empty(e, f if mode == 0 else f * (d + 1), dtype=src.dtype, device=src.device)
    _lib.call("hgb_mace_edge_mix", mode, _p(src), src.stride(0), _p(eattr), e, f, d, float(c), _p(out), _stream())
    return out


class EdgeMix(torch.autograd.Function):
    """o[e, u] = c sum_v w[e, u, v] a[e, v], a = [edge_attr, 1]: the per-edge weight of a 0e tensor-product path when the edge
    irreps carry edge attributes (MACEStack.py:198-203).  w [E, F (D+1)] may be a column block of tpw.  Its adjoint is
    EdgeMixT and vice versa, so every derivative order stays on hgb_mace_edge_mix.  eattr is data (no gradient)."""

    @staticmethod
    def forward(ctx, w, eattr, c):
        ctx.save_for_backward(eattr)
        ctx.c = c
        return _edge_mix_call(0, w, eattr, c, w.shape[1] // (eattr.shape[1] + 1))

    @staticmethod
    def backward(ctx, g):
        eattr, = ctx.saved_tensors
        return EdgeMixT.apply(g, eattr, ctx.c), None, None


class EdgeMixT(torch.autograd.Function):
    """o[e, u, v] = c g[e, u] a[e, v] as [E, F (D+1)]."""

    @staticmethod
    def forward(ctx, g, eattr, c):
        ctx.save_for_backward(eattr)
        ctx.c = c
        return _edge_mix_call(1, g, eattr, c, g.shape[1])

    @staticmethod
    def backward(ctx, go):
        eattr, = ctx.saved_tensors
        return EdgeMix.apply(go, eattr, ctx.c), None, None


def _chan_call(mode, p0, p1, n, f, p, ni, out_shape):
    p0, p1 = _chk(p0.contiguous()), _chk(p1.contiguous())
    out = torch.empty(out_shape, dtype=p0.dtype, device=p0.device)
    if n:
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


# MACE distance transforms (radial.py:151-245): codes of include/hgb.h.  ``dt`` below is the tuple (kind, z, radii, c0, c1, c2)
# that MACEStack.distance_transform_operands builds: z [N] int64 element indices and the transform's own buffers, whose device
# memory the kernels read at run time.
DIST_TRANSFORMS = {"Agnesi": 1, "Soft": 2}


def _dt_ptrs(dt):
    kind, z, radii, c0, c1, c2 = dt
    return (int(kind), _p(_chk(z, torch.int64)), _p(_chk(radii)), _p(_chk(c0)), _p(_chk(c1)), _p(_chk(c2)))


class MaceEdgeEmbedDtFn(torch.autograd.Function):
    """MaceEdgeEmbedFn with a distance transform: radial = Bessel(T(d)) x cutoff(d) (blocks.py:164-177) in the same one kernel
    per edge; the backward adds Bessel'(t) T'(d) cutoff(d).  First-order path only (as MaceEdgeEmbedFn)."""

    @staticmethod
    def forward(ctx, pos, shifts, plan, dt, lmax, num_bessel, r_max, p):
        pos, shifts = _chk(pos), _chk(shifts)
        e = plan.num_edges
        sh = torch.empty(e, (lmax + 1) ** 2, dtype=pos.dtype, device=pos.device)
        radial = torch.empty(e, num_bessel, dtype=pos.dtype, device=pos.device)
        kind, z, radii, c0, c1, c2 = _dt_ptrs(dt)
        _lib.call("hgb_mace_edge_embed_dt_fwd", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), z, e, int(lmax), int(num_bessel),
                  float(r_max), float(p), kind, radii, c0, c1, c2, _p(sh), _p(radial), _stream())
        ctx.save_for_backward(pos, shifts)
        ctx.plan, ctx.dt, ctx.cfg = plan, dt, (int(lmax), int(num_bessel), float(r_max), float(p))
        return sh, radial

    @staticmethod
    @once_differentiable
    def backward(ctx, g_sh, g_radial):
        pos, shifts = ctx.saved_tensors
        plan, (lmax, nb, rc, p) = ctx.plan, ctx.cfg
        e = plan.num_edges
        gvec = torch.empty(e, 3, dtype=pos.dtype, device=pos.device)
        kind, z, radii, c0, c1, c2 = _dt_ptrs(ctx.dt)
        _lib.call("hgb_mace_edge_embed_dt_bwd", _p(pos), _p(plan.row), _p(plan.col), _p(shifts), z, _p(_chk(g_sh.contiguous())),
                  _p(_chk(g_radial.contiguous())), e, lmax, nb, rc, p, kind, radii, c0, c1, c2, _p(gvec), _stream())
        return _edge_vec_scatter(gvec, plan), None, None, None, None, None, None, None


def _dist_transform_call(order, d, g, plan, dt):
    d = _chk(d.contiguous())
    out = torch.empty_like(d)
    kind, z, radii, c0, c1, c2 = _dt_ptrs(dt)
    _lib.call("hgb_mace_dist_transform", int(order), kind, _p(d), _p(None if g is None else _chk(g.contiguous())), _p(plan.row),
              _p(plan.col), z, radii, c0, c1, c2, plan.num_edges, _p(out), _stream())
    return out


class DistTransformFn(torch.autograd.Function):
    """t = T(d) per edge (d [E] or [E, 1]); backward g T'(d) = DistTransformGradFn (any-order path: forces and force training)."""

    @staticmethod
    def forward(ctx, d, plan, dt):
        ctx.save_for_backward(d)
        ctx.plan, ctx.dt = plan, dt
        return _dist_transform_call(0, d, None, plan, dt)

    @staticmethod
    def backward(ctx, g):
        d, = ctx.saved_tensors
        return DistTransformGradFn.apply(g, d, ctx.plan, ctx.dt, 1), None, None


class DistTransformGradFn(torch.autograd.Function):
    """g T^(order)(d), order 1 or 2.  Its backward is g' T^(order)(d) for g and g' g T^(order+1)(d) for d; the distance transform
    is differentiated at most twice (forces, then the force loss's gradients), a third derivative raises."""

    @staticmethod
    def forward(ctx, g, d, plan, dt, order):
        ctx.save_for_backward(g, d)
        ctx.plan, ctx.dt, ctx.order = plan, dt, order
        return _dist_transform_call(order, d, g, plan, dt)

    @staticmethod
    def backward(ctx, gg):
        g, d = ctx.saved_tensors
        gd = None
        if ctx.needs_input_grad[1]:
            if ctx.order >= 2:
                raise RuntimeError("MACE distance transform: only the first and second derivatives of T are implemented (no third "
                                   "derivative of the edge lengths)")
            gd = DistTransformGradFn.apply(gg * g, d, ctx.plan, ctx.dt, ctx.order + 1)
        gg_g = DistTransformGradFn.apply(gg, d, ctx.plan, ctx.dt, ctx.order) if ctx.needs_input_grad[0] else None
        return gg_g, gd, None, None, None


# =====================================================================================================
# graph-attribute conditioning (hydragnn/models/Base.py _apply_graph_conditioning): rows sorted by graph, gcsr = graph offsets
# =====================================================================================================
def raw_tc_linear_graph_add(h2, w, c, gcsr):
    """y = h2 w^T + c[graph(row)] on the tensor-core kernel (the caller checked ``graph_add_tc_ok``)."""
    m, k = h2.shape
    n = w.shape[0]
    y = torch.empty(m, n, dtype=h2.dtype, device=h2.device)
    _lib.call("hgb_tc_linear_graph_add", _p(h2), h2.stride(0), _p(w), w.stride(0), m, n, k, _p(c), c.stride(0), _p(gcsr.rowptr), gcsr.n,
              _p(y), 0 if _TC["enabled"] else 1, _stream())
    return y


def graph_add_tc_ok(h2, w, c):
    return tc_ok(h2.shape[0], w.shape[0], h2.shape[1], h2, c) and c.stride(1) == 1


class GraphAddLinearFn(torch.autograd.Function):
    """``h W_h^T + c[graph]``: concat_node's Linear(H + G, H) on [h | graph_attr[batch]] with the graph-attribute columns and the
    bias folded into the per-graph term c = graph_attr W_g^T + b [num_graphs, H].  Forward: one tensor-core pass whose epilogue
    adds each row's graph row of c.  Backward: dh (tensor-core dgrad), dW_h (weight-gradient kernel) and dc = graph_sum(dy);
    the parameter parts are skipped under ``only_data_grads``."""

    @staticmethod
    def forward(ctx, h, w, c, gcsr):
        h2 = _chk(h)
        w2 = w if w.stride(1) == 1 else w.contiguous()
        c2 = _chk(c)
        if graph_add_tc_ok(h2, w2, c2):
            y = raw_tc_linear_graph_add(h2, w2, c2, gcsr)
        else:     # shapes the tensor-core kernel does not take: the same sum from the Linear and gather kernels
            y = linear_fwd_dispatch(h2, w2, None)[0] + raw_gather(c2, gcsr.idx)
        ctx.save_for_backward(h2, w2)
        ctx.gcsr, ctx.tc = gcsr, _TC["enabled"]
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        h2, w2 = ctx.saved_tensors
        gy = _chk(gy)
        params = not _DATA_ONLY["on"]
        need_w = ctx.needs_input_grad[1] and params
        with tensor_cores(ctx.tc):
            gh, gw, _ = linear_bwd_dispatch(gy, h2, w2, ctx.needs_input_grad[0], need_w, False)
        gc = raw_segment_sum(gy, ctx.gcsr.rowptr, None, ctx.gcsr.n) if (ctx.needs_input_grad[2] and params) else None
        return gh, gw, gc, None


class FilmFn(torch.autograd.Function):
    """FiLM ``h * (1 + tanh s)[graph] + t[graph]`` with st = [s | t] [num_graphs, 2H] (hgb_film_fwd / hgb_film_bwd): dh in the
    backward pass, plus the per-graph [ds | dt] as fixed-order segmented sums unless ``only_data_grads``."""

    @staticmethod
    def forward(ctx, h, st, gcsr):
        h, st = _chk(h), _chk(st)
        n, c = h.shape
        y = torch.empty_like(h)
        _lib.call("hgb_film_fwd", _p(h), n, c, _p(st), st.stride(0), _p(gcsr.rowptr), gcsr.n, _p(y), _stream())
        ctx.save_for_backward(h, st)
        ctx.gcsr = gcsr
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        h, st = ctx.saved_tensors
        gy = _chk(gy)
        n, c = h.shape
        gh = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        gst = None
        ws, nbytes = None, 0
        if ctx.needs_input_grad[1] and not _DATA_ONLY["on"]:
            gst = torch.empty(ctx.gcsr.n, 2 * c, dtype=h.dtype, device=h.device)
            nbytes = _lib.query("hgb_film_bwd_workspace_bytes", n, c)
            ws = _ws(nbytes, h.device)
        _lib.call("hgb_film_bwd", _p(gy), _p(h), n, c, _p(st), st.stride(0), _p(ctx.gcsr.rowptr), ctx.gcsr.n, _p(gh), _p(gst), _p(ws),
                  nbytes, _stream())
        return gh, gst, None


def adamw_step(p, g, m, v, step_dev, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_adamw_step", _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2), float(eps),
              float(weight_decay), float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())


# ---- the other flat optimizer steps (hgb_optim_flat.cu): torch.optim's single-tensor algorithms over flat buffers ----------
def sgd_step(p, g, momentum_buffer, step_dev, lr, momentum, dampening, nesterov, weight_decay, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_sgd_step", _p(p), _p(g), _p(momentum_buffer), p.numel(), float(lr), float(momentum), float(dampening),
              int(bool(nesterov)), float(weight_decay), float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())


def adam_step(p, g, exp_avg, exp_avg_sq, max_exp_avg_sq, step_dev, lr, beta1, beta2, eps, weight_decay, amsgrad, grad_scale=1.0,
              hyper_dev=None):
    _lib.call("hgb_adam_step", _p(p), _p(g), _p(exp_avg), _p(exp_avg_sq), _p(max_exp_avg_sq), p.numel(), float(lr), float(beta1),
              float(beta2), float(eps), float(weight_decay), int(bool(amsgrad)), float(grad_scale), _p(step_dev), _p(hyper_dev),
              _stream())


def adamax_step(p, g, exp_avg, exp_inf, step_dev, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_adamax_step", _p(p), _p(g), _p(exp_avg), _p(exp_inf), p.numel(), float(lr), float(beta1), float(beta2), float(eps),
              float(weight_decay), float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())


def adagrad_step(p, g, state_sum, step_dev, lr, lr_decay, weight_decay, eps, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_adagrad_step", _p(p), _p(g), _p(state_sum), p.numel(), float(lr), float(lr_decay), float(weight_decay), float(eps),
              float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())


def adadelta_step(p, g, square_avg, acc_delta, step_dev, lr, rho, eps, weight_decay, grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_adadelta_step", _p(p), _p(g), _p(square_avg), _p(acc_delta), p.numel(), float(lr), float(rho), float(eps),
              float(weight_decay), float(grad_scale), _p(step_dev), _p(hyper_dev), _stream())


def rmsprop_step(p, g, square_avg, momentum_buffer, grad_avg, step_dev, lr, alpha, eps, weight_decay, momentum, centered,
                 grad_scale=1.0, hyper_dev=None):
    _lib.call("hgb_rmsprop_step", _p(p), _p(g), _p(square_avg), _p(momentum_buffer), _p(grad_avg), p.numel(), float(lr), float(alpha),
              float(eps), float(weight_decay), float(momentum), int(bool(centered)), float(grad_scale), _p(step_dev), _p(hyper_dev),
              _stream())
