"""On-device radius graphs behind the reference's transform API.

Mirror of ``get_radius_graph`` / ``get_radius_graph_pbc`` / ``*_config``
(hydragnn/preprocess/graph_samples_checks_and_updates.py:112-141): each returns a callable transform that
takes a sample (or, unlike the reference, a whole ``Batch``) and sets ``edge_index`` (+ ``edge_shifts``).
The neighbour search runs in libhgb.so; see csrc/hgb_radius.cu for the ordering / truncation rules.
"""
import torch

from . import _lib, ops
from .ops import _p, _stream

_NO_CAP = 2 ** 31 - 1


def _graph_ptr(data, n, device):
    batch = data.batch
    if batch is None:
        return torch.tensor([0, n], dtype=torch.int32, device=device), 1
    g = data.num_graphs
    ptr = getattr(data, "ptr", None)
    if ptr is not None and torch.is_tensor(ptr) and ptr.numel() == g + 1:
        return ptr.to(device=device, dtype=torch.int32), g
    return ops.graph_ptr_from_batch(batch.to(device), g).rowptr, g


def radius_graph(pos, r, graph_ptr, num_graphs, loop=False, max_num_neighbors=32, known_e=None, capacity=None):
    """edge_index [2,E] int64 (row 0 = source/neighbour, row 1 = target/query), targets ascending.
    ``known_e``: edge count from an earlier run on the same positions -- skips the host read of the count so
    the whole build can be captured in a CUDA graph (the count is verified on the device).
    ``capacity``: allocate ``edge_index [2, capacity]`` and fill its head; the true count stays on the device as
    ``rowptr[-1]`` (``hydragnn_b200.padded`` fills the tail with dummy edges) -- no host read either."""
    pos = ops._chk(pos)
    n = pos.shape[0]
    k = int(min(max_num_neighbors, _NO_CAP - 1))
    deg = torch.empty(n, dtype=torch.int32, device=pos.device)
    _lib.call("hgb_radius_graph_count", _p(pos), _p(graph_ptr), n, num_graphs, float(r), k, int(loop), _p(deg), _stream())
    rowptr = ops.exclusive_scan(deg)
    if capacity is not None:
        e = int(capacity)
    elif known_e is None:
        e = int(rowptr[-1])                                    # the one host sync: the count sizes the output
    else:
        e = int(known_e)                                       # promised by the caller; verified on the device (ops.check_guard)
        ops.expect_count(rowptr[-1:], e, ops.GUARD_EDGE_COUNT)
    ei = torch.empty(2, e, dtype=torch.int64, device=pos.device)
    _lib.call("hgb_radius_graph_fill", _p(pos), _p(graph_ptr), n, num_graphs, float(r), k, int(loop), _p(rowptr), e, _p(ei), _stream())
    return ei, rowptr


def radius_graph_pbc(pos, cell, pbc, cutoff, graph_ptr, num_graphs, max_num_neighbors=32, known=None, capacity=None):
    """Batched periodic neighbour list with nearest-k truncation.  ``cutoff`` is a per-graph fp64 tensor.
    Returns (edge_index [2,E], cell_shift [E,3] int32, edge_shifts [E,3] pos.dtype, in_degree [N] int32, outptr [N+1] int32,
    candidate count).
    ``known`` = (candidate count, edge count) from an earlier run on the same positions: no host read of either count, so the
    build can be captured in a CUDA graph; both are verified on the device (``ops.check_guard``).
    ``capacity`` = (candidate capacity, edge capacity): the buffers are sized by them and filled at the head, so the build can
    be captured while the atoms move.  The true edge count stays on the device as ``outptr[-1]``; the tail of ``cell_shift`` and
    ``edge_shifts`` is zero (``hydragnn_b200.padded`` fills the tail of ``edge_index`` with dummy edges).  A count over its
    capacity sets the guard (``ops.check_guard``) and nothing is written or read past a buffer."""
    assert pos.dtype in (torch.float32, torch.float64)
    if not pos.is_cuda:
        raise RuntimeError("hydragnn_b200 radius_graph_pbc needs CUDA tensors (move the sample to the device first)")
    pos = pos.contiguous()
    is64 = int(pos.dtype == torch.float64)
    dev = pos.device
    n, g = pos.shape[0], num_graphs
    cell = cell.to(device=dev, dtype=torch.float64).reshape(g, 3, 3).contiguous()
    pbc = pbc.to(device=dev, dtype=torch.int32).reshape(g, 3).contiguous()
    cutoff = cutoff.to(device=dev, dtype=torch.float64).contiguous()
    nimg = torch.empty(g, 3, dtype=torch.int32, device=dev)
    st = _stream()
    _lib.call("hgb_radius_pbc_range", _p(pos), is64, _p(graph_ptr), _p(cell), _p(pbc), _p(cutoff), n, g, _p(nimg), st)
    cnt = torch.empty(n, dtype=torch.int32, device=dev)
    _lib.call("hgb_radius_pbc_count", _p(pos), is64, _p(graph_ptr), _p(cell), _p(nimg), _p(cutoff), n, g, _p(cnt), st)
    candptr = ops.exclusive_scan(cnt)
    if capacity is not None:
        c = int(capacity[0])
    elif known is None:
        c = int(candptr[-1])
    else:
        c = int(known[0])
        ops.expect_count(candptr[-1:], c, ops.GUARD_EDGE_COUNT)
    csrc = torch.empty(max(c, 1), dtype=torch.int32, device=dev)
    cshift = torch.empty(max(c, 1), 3, dtype=torch.int32, device=dev)
    clen = torch.empty(max(c, 1), dtype=torch.float64, device=dev)
    _lib.call("hgb_radius_pbc_fill", _p(pos), is64, _p(graph_ptr), _p(cell), _p(nimg), _p(cutoff), n, g, _p(candptr), max(c, 1),
              _p(csrc), _p(cshift), _p(clen), st)
    k = int(min(max_num_neighbors, _NO_CAP))
    deg = torch.empty(n, dtype=torch.int32, device=dev)
    if capacity is not None:
        _lib.call("hgb_radius_pbc_cap_degree", _p(cnt), _p(candptr), n, k, c, _p(deg), _p(ops.guard_flag(dev)), st)
    else:
        _lib.call("hgb_clamp_i32", _p(cnt), k, n, _p(deg), st)
    outptr = ops.exclusive_scan(deg)
    if capacity is not None:
        e = int(capacity[1])
    elif known is None:
        e = int(outptr[-1])
    else:
        e = int(known[1])
        ops.expect_count(outptr[-1:], e, ops.GUARD_EDGE_COUNT)
    ei = torch.empty(2, e, dtype=torch.int64, device=dev)
    cell_shift = torch.empty(e, 3, dtype=torch.int32, device=dev)
    shifts = torch.empty(e, 3, dtype=pos.dtype, device=dev)
    _lib.call("hgb_radius_pbc_emit", _p(graph_ptr), _p(cell), n, g, _p(candptr), _p(csrc), _p(cshift), k, _p(outptr), e, _p(ei),
              _p(cell_shift), _p(shifts), is64, st)
    if capacity is not None:
        _lib.call("hgb_radius_pbc_zero_tail", _p(outptr[-1:]), e, _p(cell_shift), _p(shifts), is64, _p(ops.guard_flag(dev)), st)
    return ei, cell_shift, shifts, deg, outptr, c


class RadiusGraph:
    """PyG ``RadiusGraph(r, loop, max_num_neighbors)`` as the reference builds it (:112-117)."""

    def __init__(self, r, loop=False, max_num_neighbors=32):
        self.r, self.loop, self.max_num_neighbors = r, loop, max_num_neighbors

    def __call__(self, data):
        pos = data.pos
        if pos.dtype != torch.float32:
            raise RuntimeError("b200 radius graph: open-boundary search runs in fp32 (got %s)" % pos.dtype)
        gptr, g = _graph_ptr(data, pos.shape[0], pos.device)
        data.edge_index, rowptr = radius_graph(pos, self.r, gptr, g, self.loop, self.max_num_neighbors)
        data._hgb_col_sorted = (data.edge_index, rowptr, gptr)   # edges grouped by target and by graph: both CSR views are cheap
        data.edge_attr = None                     # PyG RadiusGraph.forward resets edge_attr [3P-memory B.6]
        return data

    def __repr__(self):
        return "%s(r=%s)" % (self.__class__.__name__, self.r)


class RadiusGraphPBC(RadiusGraph):
    """``RadiusGraphPBC.__call__`` (:149-256) for a sample or a batch: per-graph ``cell [3,3]`` / ``pbc [3]``."""

    def __call__(self, data):
        assert data.cell is not None, "data.cell required for PBC."
        assert data.pbc is not None, "data.pbc required for PBC."
        pos = data.pos
        if not torch.is_tensor(pos):
            pos = torch.tensor(pos)
        if pos.dtype not in (torch.float32, torch.float64):
            pos = pos.to(torch.get_default_dtype())
        dev = pos.device
        n = pos.shape[0]
        if not pos.is_cuda:
            raise RuntimeError("hydragnn_b200 RadiusGraphPBC runs on the device: move the sample / batch to CUDA first "
                               "(the reference runs this transform on the CPU at preprocessing time)")
        gptr, g = _graph_ptr(data, n, dev)
        cell = torch.as_tensor(data.cell, dtype=torch.float64).reshape(g, 3, 3)
        pbc = torch.as_tensor(data.pbc).reshape(g, 3)
        cutoff = torch.full((g,), float(self.r), dtype=torch.float64, device=dev)
        node_graph = torch.repeat_interleave(torch.arange(g, device=dev), (gptr[1:] - gptr[:-1]).long())
        for attempt in range(3):                                    # radius growth x1.25 (:168-205)
            ei, cs, sh, deg, outptr, _ = radius_graph_pbc(pos, cell, pbc, cutoff, gptr, g, self.max_num_neighbors)
            lonely = deg == 0
            if not bool(lonely.any()):
                break
            if attempt < 2:
                bad = torch.zeros(g, dtype=torch.bool, device=dev)
                bad[node_graph[lonely]] = True
                cutoff = torch.where(bad, cutoff * 1.25, cutoff)
            else:                                                   # _ensure_connected (:300-322), deterministic source
                m = torch.nonzero(lonely).flatten()
                lo, hi = gptr[node_graph[m]].long(), gptr[node_graph[m] + 1].long()
                srcn = torch.where(hi - lo > 1, lo + (m - lo + 1) % (hi - lo), m)
                ei = torch.cat([ei, torch.stack([srcn, m])], dim=1)
                sh = torch.cat([sh, sh.new_zeros(m.numel(), 3)])
        if self.loop:                                               # appended after truncation (:221-232)
            ar = torch.arange(n, device=dev)
            ei = torch.cat([ei, torch.stack([ar, ar])], dim=1)
            sh = torch.cat([sh, sh.new_zeros(n, 3)])
        data.pos = pos
        data.edge_index, data.edge_shifts = ei, sh
        return data


def get_radius_graph(radius, max_neighbours, loop=False):
    return RadiusGraph(r=radius, loop=loop, max_num_neighbors=max_neighbours)


def get_radius_graph_pbc(radius, max_neighbours, loop=False):
    return RadiusGraphPBC(r=radius, loop=loop, max_num_neighbors=max_neighbours)


def get_radius_graph_config(config, loop=False):
    return RadiusGraph(r=config["radius"], loop=loop, max_num_neighbors=config["max_neighbours"])


def get_radius_graph_pbc_config(config, loop=False):
    return RadiusGraphPBC(r=config["radius"], loop=loop, max_num_neighbors=config["max_neighbours"])
