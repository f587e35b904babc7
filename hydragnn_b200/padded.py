"""Capacity-padded, CUDA-graph-captured training step: ONE captured graph serves every batch of a loader.

The reference's hot loop (hydragnn/train/train_validate_test.py:683-791) sees batches whose node, edge and graph counts all
change from step to step; a CUDA graph wants static shapes.  ``PaddedGraphStep`` owns static device buffers sized by
capacities (``node_cap``, ``edge_cap``, ``graph_cap``) and pads every batch up to them with FILLER GRAPHS:

* unused graph slots receive filler atoms on a line (1.5 A apart, species 1): ordinary little molecules whose outputs
  are masked out of the loss, so they contribute exactly zero to every gradient (0 x finite);
* the unused tail of the edge list receives dummy edges between consecutive filler atoms (``hgb_pad_edges``);
* the real counts live on the device (``valid`` = [graphs, nodes, edges]); losses are means over the real prefix
  (``hgb_loss_fwd_bwd``, or ``hgb_gnll_fwd_bwd`` for mean-and-variance heads, with ``valid_rows``; masked ATen means on the
  any-order MLIP path).

Nothing in the step reads a size back to the host: neighbour build (optional: edges may also come with the batch, as the
reference builds them at preprocessing time), CSR plans, forward, loss, backward, flat all-reduce and fused AdamW replay as
one graph.  A batch larger than a capacity re-captures with grown capacities (host-known sizes) or trips the device guard
(edge count of an on-device neighbour build, checked by ``check()`` / at the end of ``train``).

Supported: EGNN / PaiNN / MACE / PNAEq stacks without BatchNorm-carrying wrappers (GPS mixes every atom of the mini-batch:
filler atoms would leak into real ones) or BatchNorm feature layers (PNA: the same leak through the batch statistics), heads
all of graph type, or the MLIP wrapper (energy + forces).  Any number of dataset branches, as long as the branches of every
head share one architecture: they are decoded by the grouped kernels, which read no group size back to the host
(``stacks.grouped_decode``).  ``dataset_name`` then travels with the batch; filler graphs belong to branch 0.  Models whose
branches differ decode with boolean masks over ``dataset_name.unique()`` and train eagerly.
"""
import torch
import torch.distributed as dist

from . import _lib, ops, radius
from .data import Batch
from .ops import _p, _stream
from .stacks import branches_grouped, forget_plans


def _round_up(x, m):
    return ((int(x) + m - 1) // m) * m


def filler_layout(batch_vec, g, n_cap, g_cap):
    """Host-side layout of a padded batch: (ptr [g_cap + 1] int32, batch [n_cap] int64, fill = number of filler atoms).
    Unused graph slots g .. g_cap - 1 each receive two filler atoms, the last one all that remain."""
    n = int(batch_vec.numel())
    unused, fill = g_cap - g, n_cap - n
    if unused < 1 or fill < 2 * unused:
        raise ValueError("padded batch does not fit: %d graphs / %d atoms into capacities %d / %d" % (g, n, g_cap, n_cap))
    counts = torch.full((unused,), 2, dtype=torch.int64)
    counts[-1] = fill - 2 * (unused - 1)
    allc = torch.cat([torch.bincount(batch_vec, minlength=g), counts])
    ptr = torch.zeros(g_cap + 1, dtype=torch.int32)
    ptr[1:] = torch.cumsum(allc, 0).to(torch.int32)
    bfull = torch.cat([batch_vec, torch.repeat_interleave(torch.arange(g, g_cap), counts)])
    return ptr, bfull, fill


def supported(model):
    m = getattr(model, "module", model)
    inner = getattr(m, "model", m)
    if getattr(inner, "use_global_attn", False) or getattr(inner, "global_attn_engine", None):
        return False
    # SchNet builds its radius graphs in the layers (or, with edge attributes, was not checked against the padded step): eager
    if str(inner) == "SCFStack":
        return False
    # BatchNorm feature layers (PNA) take batch statistics over every row: the filler atoms of a padded batch would enter them
    if any(isinstance(f, torch.nn.BatchNorm1d) for layer in getattr(inner, "feature_layers", ()) for f in layer.modules()):
        return False
    if getattr(m, "model", None) is None and not all(t == "graph" for t in inner.head_type):     # else the MLIP wrapper: one head
        return False
    return getattr(inner, "num_branches", 1) == 1 or _branches_grouped(inner)


def _branches_grouped(inner):
    """Do the branches of every head (of every MACE readout) share one architecture?"""
    return all(branches_grouped(kind, head, dec.graph_shared, inner.num_branches)
               for dec in getattr(inner, "multihead_decoders", [inner]) for head, kind in zip(dec.heads_NN, dec.head_type))


def batch_fields(inner, first_batch, reads_edge_attr, targets=True):
    """The fields a padded batch carries: name -> (shape of one row, dtype), from a representative batch.  ``targets``: the
    loss's targets and the dataset branch of every graph too (a prediction of every branch reads neither)."""
    g = int(first_batch.num_graphs)
    keys = ("x", "pos", "y", "energy", "forces", "edge_shifts") if targets else ("x", "pos", "edge_shifts")
    fields = {k: (tuple(v.shape[1:]), v.dtype) for k, v in first_batch.items()
              if torch.is_tensor(v) and (k in keys or k == "edge_attr" and reads_edge_attr)}
    if targets and getattr(inner, "num_branches", 1) > 1:
        # the dataset branch of every graph, [graphs, 1] int64; filler graphs decode with branch 0
        if getattr(first_batch, "dataset_name", None) is None:
            raise ValueError("PaddedGraphStep: a model with %d dataset branches needs dataset_name in every batch" % inner.num_branches)
        fields["dataset_name"] = ((1,), torch.int64)
    if getattr(inner, "use_graph_attr_conditioning", False):
        # carried as [graphs, G] (1-D per-graph attributes reshaped), zero rows for the filler graphs
        ga = first_batch.graph_attr
        fields["graph_attr"] = ((ga.numel() // g,), ga.dtype)
    return fields


def stage(buf, key, src, g, n, fill):
    """Copy field ``key`` of a batch with ``g`` graphs and ``n`` atoms into its host buffer ``buf``; the rows after it are the
    filler graphs' or atoms' (``fill`` filler atoms on a line, species 1), or zero."""
    if key == "graph_attr":
        src = src.reshape(g, -1)
    rows = src.shape[0]
    buf[:rows] = src.reshape((rows,) + tuple(buf.shape[1:]))
    if key == "pos":
        buf[n:] = 0
        buf[n:, 0] = 1.5 * torch.arange(fill, dtype=buf.dtype)
    elif key == "x":
        buf[n:] = 1
    elif key == "cell":
        buf[rows:] = torch.eye(3, dtype=buf.dtype)           # filler graphs: open boundaries, but every cell is inverted
    else:
        buf[rows:] = 0


class PaddedBatch:
    """The static device buffers of a capacity-padded batch, their pinned staging and the recapture on growth, shared by the
    captured training step (``PaddedGraphStep``) and the captured prediction (``predict.PaddedPredictStep``).  A subclass
    provides ``_do_capture`` (warm-up and capture of its body, which starts with ``_prologue``)."""

    def __init__(self, model, first_batch, neighbour_build, node_cap, edge_cap, graph_cap, slack, warmup, targets=True,
                 extra=None, periodic=False):
        """``first_batch``: a representative (CPU or CUDA) batch -- sizes capacities, field widths and dtypes.
        ``neighbour_build`` = (radius, max_neighbours): build the radius graph inside the captured step from ``pos``;
        None: ``edge_index`` (+ ``edge_shifts``) arrive with every batch.  ``extra``: per-graph fields that ``load`` takes
        besides the batch, name -> (shape of one row, dtype); filler graphs get zero rows.  ``periodic``: the neighbour build
        is ``radius.radius_graph_pbc`` on the per-graph ``cell`` [3, 3] fp64 and ``pbc`` [3] int32 that ``extra`` carries
        (filler graphs: the identity cell, open boundaries), with capacities (``cand_cap``, ``e_cap``) that the subclass sets
        in its ``_capture``."""
        self.model, self.nb, self.periodic = model, neighbour_build, periodic
        self.m = getattr(model, "module", model)
        inner = getattr(self.m, "model", self.m)
        reads_edge_attr = bool(getattr(inner, "use_edge_attr", False))
        if neighbour_build and reads_edge_attr:
            raise ValueError("%s: neighbour_build makes edges without features, but this model reads edge_attr "
                             "(edge_dim > 0); pass edge_index and edge_attr with every batch instead" % type(self).__name__)
        self.dev = next(model.parameters()).device
        self.warmup, self.slack = warmup, slack
        n, g = int(first_batch.pos.shape[0]), int(first_batch.num_graphs)
        e = 0 if neighbour_build else int(first_batch.edge_index.shape[1])
        self._widths = batch_fields(inner, first_batch, reads_edge_attr, targets)
        self._extra = dict(extra or {})
        self._widths.update(self._extra)
        self._capture(node_cap or n, edge_cap or e, graph_cap or g)
        self.recaptures = 0

    # ---- static buffers + capture -----------------------------------------------------------------------------------
    def _capture(self, n_need, e_need, g_need):
        dev = self.dev
        self.g_cap = g_need + 1                                              # at least one filler graph
        self.n_cap = _round_up(n_need * self.slack + 2 * 8, 64)
        if self.nb:
            k = int(self.nb[1])
            self.e_cap = self.n_cap * (k + 1)                                # torch_cluster keeps at most k + 1 (quirk), so this bounds it
        else:
            self.e_cap = _round_up(e_need * self.slack + 64, 64)
        d = Batch()
        hosts = [{}, {}]                                   # two pinned staging sets: the host fills one while the other's copy is in flight
        for key, (tail, dt) in self._widths.items():
            rows = self.g_cap if key in self._extra else {
                "x": self.n_cap, "pos": self.n_cap, "forces": self.n_cap, "y": self.g_cap, "energy": self.g_cap,
                "edge_shifts": self.e_cap, "edge_attr": self.e_cap, "graph_attr": self.g_cap, "dataset_name": self.g_cap}[key]
            if key == "edge_shifts" and self.nb:
                continue
            for h in hosts:
                h[key] = torch.zeros((rows,) + tail, dtype=dt).pin_memory()
            d[key] = torch.zeros((rows,) + tail, dtype=dt, device=dev)
        for h in hosts:
            h["batch"] = torch.zeros(self.n_cap, dtype=torch.int64).pin_memory()
            h["ptr"] = torch.zeros(self.g_cap + 1, dtype=torch.int32).pin_memory()
            h["valid"] = torch.zeros(3, dtype=torch.int32).pin_memory()
            if not self.nb:
                h["edge_index"] = torch.zeros(2, self.e_cap, dtype=torch.int64).pin_memory()
        d.batch = torch.zeros(self.n_cap, dtype=torch.int64, device=dev)
        d.ptr = torch.zeros(self.g_cap + 1, dtype=torch.int32, device=dev)
        d._num_graphs = self.g_cap
        self.valid = torch.zeros(3, dtype=torch.int32, device=dev)
        if not self.nb:
            d.edge_index = torch.zeros(2, self.e_cap, dtype=torch.int64, device=dev)
        d._hgb_valid = self.valid
        if self.periodic:
            self.cutoff = torch.full((self.g_cap,), float(self.nb[0]), dtype=torch.float64, device=dev)
        self.data, self.hosts, self._turn = d, hosts, 0
        self._copied = [None, None]
        self._captured = False

    def _prologue(self):
        """The first part of every captured body: the edges of the batch (built from ``pos``, or the loaded ones padded with
        the filler edges) and the index plans rebuilt in the captured region."""
        d = self.data
        if self.periodic:
            ei, _, d.edge_shifts, _, outptr, _ = radius.radius_graph_pbc(d.pos.detach(), d.cell, d.pbc, self.cutoff, d.ptr, self.g_cap,
                                                                         int(self.nb[1]), capacity=(self.cand_cap, self.e_cap))
            d.edge_index = ei
            e_real = outptr[-1:]
        elif self.nb:
            r, k = self.nb
            ei, rowptr = radius.radius_graph(d.pos.detach(), float(r), d.ptr, self.g_cap, False, int(k), capacity=self.e_cap)
            d.edge_index = ei
            e_real = rowptr[-1:]
        else:
            e_real = self.valid[2:3]
        _lib.call("hgb_pad_edges", _p(e_real), _p(self.valid[1:2]), self.n_cap, self.e_cap, _p(d.edge_index), _p(ops.guard_flag(self.dev)),
                  _stream())
        forget_plans(d)                     # index plans are part of the step: every batch brings new edges and elements

    # ---- per batch ------------------------------------------------------------------------------------------------------
    def load(self, batch, **extra):
        """Pad ``batch`` (CPU or CUDA tensors) and the per-graph ``extra`` fields into the static buffers.  Re-captures with
        grown capacities when it does not fit."""
        n, g = int(batch.pos.shape[0]), int(batch.num_graphs)
        e = 0 if self.nb else int(batch.edge_index.shape[1])
        unused = self.g_cap - g
        if unused < 1 or self.n_cap - n < 2 * unused or (not self.nb and e > self.e_cap):
            self._capture(max(n, int(self.n_cap / self.slack)), max(e, 0 if self.nb else int(self.e_cap / self.slack)), max(g, self.g_cap - 1))
            self.recaptures += 1
            unused = self.g_cap - g
        self._turn ^= 1
        h, d = self.hosts[self._turn], self.data
        if self._copied[self._turn] is not None:
            self._copied[self._turn].synchronize()          # the copy that last read this staging set has finished (two steps ago)
        # filler atoms: two per unused slot, the rest in the last slot; on a line 1.5 A apart
        ptr, bfull, fill = filler_layout(batch.batch.to("cpu", torch.int64), g, self.n_cap, self.g_cap)
        h["ptr"].copy_(ptr)
        h["batch"].copy_(bfull)
        h["valid"][0], h["valid"][1], h["valid"][2] = g, n, e
        for key in self._widths:
            if key not in h:
                continue
            stage(h[key], key, (extra[key] if key in self._extra else batch[key]).to("cpu"), g, n, fill)
        if not self.nb:
            h["edge_index"][:, :e] = batch.edge_index.to("cpu")
        for key, buf in h.items():
            dst = self.valid if key == "valid" else d[key]
            dst.detach().copy_(buf, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._copied[self._turn] = ev
        self.real = g, n
        if not self._captured:
            self._do_capture()
        return g

    def check(self):
        ops.check_guard(self.dev)


class PaddedGraphStep(PaddedBatch):
    def __init__(self, model, opt, first_batch, compute_grad_energy=False, neighbour_build=None, node_cap=None, edge_cap=None,
                 graph_cap=None, slack=1.12, warmup=2, capture_allreduce=True):
        """``first_batch``: a representative (CPU or CUDA) batch -- sizes capacities, field widths and dtypes.
        ``neighbour_build`` = (radius, max_neighbours): build the radius graph inside the captured step from ``pos``;
        None: ``edge_index`` (+ ``edge_shifts``) arrive with every batch."""
        if not supported(model):
            raise ValueError("PaddedGraphStep: this model (global attention / node heads / branches of differing architectures) "
                             "needs the eager train_step")
        self.opt, self.mlip = opt, bool(compute_grad_energy)
        self.hyper = None                                   # what the captured optimizer step holds besides lr (_do_capture)
        self.ws = dist.get_world_size() if dist.is_initialized() else 1
        self.capture_allreduce = capture_allreduce
        super().__init__(model, first_batch, neighbour_build, node_cap, edge_cap, graph_cap, slack, warmup)

    def _capture(self, n_need, e_need, g_need):
        super()._capture(n_need, e_need, g_need)
        self.g_fb = self.g_opt = None

    def _masked_loss(self, pred):
        m, d = self.m, self.data
        inner = getattr(m, "model", m)
        var = None
        if inner.var_output:                                 # mean-and-variance heads: the NLL over the real graphs only
            pred, var = pred
        tot, tasks, off = 0, [], 0
        for ih in range(inner.num_heads):
            w = inner.head_dims[ih]
            tgt = d.y[:, off:off + w] if d.y.dim() == 2 else d.y.reshape(-1, 1)
            off += w
            if var is None:
                li = inner.loss_function.masked(pred[ih], tgt.contiguous(), self.valid[0:1], w)
            else:
                li = inner.loss_function.masked(pred[ih], tgt.contiguous(), var[ih], self.valid[0:1], w)
            tot = tot + li * inner.loss_weights[ih]
            tasks.append(li)
        return tot, tasks

    def _step_body(self, with_opt):
        d, m = self.data, self.m
        self._prologue()
        self.opt.zero_grad()
        if self.mlip:
            d.pos.requires_grad_(True)
            loss, tasks = m.energy_force_loss(self.model(d), d)
        else:
            loss, tasks = self._masked_loss(self.model(d))
        self.opt.backward(loss)
        if with_opt:
            if self.ws > 1:
                dist.all_reduce(self.opt.flat_g)
            self.opt.step(1.0 / self.ws)
        self.loss, self.tasks = loss.detach(), torch.stack([t.detach() for t in tasks])

    def _do_capture(self):
        self.opt.sync_hyper(1.0 / self.ws)
        self.hyper = self.opt.captured_hyper()
        # warm-up on a side stream WITHOUT touching the parameters' trajectory: run the body, then restore
        state = self.opt.state_tensors()
        keep = [self.opt.flat_p.clone()] + [t.clone() for t in state]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self._step_body(True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        one = self.ws == 1 or self.capture_allreduce
        self.g_fb = torch.cuda.CUDAGraph()
        with ops.capture_graph(self.g_fb):
            self._step_body(one)
        if not one:
            self.g_opt = torch.cuda.CUDAGraph()
            with ops.capture_graph(self.g_opt):
                self.opt.step(1.0 / self.ws)
        for dst, src in zip([self.opt.flat_p] + state, keep):
            dst.copy_(src)
        self._captured = True

    def run(self):
        self.opt.sync_hyper()
        self.g_fb.replay()
        if self.g_opt is not None:
            dist.all_reduce(self.opt.flat_g)
            self.g_opt.replay()
        return self.loss, self.tasks
