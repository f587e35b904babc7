"""Oracle: model assembly (encoder loop, pooling, multi-head decoder).

Test infrastructure only.  Restates ``Base`` (hydragnn/models/Base.py:36-982) once, as
``StackOracle``, which every oracle stack subclasses; ``EGCLStack``
(hydragnn/models/EGCLStack.py:22-152), ``PAINNStack`` (hydragnn/models/PAINNStack.py:27-191)
and ``PNAEqStack`` as ``OracleModel``; and the ``create_model`` dispatch
(hydragnn/models/create.py:112-584) over every stack.  The PNA, PNAPlus, CGCNN, GAT, SchNet,
SAGE, MFC and MACE stacks are in oracle/{pna,pnaplus,cgcnn,gat,schnet,sage,mace}.py.
Parameter names follow the reference (PyG ``Sequential`` names its children ``module_<i>``
[3P-memory B.5]) so state dicts interchange with the engine.
"""
import torch
from torch import nn

from .egnn import EGCL
from .geometry import edge_vectors_and_lengths, graph_pool
from .painn import PainnMessage, PainnUpdate
from . import pnaeq
from .gps import GPSConv, PyGBatchNorm


def activation(name):
    """hydragnn/utils/model/model.py:30-46."""
    table = {
        "relu": nn.ReLU, "selu": nn.SELU, "prelu": nn.PReLU, "elu": nn.ELU,
        "lrelu_01": lambda: nn.LeakyReLU(0.1), "lrelu_025": lambda: nn.LeakyReLU(0.25),
        "lrelu_05": lambda: nn.LeakyReLU(0.5), "sigmoid": nn.Sigmoid,
    }
    return table[name]() if name in table else None


def loss_function(name):
    """hydragnn/utils/model/model.py:49-62."""
    F = torch.nn.functional
    if name == "mse":
        return F.mse_loss
    if name == "mae":
        return F.l1_loss
    if name == "rmse":
        return lambda a, b: torch.sqrt(F.mse_loss(a, b))
    if name == "GaussianNLLLoss":
        return torch.nn.GaussianNLLLoss()
    raise ValueError("oracle supports mse / mae / rmse / GaussianNLLLoss, got " + str(name))


def normalize_heads(output_heads):
    """``update_multibranch_heads`` (hydragnn/utils/model/model.py:314-349)."""
    out = {}
    for key, val in output_heads.items():
        out[key] = val if isinstance(val, list) else [{"type": "branch-0", "architecture": val}]
    return out


class _Conv(nn.Module):
    """Stand-in for the PyG ``Sequential`` built by ``get_conv``; holds children under
    the names PyG would give them."""

    def __init__(self, mods):
        super().__init__()
        for i, m in enumerate(mods):
            if m is not None:
                self.add_module("module_%d" % i, m)


class StackOracle(nn.Module):
    """``Base`` (hydragnn/models/Base.py:36-982): loss weights and pooling, the GPS node and edge embeddings, the encoder loop,
    ``graph_shared``, the graph heads, the ``mlp`` / ``mlp_per_node`` / ``conv`` node heads, single- and multi-branch decoding and
    ``loss_hpweighted``.  Under ``loss_function_type="GaussianNLLLoss"`` every head is a mean-and-variance head: its last layer
    is ``(1 + var_output) d`` wide, ``forward`` returns (means, variances) and the loss is ``GaussianNLLLoss`` per head; all
    three follow the ``loss_function_type`` given to this constructor.  Graph-attribute conditioning is refused: only MACE's
    is restated.  A stack sets its own attributes (``edge_dim`` first of all) before calling this constructor and supplies the
    hooks the reference's stacks override:

    * ``_get_conv(fin, fout, last, edge_dim=None)``: one conv under the reference's child names;
    * ``_feature_layer(width)``: what follows every encoder conv (Identity here, a BatchNorm in ``Base._init_conv``);
    * ``_conv_width(fout, last)``: what a conv built for ``fout`` outputs (GAT's concat convs: ``fout`` times its heads);
    * ``_embedding(data) -> (x, equiv, ctx)``: the per-forward node features, equivariant features and context every conv reads;
    * ``_run_conv(conv, x, equiv, ctx) -> (x, equiv)``: one conv, unwrapped from GPS.

    ``_init_conv`` and ``_init_node_conv`` are overridden where the reference's stack overrides them.
    """

    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, activation_function="relu",
                 loss_function_type="mse", task_weights=None, num_conv_layers=2, num_nodes=None, equivariance=False,
                 graph_pooling="mean", global_attn_engine=None, global_attn_type=None, global_attn_heads=0, pe_dim=0, dropout=0.25,
                 use_graph_attr_conditioning=False, **_unused):
        super().__init__()
        if use_graph_attr_conditioning:
            raise ValueError("oracle restates graph-attribute conditioning for MACE only")
        self.use_global_attn = bool(global_attn_engine)
        if self.use_global_attn and (global_attn_engine != "GPS" or global_attn_type != "multihead"):
            raise ValueError("oracle supports global_attn_engine='GPS' with global_attn_type='multihead'")
        self.global_attn_heads, self.pe_dim, self.dropout = global_attn_heads, pe_dim, dropout
        self.input_dim, self.hidden_dim = input_dim, hidden_dim
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        self.num_heads = len(self.head_dims)
        self.config_heads = normalize_heads(output_heads)
        self.activation_function = activation(activation_function)
        self.loss_function_type = loss_function_type
        self.loss_function = loss_function(loss_function_type)
        w = list(task_weights if task_weights is not None else [1.0] * self.num_heads)
        if len(w) != self.num_heads:
            raise ValueError("Inconsistent number of loss weights and tasks")
        tot = sum(abs(t) for t in w)
        self.loss_weights = [t / tot for t in w]                           # Base.py:121-132
        mode = graph_pooling.lower()
        self.graph_pooling = "add" if mode == "sum" else mode
        self.num_conv_layers, self.num_nodes = num_conv_layers, num_nodes
        self.equivariance = bool(equivariance)
        self.use_edge_attr = self.edge_dim is not None and self.edge_dim > 0   # Base.py:135-141
        if self.use_global_attn:                                               # Base.py:179-215
            self.embed_dim = self.edge_embed_dim = hidden_dim
            self.pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if input_dim:
                self.node_emb = nn.Linear(input_dim, hidden_dim, bias=False)
                self.node_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
            self.rel_pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if self.use_edge_attr:
                self.edge_emb = nn.Linear(self.edge_dim, hidden_dim, bias=False)
                self.edge_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
        else:
            self.embed_dim, self.edge_embed_dim = input_dim, self.edge_dim
        self.graph_convs, self.feature_layers = nn.ModuleList(), nn.ModuleList()
        self._init_conv()
        self._multihead()

    def _wrap(self, conv):
        """Base._apply_global_attn (:234-247)."""
        return GPSConv(self.hidden_dim, conv, heads=self.global_attn_heads, dropout=self.dropout) if self.use_global_attn else conv

    def _init_conv(self):
        """First layer at embed_dim (= input_dim without GPS, Q4), last layer flagged (EGCLStack.py:45-70, Base.py:446-463)."""
        for i in range(self.num_conv_layers):
            last = i == self.num_conv_layers - 1
            conv = self._get_conv(self.embed_dim if i == 0 else self.hidden_dim, self.hidden_dim, last, edge_dim=self.edge_embed_dim)
            self.graph_convs.append(self._wrap(conv))
            self.feature_layers.append(self._feature_layer(self.hidden_dim))

    def _feature_layer(self, width):
        return nn.Identity()

    def _multihead(self):
        """Base._multihead (:590-691), single or multi branch."""
        act = self.activation_function
        self.heads_NN = nn.ModuleList()          # registered before graph_shared, as in Base.__init__:83
        self.convs_node_hidden, self.batch_norms_node_hidden = nn.ModuleDict(), nn.ModuleDict()       # Base.py:88-91
        self.convs_node_output, self.batch_norms_node_output = nn.ModuleDict(), nn.ModuleDict()
        self.graph_shared = nn.ModuleDict()
        self.num_branches = 1
        if "graph" in self.config_heads:
            self.num_branches = len(self.config_heads["graph"])
            for br in self.config_heads["graph"]:
                a = br["architecture"]
                layers = [nn.Linear(self.hidden_dim, a["dim_sharedlayers"]), act]
                for _ in range(a["num_sharedlayers"] - 1):
                    layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), act]
                self.graph_shared[br["type"]] = nn.Sequential(*layers)
        if "node" in self.config_heads:
            self._init_node_conv()
        inode = 0
        for ih in range(self.num_heads):
            head = nn.ModuleDict()
            if self.head_type[ih] == "graph":
                for br in self.config_heads["graph"]:
                    a = br["architecture"]
                    dims = [a["dim_sharedlayers"]] + list(a["dim_headlayers"][: a["num_headlayers"]])
                    layers = []
                    for d0, d1 in zip(dims[:-1], dims[1:]):
                        layers += [nn.Linear(d0, d1), act]
                    layers.append(nn.Linear(dims[-1], self._out_width(ih)))
                    head[br["type"]] = nn.Sequential(*layers)
            elif self.head_type[ih] == "node":
                for br in self.config_heads["node"]:
                    a = br["architecture"]
                    if a["type"] in ("mlp", "mlp_per_node"):                       # Base.py:648-664
                        per_node = a["type"] == "mlp_per_node"
                        if per_node:
                            assert self.num_nodes is not None, "num_nodes must be provided for mlp_per_node; use 'mlp' for variable-size graphs"
                        head[br["type"]] = _MLPNode(self.hidden_dim, self._out_width(ih), a["dim_headlayers"], act,
                                                    num_mlp=self.num_nodes if per_node else 1, num_nodes=self.num_nodes if per_node else None)
                    elif a["type"] == "conv":                                       # Base.py:665-680: the SAME modules, listed again
                        key, mods = br["type"], nn.ModuleList()
                        for conv, bn in zip(self.convs_node_hidden[key], self.batch_norms_node_hidden[key]):
                            mods.append(conv)
                            mods.append(bn)
                        mods.append(self.convs_node_output[key][inode])
                        mods.append(self.batch_norms_node_output[key][inode])
                        head[key] = mods
                        inode += 1
                    else:
                        raise ValueError("Unknown head NN structure for node features" + a["type"])
            else:
                raise ValueError("Unknown head type" + str(self.head_type[ih]))
            self.heads_NN.append(head)

    def _init_node_conv(self):
        """Base._init_node_conv (:508-588): conv-type node heads share their hidden convolutions between heads."""
        cfgs = self.config_heads["node"]
        if any(br["architecture"]["type"] != "conv" for br in cfgs):
            return
        node_heads = [i for i, t in enumerate(self.head_type) if t == "node"]
        if not node_heads:
            return
        for br in cfgs:
            a = br["architecture"]
            hid = a["dim_headlayers"]
            ch, bh, co, bo = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
            w = self._conv_width
            ch.append(self._get_conv(self.hidden_dim, hid[0], False))
            bh.append(PyGBatchNorm(w(hid[0], False)))
            for k in range(a["num_headlayers"] - 1):
                ch.append(self._get_conv(w(hid[k], False), hid[k + 1], False))
                bh.append(PyGBatchNorm(w(hid[k + 1], False)))
            for ih in node_heads:
                co.append(self._get_conv(w(hid[-1], False), self._out_width(ih), True))
                bo.append(PyGBatchNorm(w(self._out_width(ih), True)))
            key = br["type"]
            self.convs_node_hidden[key], self.batch_norms_node_hidden[key] = ch, bh
            self.convs_node_output[key], self.batch_norms_node_output[key] = co, bo

    def _var_output(self):
        """``var_output`` (Base.py:109-111): 1 under GaussianNLLLoss, else 0."""
        return int(self.loss_function_type == "GaussianNLLLoss")

    def _out_width(self, ih):
        """Width of head ``ih``'s last layer: the mean, then the variance's square root under GaussianNLLLoss."""
        return self.head_dims[ih] * (1 + self._var_output())

    def _conv_width(self, fout, last):
        """Width of what a conv built for ``fout`` outputs."""
        return fout

    def _node_edge_features(self, data):
        """(x, edge_attr) entering the first conv: the input features, or the GPS node and edge embeddings (Base._embedding
        :477-491)."""
        eattr = data.edge_attr if self.use_edge_attr else None
        if not self.use_global_attn:
            return data.x, eattr
        x = self.pos_emb(data.pe)
        if self.input_dim:
            x = self.node_lin(torch.cat((self.node_emb(data.x.to(x.dtype)), x), 1))
        e = self.rel_pos_emb(data.rel_pe)
        if self.use_edge_attr:
            e = self.edge_lin(torch.cat((self.edge_emb(eattr), e), 1))
        return x, e

    def _embedding(self, data):
        x, eattr = self._node_edge_features(data)
        return x, None, {"edge_index": data.edge_index, "edge_attr": eattr}

    def _layer(self, conv, x, equiv, ctx):
        """One encoder conv, through GPSConv when global attention is on."""
        if self.use_global_attn:
            return conv(x, equiv, lambda a, b: self._run_conv(conv.conv, a, b, ctx))
        return self._run_conv(conv, x, equiv, ctx)

    def forward(self, data):
        x, equiv, ctx = self._embedding(data)
        for conv, feat in zip(self.graph_convs, self.feature_layers):
            x, equiv = self._layer(conv, x, equiv, ctx)
            x = self.activation_function(feat(x))                             # Base.py:726
        batch = getattr(data, "batch", None)
        if batch is None:
            batch = torch.zeros(x.shape[0], dtype=torch.long, device=x.device)
        G = int(batch.max()) + 1
        xg = graph_pool(x, batch, G, self.graph_pooling)                     # Base.py:733-738
        ds = getattr(data, "dataset_name", None)
        outs = []
        for ih, (head, kind) in enumerate(zip(self.heads_NN, self.head_type)):
            if self.num_branches == 1:
                if kind == "graph":
                    outs.append(head["branch-0"](self.graph_shared["branch-0"](xg)))
                elif isinstance(head["branch-0"], nn.ModuleList):          # conv-type node head (Base.py:800-810)
                    a, b = x, equiv
                    mods = head["branch-0"]
                    for conv, bn in zip(mods[0::2], mods[1::2]):
                        a, b = self._run_conv(conv, a, b, ctx)
                        a = self.activation_function(bn(a))
                    outs.append(a)
                else:
                    outs.append(head["branch-0"](x, batch))
                continue
            # multi-branch masking (Base.py:770-780, 816-840)
            ids = ds[:, 0]
            if kind == "graph":
                out = x.new_zeros(G, self._out_width(ih))
                for b in ids.unique():
                    m = ids == b
                    key = "branch-%d" % int(b)
                    out[m] = head[key](self.graph_shared[key](xg[m]))
            else:
                out = x.new_zeros(x.shape[0], self._out_width(ih))
                for b in ids.unique():
                    m = (ids == b)[batch]
                    if isinstance(head["branch-%d" % int(b)], nn.ModuleList):
                        raise ValueError("oracle: conv-type node heads with several branches are not restated")
                    out[m] = head["branch-%d" % int(b)](x[m], batch[m])
            outs.append(out)
        mean = [o[:, :hd] for o, hd in zip(outs, self.head_dims)]          # Base.py:764-846
        if not self._var_output():
            return mean
        return mean, [o[:, hd:] ** 2 for o, hd in zip(outs, self.head_dims)]

    def loss(self, pred, value, head_index):
        """``loss_hpweighted`` (Base.py:848-906); ``pred`` is (means, variances) under GaussianNLLLoss."""
        pred, var = pred if self._var_output() else (pred, None)
        tot, tasks = 0, []
        for ih in range(self.num_heads):
            tgt = value[head_index[ih]].reshape(pred[ih].shape).to(pred[ih].dtype)
            li = self.loss_function(pred[ih], tgt) if var is None else self.loss_function(pred[ih], tgt, var[ih])
            tot = tot + li * self.loss_weights[ih]
            tasks.append(li)
        return tot, tasks


class OracleModel(StackOracle):
    """``EGCLStack`` (hydragnn/models/EGCLStack.py:22-152), ``PAINNStack`` (hydragnn/models/PAINNStack.py:27-191) and
    ``PNAEqStack`` (hydragnn/models/PNAEqStack.py) on the skeleton, chosen by ``mpnn_type``."""

    def __init__(self, mpnn_type, input_dim, hidden_dim, output_dim, output_type, output_heads, edge_dim=None, num_radial=None,
                 radius=None, pna_deg=None, **kw):
        if mpnn_type == "PNAEq":
            assert pna_deg is not None, "PNAEq requires degree input."
            self.deg = pnaeq.sanitize_degree(pna_deg)
        if mpnn_type not in ("EGNN", "PAINN", "PNAEq"):
            raise ValueError("Unknown mpnn_type: {0}".format(mpnn_type))
        self.mpnn_type, self.num_radial, self.radius = mpnn_type, num_radial, radius
        if mpnn_type == "EGNN":
            self.edge_dim = 0 if edge_dim is None else edge_dim            # EGCLStack.py:33-35
        else:
            self.edge_dim = edge_dim                                        # PAINNStack.py:43
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)

    # EGCLStack.get_conv :72-109 / PAINNStack.get_conv :76-147
    def _get_conv(self, fin, fout, last, edge_dim=None):
        ed = self.edge_embed_dim                                        # hidden_dim under GPS, else the stack's edge_dim
        if self.mpnn_type == "EGNN":
            return _Conv([EGCL(fin, fout, self.hidden_dim, edge_attr_dim=ed or self.edge_dim,
                               equivariant=self.equivariance and not last)])
        if self.mpnn_type == "PNAEq":                                   # PNAEqStack.get_conv :119-192
            msg = pnaeq.PainnMessage(fin, self.deg, ed, self.num_radial)
            upd = pnaeq.PainnUpdate(fin, last_layer=last)
        else:
            msg = PainnMessage(fin, self.num_radial, self.radius, edge_dim=ed)
            upd = PainnUpdate(fin, last_layer=last)
        s_out = nn.Sequential(nn.Linear(fin, fout), nn.Tanh(), nn.Linear(fout, fout))
        v_out = None if last else nn.Linear(fin, fout)
        return _Conv([msg, upd, s_out, v_out])

    def _embedding(self, data):
        x, eattr = self._node_edge_features(data)
        pos, ei = data.pos, data.edge_index.to(torch.long)
        shifts = getattr(data, "edge_shifts", None)
        if shifts is None:                                                   # Base.py:466-469
            shifts = torch.zeros(ei.shape[1], 3, dtype=pos.dtype, device=pos.device)
        ctx = {"edge_index": ei, "edge": ei.t(), "edge_attr": eattr, "shifts": shifts}
        if self.mpnn_type == "EGNN":
            return x, pos, ctx
        # PAINNStack.py:157-159 / PNAEqStack.py:202-205
        ctx["vec"], ctx["dist"] = edge_vectors_and_lengths(pos, ei, shifts, normalize=True)
        if self.mpnn_type == "PNAEq":
            ctx["rbf"] = pnaeq.rbf_basis(ctx["dist"].squeeze(-1), self.num_radial, self.radius)
        return x, torch.zeros(x.shape[0], 3, x.shape[1], dtype=x.dtype, device=x.device), ctx

    def _run_conv(self, c, a, b, ctx):
        if self.mpnn_type == "EGNN":
            return c.module_0(a, b, ctx["edge_index"], ctx["edge_attr"], ctx["shifts"])
        if self.mpnn_type == "PNAEq":
            a, b2 = c.module_0(a, b, ctx["edge"], ctx["rbf"], ctx["vec"], ctx["edge_attr"])
        else:
            a, b2 = c.module_0(a, b, ctx["edge"], ctx["vec"], ctx["dist"], ctx["edge_attr"])
        a, b3 = c.module_1(a, b2)
        a = c.module_2(a)
        return a, (c.module_3(b3) if b3 is not None else b2)


class _MLPNode(nn.Module):
    """``MLPNode`` (Base.py:912-979): one shared MLP ('mlp') or one MLP per node position ('mlp_per_node', graphs of exactly
    ``num_nodes`` atoms: node i of every graph goes through ``mlp[i]``)."""

    def __init__(self, fin, fout, hidden, act, num_mlp=1, num_nodes=None):
        super().__init__()
        self.num_nodes, self.fout = num_nodes, fout
        self.activation_function = act                    # before mlp, as MLPNode (Base.py:929): a PReLU's slope is listed here
        self.mlp = nn.ModuleList()
        for _ in range(num_mlp):
            dims = [fin] + list(hidden)
            layers = []
            for d0, d1 in zip(dims[:-1], dims[1:]):
                layers += [nn.Linear(d0, d1), act]
            layers.append(nn.Linear(dims[-1], fout))
            self.mlp.append(nn.Sequential(*layers))

    def forward(self, x, batch=None):
        if self.num_nodes is None:
            return self.mlp[0](x)
        outs = x.new_zeros(x.shape[0], self.fout)
        for i in range(self.num_nodes):
            outs[i::self.num_nodes] = self.mlp[i](x[i::self.num_nodes])
        return outs


def stack_class(mpnn_type):
    """The oracle stack class of ``mpnn_type`` (create.py:112-584).  Every one takes ``create_model``'s keyword arguments,
    ``mpnn_type`` among them: ``OracleModel`` (EGNN, PAINN and PNAEq) reads it and refuses any other name."""
    from .cgcnn import CGCNNStackOracle
    from .gat import GATStackOracle
    from .mace import MACEOracle
    from .pna import PNAStackOracle
    from .pnaplus import PNAPlusStackOracle
    from .sage import MFCStackOracle, SAGEStackOracle
    from .schnet import SCFStackOracle
    stacks = {"PNA": PNAStackOracle, "PNAPlus": PNAPlusStackOracle, "CGCNN": CGCNNStackOracle, "GAT": GATStackOracle,
              "SAGE": SAGEStackOracle, "MFC": MFCStackOracle, "SchNet": SCFStackOracle, "MACE": MACEOracle}
    return stacks.get(mpnn_type, OracleModel)


def case_kwargs(mpnn_type, case):
    """``create_model`` keyword arguments of a case of tests/golden/models_*.pt: its ``cfg``, the ``deg`` histogram as ``pna_deg``
    and its ``task_weights`` (1.0 per head by default).  The cases' GPS runs use 4 attention heads and 4-wide encodings."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps", False):
        cfg.update(global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4, pe_dim=4)
    if "deg" in case:
        cfg["pna_deg"] = case["deg"]
    return dict(cfg, mpnn_type=mpnn_type, task_weights=case.get("task_weights", [1.0] * len(cfg["output_type"])))


def oracle_from_case(stack, case, state=None, dtype=torch.float64):
    """The oracle stack of a case of tests/golden/models_*.pt, with ``state`` (the case's own by default) loaded strictly, in
    ``dtype``.  ``stack`` is the case's ``mpnn_type``, or an oracle stack class that needs none.  The cases' train-mode steps
    were recorded with dropout off."""
    mpnn_type = stack if isinstance(stack, str) else None
    cls = stack_class(mpnn_type) if mpnn_type else stack
    m = cls(**case_kwargs(mpnn_type, case), dropout=0.0)
    m.load_state_dict(case["state"] if state is None else state, strict=True)
    return m.to(dtype)


def create_model(**kw):
    """Mirror of ``create_model`` (hydragnn/models/create.py:112-766): seeds the RNG
    (:164) and wraps the stack for MLIP training when asked (:586-756)."""
    from .mlip import MLIPWrapper
    torch.manual_seed(0)
    model = stack_class(kw.get("mpnn_type"))(**kw)
    if kw.get("enable_interatomic_potential", False):
        model = MLIPWrapper(model, kw.get("energy_weight", 0.0), kw.get("energy_peratom_weight", 0.0),
                            kw.get("force_weight", 0.0))
    return model
