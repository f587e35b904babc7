"""CGCNN stack on libhgb.so.

Host-side mirror of ``hydragnn/models/CGCNNStack.py`` with torch_geometric 2.6.1 ``CGConv(channels, dim, aggr="add",
batch_norm=False, bias=True)`` and the default ``Base._init_conv`` (hydragnn/models/Base.py:446-463): every conv is followed
by a PyG ``BatchNorm(hidden_dim)`` feature layer.  Module and parameter names are the reference's
(``graph_convs.<i>.module_0.{lin_f, lin_s}``, under GPS ``graph_convs.<i>.conv.module_0``, ``feature_layers.<i>.module``), so
reference checkpoints load.

CGConv's two Linears act on z_e = [x_i | x_j | a_e] (i = edge_index[1] the target, j the source) and are affine in its blocks:
with W_f = [A_f | B_f | C_f] (and W_s alike) one per-node Linear gives [P_f | P_s | Q_f | Q_s] = x [A_f; A_s; B_f; B_s]^T, and
``ops.CgConvFn`` forms f_e = P_f[i] + Q_f[j] + C_f a_e + b_f and s_e in registers, gates them and sums
sigmoid(f_e) * softplus(s_e) onto the residual x_i.  Under GPS the conv's edge input is linear in the raw r_e = [edge_attr |
rel_pe] (or rel_pe alone), so the kernel takes Mt = ((C_f; C_s) L)^T with L built from the bias-free embedding weights
(``Base._raw_edge_input``), and the [E, hidden] edge embedding is never formed.  Higher-order passes and shapes
``ops.cgconv_supported`` refuses run the same math composed from GatherRows, Linear, ATen sigmoid / softplus and SegmentSum.
"""
import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .ops import GatherRows, SegmentSum
from .gps import PyGBatchNorm
from .stacks import Base, SingleConv


class CGConv(nn.Module):
    """torch_geometric 2.6.1 ``CGConv(channels, dim, aggr="add", batch_norm=False, bias=True)``: ``lin_f`` and ``lin_s`` are
    ``Linear(2 channels + dim, channels)``, drawn at construction and again by ``reset_parameters`` (lin_f, then lin_s), as PyG
    does: the second draw fixes the seeded values."""

    def __init__(self, channels, dim=0):
        super().__init__()
        self.channels, self.dim = channels, dim
        self.lin_f = nn.Linear(2 * channels + dim, channels)
        self.lin_s = nn.Linear(2 * channels + dim, channels)
        self.reset_parameters()

    def reset_parameters(self):
        self.lin_f.reset_parameters()
        self.lin_s.reset_parameters()

    def forward(self, x, plan, edge_raw=None, higher_order=False):
        """``edge_raw`` = (r, L): the conv's edge input is r L^T (L None: r itself), or None without one."""
        r, emb = edge_raw if edge_raw is not None else (None, None)
        if (self.dim > 0) != (r is not None):
            # PyG would hand a z of the wrong width to lin_f and fail; dropping the C columns would run another model
            raise ValueError("CGConv was built with dim=%d but called %s edge_attr" % (self.dim, "without" if r is None else "with"))
        fc = self.channels
        w = torch.cat([self.lin_f.weight, self.lin_s.weight], dim=0)                  # [2F, 2F + dim] = [A | B | C]
        cvec = torch.cat([self.lin_f.bias, self.lin_s.bias])
        tgt = plan.by_col                                                            # aggr "add" at i = edge_index[1]
        if not higher_order and x.is_cuda and ops.cgconv_supported(fc, 0 if r is None else r.shape[1]):
            pq = ops.linear_act(x, torch.cat([w[:, :fc], w[:, fc:2 * fc]], dim=0), None)     # [N, 4F] = [P_f | P_s | Q_f | Q_s]
            mt = None
            if r is not None:
                c = w[:, 2 * fc:]
                mt = c.t() if emb is None else ops.MatMul.apply(emb, c, True, True)          # (C L)^T  [d, 2F]
            return ops.CgConvFn.apply(pq, r, mt, cvec, x, plan)
        lin = ops.linear_any_order if higher_order else ops.linear_act
        h = GatherRows.apply(lin(x, w[:, :fc], None), tgt) + GatherRows.apply(lin(x, w[:, fc:2 * fc], None), plan.by_row)
        if r is not None:
            h = h + lin(r if emb is None else lin(r, emb, None), w[:, 2 * fc:], cvec)
        else:
            h = h + cvec
        m = torch.sigmoid(h[:, :fc]) * F.softplus(h[:, fc:])
        return SegmentSum.apply(m, tgt) + x


class CGCNNStack(Base):
    is_edge_model = True

    def __init__(self, edge_dim, *args, **kwargs):
        self.edge_dim = edge_dim
        super().__init__(*args, **kwargs)

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def get_conv(self, input_dim, output_dim=None, last_layer=False, edge_dim=None):
        # CGConv keeps its width: the reference passes input_dim as the channels and ignores output_dim
        if edge_dim is None:
            raise ValueError("CGCNN needs an integer edge_dim without global attention (update_config sets 0 when there are no "
                             "edge features); PyG's CGConv fails computing sum(channels) + None")
        return SingleConv(CGConv(input_dim, edge_dim))

    def _init_node_conv(self):
        """CGCNNStack._init_node_conv (:84-110), statement for statement: conv-type node heads are not built.  It raises the
        reference's ValueError for a node branch whose own "type" is "conv"; other conv-type configurations fail where the
        reference's fail (a missing key here, or in Base._multihead)."""
        node_feature_ind = [i for i, head_type in enumerate(self.head_type) if head_type == "node"]
        if len(node_feature_ind) == 0:
            return
        nodeconfiglist = self.config_heads["node"]
        for branchdict in nodeconfiglist:
            if branchdict["architecture"]["type"] != "conv":
                return
        self.num_conv_layers_node = nodeconfiglist[0]["num_headlayers"]
        self.hidden_dim_node = nodeconfiglist[0]["dim_headlayers"]
        for ihead in range(self.num_heads):
            for branchdict in nodeconfiglist:
                assert self.num_conv_layers_node == branchdict["num_headlayers"]
                assert self.hidden_dim_node == branchdict["dim_headlayers"]
                if self.head_type[ihead] == "node" and branchdict["type"] == "conv":
                    raise ValueError(
                        '"conv" for node features decoder part in CGCNN is not ready yet. Please set config["NeuralNetwork"]'
                        '["Architecture"]["output_heads"]["node"]["type"] to be "mlp" or "mlp_per_node" in input file.')

    def _forward(self, data, higher):
        if not self.use_global_attn and self.hidden_dim != self.input_dim:
            # the convs keep input_dim channels while the feature layers are BatchNorm(hidden_dim): the reference fails at the
            # first BatchNorm, so no kernel is launched here (update_config sets hidden_dim = input_dim without GPS)
            raise ValueError("CGCNN without global attention runs at input_dim = %d channels but hidden_dim is %d"
                             % (self.input_dim, self.hidden_dim))
        return super()._forward(data, higher)

    def _embedding(self, data, plan, higher):
        x, edge_raw = self._raw_edge_input(data, higher)
        return x, data.pos, {"edge_raw": edge_raw}

    def __str__(self):
        return "CGCNNStack"
