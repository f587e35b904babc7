"""fp64 CPU restatement of the reference's MACE with graph-attribute conditioning, built on tests/mace_edge_oracle.py.

hydragnn/models/Base.py:97-106 checks the mode, :249-297 creates the conditioning modules at the first forward (on the CPU
generator), :299-391 conditions the invariant channels; MACEStack.forward (:375-421) applies it after the embedding and after
each convolution, after that layer's readout.  "fuse_pool" only checks graph_attr: MACEStack never pools with it.
tests/golden/models_mace_cond.pt pins this against the reference's code.
"""
import torch
from torch import nn

from mace_edge_oracle import MACEEdgeOracle
from oracle.geometry import edge_vectors_and_lengths, segment_sum
from oracle import e3


class MACECondOracle(MACEEdgeOracle):
    def __init__(self, *args, use_graph_attr_conditioning=False, graph_attr_conditioning_mode="concat_node", **kwargs):
        self.use_graph_attr_conditioning = use_graph_attr_conditioning
        self.graph_attr_conditioning_mode = graph_attr_conditioning_mode.lower()
        if self.graph_attr_conditioning_mode not in ("film", "concat_node", "fuse_pool"):
            raise ValueError("graph_attr_conditioning_mode must be one of: 'film', 'concat_node', 'fuse_pool'.")
        super().__init__(*args, **kwargs)
        self.graph_conditioner = None
        self.graph_concat_projector = None
        self.graph_concat_projector_in_dim = None
        self.device = torch.device("cpu")          # Base.py:66; read by load_existing_model

    def _ensure_graph_conditioner(self, graph_attr_dim, device):
        if self.graph_conditioner is None:
            hidden = max(self.hidden_dim, graph_attr_dim)
            self.graph_conditioner = nn.Sequential(nn.Linear(graph_attr_dim, hidden), self.activation_function, nn.Linear(hidden, 2 * self.hidden_dim))
        self.graph_conditioner = self.graph_conditioner.to(device=device, dtype=self.node_embedding.linear.weight.dtype)

    def _ensure_graph_concat_projector(self, graph_attr_dim, channel_dim, device, dtype=None):
        in_dim = channel_dim + graph_attr_dim
        if self.graph_concat_projector is None or self.graph_concat_projector_in_dim != in_dim:
            self.graph_concat_projector = nn.Linear(in_dim, channel_dim)
            self.graph_concat_projector_in_dim = in_dim
        self.graph_concat_projector = self.graph_concat_projector.to(device=device,
                                                                     dtype=dtype or self.node_embedding.linear.weight.dtype)

    def condition(self, inv, batch, data, num_graphs):
        if not self.use_graph_attr_conditioning:
            return inv
        ga = getattr(data, "graph_attr", None)
        if ga is None:
            raise ValueError("use_graph_attr_conditioning=True but data.graph_attr is missing.")
        ga = ga.to(device=inv.device, dtype=inv.dtype)
        if ga.dim() == 1:
            if ga.numel() % num_graphs:
                raise ValueError(f"One-dimensional graph_attr with numel={ga.numel()} is not divisible by num_graphs={num_graphs}.")
            ga = ga.view(num_graphs, ga.numel() // num_graphs)
        elif ga.dim() == 2:
            if ga.size(0) != num_graphs:
                raise ValueError(f"graph_attr first dim {ga.size(0)} does not match num_graphs={num_graphs}.")
        else:
            raise ValueError(f"Unsupported graph_attr ndim={ga.dim()}; expected 1/2.")
        mode = self.graph_attr_conditioning_mode
        if mode == "film":
            self._ensure_graph_conditioner(ga.size(-1), inv.device)
            scale, shift = self.graph_conditioner(ga).split(self.hidden_dim, dim=-1)
            return inv * (1 + torch.tanh(scale)[batch]) + shift[batch]
        if mode == "concat_node":
            self._ensure_graph_concat_projector(ga.size(-1), inv.size(-1), inv.device, inv.dtype)
            return self.graph_concat_projector(torch.cat([inv, ga[batch]], dim=-1))
        return inv

    def forward(self, data):
        pos, batch = data.pos, data.batch
        num_graphs = int(data.num_graphs)
        dtype = self.node_embedding.linear.weight.dtype
        mean_pos = segment_sum(pos, batch, num_graphs) / segment_sum(torch.ones_like(pos[:, :1]), batch, num_graphs).clamp(min=1)
        pos = pos - mean_pos[batch]
        shifts = getattr(data, "edge_shifts", None)
        vec, dist = edge_vectors_and_lengths(pos, data.edge_index, shifts)
        attrs = self.node_attributes(data.x).to(dtype)
        feats = self.node_embedding.linear(attrs)
        edge_attrs = e3.spherical_harmonics(self.max_ell, vec, normalize=True, normalization="component")
        if self.edge_dim:
            edge_attrs = torch.cat([data.edge_attr.to(edge_attrs.dtype), edge_attrs], dim=1)
        edge_feats = self.radial_embedding(dist)
        inv, equiv = feats[:, :self.hidden_dim], feats[:, self.hidden_dim:]
        inv = self.condition(inv, batch, data, num_graphs)
        ds = getattr(data, "dataset_name", None)
        outputs = self.multihead_decoders[0](attrs, batch, num_graphs, ds)
        for conv, readout in zip(self.graph_convs, self.multihead_decoders[1:]):
            inv, equiv = conv(inv, equiv, attrs, edge_attrs, edge_feats, data.edge_index)
            out = readout(torch.cat([inv, equiv], dim=1), batch, num_graphs, ds)
            inv = self.condition(inv, batch, data, num_graphs)
            outputs = [a + b for a, b in zip(outputs, out)]
        return outputs
