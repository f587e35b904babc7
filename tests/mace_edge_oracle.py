"""fp64 CPU restatement of the reference's MACE with edge attributes (edge_dim > 0), built on oracle/mace.py.

MACEStack.py:198-203 widens the edge irreps to (Dx0e + sh).simplify() = (D+1)x0e + 1x1o + ..., and :459-461 feeds
cat([edge_attr, sh]) to every interaction.  Nothing else changes: the "uvu" tensor product (oracle/e3.py) already handles
a multiplicity D+1 on its second input, with the path constant sqrt((2 l3 + 1) / (D+1)) for the 0e paths, and the radial
MLP's last layer grows to the new weight_numel.  tests/golden/models_mace_edge.pt pins this against the reference's code.
"""
import math

import torch

from oracle import e3
from oracle.geometry import edge_vectors_and_lengths, segment_sum
from oracle.mace import Interaction, MACEOracle, Product, _MaceConv


class MACEEdgeOracle(MACEOracle):
    def __init__(self, *args, edge_dim=None, **kwargs):
        self.edge_dim = int(edge_dim or 0)              # read by _get_conv during MACEOracle.__init__
        super().__init__(*args, edge_dim=None, **kwargs)

    def _edge_attrs_irreps(self):
        if not self.edge_dim:
            return self.sh_irreps
        return (e3.Irreps("%dx0e" % self.edge_dim) + self.sh_irreps).simplify()

    def _get_conv(self, input_dim, output_dim, first_layer=False, last_layer=False):
        """MACEOracle._get_conv with edge_attrs_irreps in place of sh_irreps for the interaction (MACEStack.py:277-377)."""
        hidden_dim = output_dim if input_dim == 1 else input_dim
        mlp_dim = math.ceil(float(hidden_dim) / 3)
        node_feats_irreps = e3.Irreps(e3.create_irreps_string(input_dim, 0 if first_layer else self.node_max_ell))
        hidden_irreps = e3.Irreps(e3.create_irreps_string(hidden_dim, self.node_max_ell))
        interaction_irreps = (self.sh_irreps * hidden_dim).sort()[0].simplify()
        output_irreps = e3.Irreps(e3.create_irreps_string(output_dim, self.node_max_ell))
        if last_layer:
            hidden_irreps, output_irreps = hidden_irreps[:1], output_irreps[:1]
        inter = Interaction(node_feats_irreps, self._edge_attrs_irreps(), self.edge_feats_irreps, interaction_irreps, hidden_irreps,
                            self.avg_num_neighbors, [mlp_dim] * 3)
        prod = Product(interaction_irreps, hidden_irreps, self.correlation[0], self.num_elements, use_sc=True)
        sizing = e3.Linear(hidden_irreps, output_irreps)
        return _MaceConv(inter, prod, sizing, output_irreps.count("0e"))

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
        ds = getattr(data, "dataset_name", None)
        outputs = self.multihead_decoders[0](attrs, batch, num_graphs, ds)
        for conv, readout in zip(self.graph_convs, self.multihead_decoders[1:]):
            inv, equiv = conv(inv, equiv, attrs, edge_attrs, edge_feats, data.edge_index)
            out = readout(torch.cat([inv, equiv], dim=1), batch, num_graphs, ds)
            outputs = [a + b for a, b in zip(outputs, out)]
        return outputs
