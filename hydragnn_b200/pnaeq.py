"""PNA-equivariant stack on libhgb.so.

Host-side mirror of ``hydragnn/models/PNAEqStack.py`` (class names ``PainnMessage`` / ``PainnUpdate`` /
``PNAEqStack`` and attribute names ``aggr_module``, ``F_in``, ``F_out``, ``towers``, ``pre_nns``, ``post_nns`` are
kept: the reference's equivariance test monkey-patches them, tests/test_forces_equivariant.py:48-78).

Gathers, segment sums and every Linear run in libhgb kernels.  First-order passes reduce the scalar messages into
[mean | min | max | std] in one ``ops.PnaAggregateFn`` pass and fold the five degree scalers into the post Linear
(``post_linear_scaled``), so the 20 F-wide aggregate is never built; the update block is ``ops.PainnUpdateFn``.
Higher-order passes (MLIP training) run the same math composed from the closed primitives and
``DegreeScalerAggregation``, with the Linears on the any-order MatMul.
"""
import math

import torch
from torch import nn

from . import _lib, ops
from .ops import GatherRows, SegmentSum, _p, _stream
from .stacks import Base, PainnConv, edge_geometry, run_mlp

X_AGGREGATORS = ["mean", "min", "max", "std"]
X_SCALERS = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]


def sanitize_degree(deg):
    """``PNAEqStack._sanitize_degree`` (hydragnn/models/PNAEqStack.py:75-90)."""
    deg = torch.as_tensor(deg, dtype=torch.float32)
    if deg.numel() == 0:
        return deg.new_ones((1,))
    finite = torch.isfinite(deg)
    max_finite = deg[finite].max() if finite.any() else deg.new_tensor(1.0)
    deg = torch.nan_to_num(deg, nan=1.0, neginf=1.0, posinf=float(max_finite))
    return deg.clamp_min(1.0)


class DegreeScalerAggregation(nn.Module):
    """torch_geometric 2.6.1 ``DegreeScalerAggregation(aggr, scaler, deg)`` over a CSR view."""

    def __init__(self, aggr, scaler, deg):
        super().__init__()
        self.aggr, self.scaler = list(aggr), list(scaler)
        self.deg = deg
        d = deg.to(torch.float)
        n = int(d.sum())
        bins = torch.arange(d.numel(), dtype=torch.float)
        self.register_buffer("avg_deg_lin", torch.tensor(float((bins * d).sum()) / n))
        self.register_buffer("avg_deg_log", torch.tensor(float(((bins + 1).log() * d).sum()) / n))

    def scaler_factors(self, csr):
        """[N, num_scalers] per-node factors of the degree scalers (PyG DegreeScalerAggregation.forward)."""
        deg = (csr.rowptr[1:] - csr.rowptr[:-1]).to(torch.float32).clamp(min=1)
        cols = []
        for s in self.scaler:
            if s == "identity":
                cols.append(torch.ones_like(deg))
            elif s == "amplification":
                cols.append(torch.log(deg + 1) / self.avg_deg_log)
            elif s == "attenuation":
                cols.append(self.avg_deg_log / torch.log(deg + 1))
            elif s == "linear":
                cols.append(deg / self.avg_deg_lin)
            elif s == "inverse_linear":
                cols.append(self.avg_deg_lin / deg)
            else:
                raise ValueError("unsupported scaler " + str(s))
        return torch.stack(cols, dim=1)

    def forward(self, x, csr):
        n, c = csr.n, x.shape[1]
        x = x.contiguous()
        cnt = (csr.rowptr[1:] - csr.rowptr[:-1]).to(x.dtype)
        cnt1 = cnt.clamp(min=1)[:, None]
        outs = []
        args = None
        for a in self.aggr:
            if a == "mean":
                outs.append(SegmentSum.apply(x, csr) / cnt1)
            elif a in ("min", "max"):
                if args is None:
                    amin = torch.empty(n, c, dtype=torch.int64, device=x.device)
                    amax = torch.empty_like(amin)
                    _lib.call("hgb_segment_argminmax", _p(x.detach()), _p(csr.rowptr), _p(csr.perm), n, c, _p(amin), _p(amax), _stream())
                    args = {"min": amin, "max": amax}
                idx = args[a]
                val = torch.gather(x, 0, idx.clamp(min=0))
                outs.append(torch.where(idx >= 0, val, torch.zeros_like(val)))
            elif a == "std":
                mean = SegmentSum.apply(x, csr) / cnt1
                mean2 = SegmentSum.apply(x * x, csr) / cnt1
                std = (mean2 - mean * mean).clamp(min=1e-5).sqrt()
                outs.append(std.masked_fill(std <= math.sqrt(1e-5), 0.0))
            else:
                raise ValueError("unsupported aggregator " + str(a))
        out = torch.cat(outs, dim=-1)
        f = self.scaler_factors(csr)
        return torch.cat([out if s == "identity" else out * f[:, k, None] for k, s in enumerate(self.scaler)], dim=-1)


def post_linear_scaled(post, x, agg4, aggr_module, csr):
    """``post([x | s_1 A | ... | s_k A])`` for the post Linear of a PNA layer, A = ``agg4`` [N, 4 F_in] = [mean | min | max | std]
    and s_k the per-node degree scalers of ``aggr_module`` over ``csr``.  The scalers are per-node factors, so
        post([x | s_1 A | ... | s_k A]) = x W_x^T + b + sum_k s_k (A W_k^T):
    the (4k + 1) F_in-wide input is never built."""
    fin, fout = x.shape[1], post.weight.shape[0]
    ns = len(aggr_module.scaler)
    wk = post.weight[:, fin:].reshape(fout, ns, 4 * fin).permute(1, 0, 2).reshape(ns * fout, 4 * fin)
    bk = ops.linear_act(agg4, wk, None).reshape(-1, ns, fout)                        # [N, k, F_out]
    return ops.linear_act(x, post.weight[:, :fin], post.bias) + (bk * aggr_module.scaler_factors(csr)[:, :, None]).sum(dim=1)


class PainnMessage(nn.Module):
    def __init__(self, node_size, x_aggregators, x_scalers, deg, edge_dim, num_radial):
        super().__init__()
        F = node_size
        self.node_size, self.num_radial, self.edge_dim = F, num_radial, edge_dim
        self.towers, self.F_in, self.F_out = 1, F, F
        self.aggr_module = DegreeScalerAggregation(x_aggregators, x_scalers, deg)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear((4 if edge_dim else 3) * F, F))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear((len(x_aggregators) * len(x_scalers) + 1) * F, F))])
        self.rbf_emb = nn.Sequential(nn.Linear(num_radial, F), nn.Tanh())
        if edge_dim is not None:
            self.edge_encoder = nn.Linear(edge_dim, F)
        self.rbf_lin = nn.Linear(num_radial, 3 * F, bias=False)
        self.scalar_message_mlp = nn.Sequential(nn.Linear(F, F), nn.Tanh(), nn.Linear(F, F), nn.SiLU(), nn.Linear(F, 3 * F))

    def forward(self, x, v, plan, geom, edge_attr=None, higher_order=False):
        rbf, vec = geom["rbf"], geom["unit"]
        F = self.node_size
        src, dst = plan.by_row, plan.by_col                          # src = edge_index[0], dst = edge_index[1] (:341)
        lin = ops.linear_any_order if higher_order else ops.linear_act
        # pre_nn (:352-357) on [x_src | x_dst | rbf_emb | edge_enc]: linear in the blocks -> the two node blocks are multiplied
        # per NODE (N rows instead of E) and gathered per edge afterwards
        pre = self.pre_nns[0][0]
        w0 = pre.weight
        m = GatherRows.apply(lin(x, w0[:, :F], None), src) + GatherRows.apply(lin(x, w0[:, F:2 * F], None), dst)
        m = m + lin(run_mlp(self.rbf_emb, rbf, higher_order), w0[:, 2 * F:3 * F], pre.bias)
        if edge_attr is not None:
            m = m + lin(run_mlp(nn.Sequential(self.edge_encoder), edge_attr, higher_order), w0[:, 3 * F:], None)
        f = run_mlp(self.scalar_message_mlp, m, higher_order) * run_mlp(nn.Sequential(self.rbf_lin), rbf, higher_order)
        g_v, g_e, m_s = torch.split(f, F, dim=-1)
        m_v = GatherRows.apply(v, dst) * g_v.unsqueeze(1) + g_e.unsqueeze(1) * vec.unsqueeze(-1)
        am = self.aggr_module
        if not higher_order and am.aggr == ["mean", "min", "max", "std"]:
            # fused: the four aggregators in one pass; the degree scalers are folded into post_nn (the 20F-wide tensor is never built)
            agg4 = ops.PnaAggregateFn.apply(m_s.contiguous(), src)                   # [N, 4F]
            dx = post_linear_scaled(self.post_nns[0][0], x, agg4, am, src)
        else:
            agg = am(m_s, src)                                        # :396-400
            dx = run_mlp(self.post_nns[0], torch.cat([x, agg], dim=-1), higher_order)
        dv = SegmentSum.apply(m_v.contiguous(), src)
        return x + dx, v + dv


class PainnUpdate(nn.Module):
    def __init__(self, node_size, last_layer=False):
        super().__init__()
        self.update_X = nn.Linear(node_size, node_size)
        self.update_V = nn.Linear(node_size, node_size)
        self.last_layer = last_layer
        self.update_mlp = nn.Sequential(nn.Linear(node_size * 2, node_size), nn.SiLU(),
                                        nn.Linear(node_size, node_size * (2 if last_layer else 3)))

    def forward(self, x, v, higher_order=False):
        f = v.shape[-1]
        if higher_order:
            xv = ops.linear_any_order(v, self.update_X.weight, self.update_X.bias)
            vv = ops.linear_any_order(v, self.update_V.weight, self.update_V.bias)
            a = run_mlp(self.update_mlp, torch.cat([torch.linalg.norm(vv, dim=1), x], dim=-1), True)
            inner = (xv * vv).sum(dim=1)
            if self.last_layer:
                a_xv, a_xx = torch.split(a, f, dim=-1)
                return x + a_xv * inner + a_xx, None
            a_vv, a_xv, a_xx = torch.split(a, f, dim=-1)
            return x + a_xv * inner + a_xx, v + a_vv.unsqueeze(1) * xv
        s_out, v_out = ops.PainnUpdateFn.apply(x, v, self.update_X.weight, self.update_X.bias, self.update_V.weight,
                                               self.update_V.bias, self.update_mlp[0].weight, self.update_mlp[0].bias,
                                               self.update_mlp[2].weight, self.update_mlp[2].bias, self.last_layer)
        return s_out, (None if self.last_layer else v_out)


def rbf_basis(dist, num_radial, cutoff):
    """``rbf_BasisLayer.forward`` (hydragnn/models/PNAEqStack.py:479-538); ``dist`` [E]."""
    n = torch.arange(1, num_radial + 1, device=dist.device, dtype=dist.dtype)
    d = dist.unsqueeze(-1)
    sinc = torch.sin(d * n * math.pi / cutoff) / d.clamp_min(1e-9)
    sinc = torch.where(d.abs() < 1e-9, (n * math.pi / cutoff).expand_as(sinc), sinc)
    fc = torch.where(dist < cutoff, 0.5 * (torch.cos(math.pi * dist / cutoff) + 1), torch.zeros_like(dist))
    return sinc * fc.unsqueeze(-1)


class PNAEqStack(Base):
    is_edge_model = True

    def __init__(self, deg, edge_dim, num_radial, radius, *args, **kwargs):
        self.x_aggregators, self.x_scalers = list(X_AGGREGATORS), list(X_SCALERS)
        self.deg = sanitize_degree(deg)
        self.edge_dim, self.num_radial, self.radius = edge_dim, num_radial, radius
        super().__init__(*args, **kwargs)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        hidden = output_dim if input_dim == 1 else input_dim
        assert hidden > 1, "PNAEq requires more than one hidden dimension between input_dim and output_dim."
        msg = PainnMessage(input_dim, self.x_aggregators, self.x_scalers, self.deg,
                           edge_dim if edge_dim is not None else self.edge_dim, self.num_radial)
        upd = PainnUpdate(input_dim, last_layer)
        node_embed_out = nn.Sequential(nn.Linear(input_dim, output_dim), nn.Tanh(), nn.Linear(output_dim, output_dim))
        vec_embed_out = nn.Linear(input_dim, output_dim) if not last_layer else None
        return PainnConv(msg, upd, node_embed_out, vec_embed_out)

    def _embedding(self, data, plan, higher):
        assert data.pos is not None, "PNAEq requires node positions (data.pos) to be set."
        ln, unit = edge_geometry(data.pos, data.edge_shifts, plan, 1e-9, higher)        # PNAEqStack.py:202-204
        geom = {"rbf": rbf_basis(ln.squeeze(-1), self.num_radial, self.radius), "unit": unit}
        x, eattr = data.x, (data.edge_attr if self.use_edge_attr else None)
        if self.use_global_attn:
            x, eattr = self._gps_embed(data, higher)
        v = torch.zeros(x.shape[0], 3, x.shape[1], dtype=x.dtype, device=x.device)
        return x, v, {"edge_attr": eattr, "geom": geom}

    def __str__(self):
        return "Base"       # quirk Q10: the reference class defines no __str__, so the model calls itself "Base" (Base.py:908)
