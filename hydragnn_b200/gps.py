"""GPS layer on libhgb.so: local MPNN + dense multi-head self-attention + MLP, three BatchNorms.

Host-side mirror of ``GPSConv`` (hydragnn/globalAtt/gps.py:32-152), ``attn_type == "multihead"``.  Parameter
names are the reference's (``conv.*``, ``attn.in_proj_weight`` ..., ``mlp.0/3``, ``norm{1,2,3}.module.*``).
The attention itself is ``hgb_mha_{fwd,bwd}`` (flash-style, one sequence = the whole mini-batch: quirk Q1);
in/out projections and the MLP are the engine's Linear kernels; BatchNorm stays ATen (SURVEY 2.1: not named by
the north star); dropout is ATen RNG.
"""
import math

import torch
from torch import nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _lib, ops
from .ops import _chk, _p, _stream
from .stacks import run_mlp


class PyGBatchNorm(nn.Module):
    """torch_geometric.nn.BatchNorm: a module holding ``self.module = BatchNorm1d(channels)`` [3P-memory]."""

    def __init__(self, channels):
        super().__init__()
        self.module = nn.BatchNorm1d(channels)

    def forward(self, x):
        return self.module(x)


class MhaFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, heads):
        qkv = _chk(qkv)
        n, f3 = qkv.shape
        f = f3 // 3
        out = torch.empty(n, f, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(n, heads, dtype=qkv.dtype, device=qkv.device)
        # head_dim 8: tensor-core kernels (3xTF32 = fp32-level accuracy in fp32 mode, plain TF32 under precision="bf16").  They
        # move rows as float4, so a view that does not start on a 16-byte boundary takes the SIMT kernels (scalar accesses).
        ctx.tc = bool(_lib.query("hgb_mha_tc_supported", f, heads)) and qkv.data_ptr() % 16 == 0
        ctx.exact = 0 if ops._TC["enabled"] else 1
        if n == 0:
            pass
        elif ctx.tc:
            _lib.call("hgb_mha_tc_fwd", _p(qkv), n, f, heads, ctx.exact, _p(out), _p(lse), _stream())
        else:
            _lib.call("hgb_mha_fwd", _p(qkv), n, f, heads, _p(out), _p(lse), _stream())
        ctx.save_for_backward(qkv, out, lse)
        ctx.heads = heads
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        qkv, out, lse = ctx.saved_tensors
        n, f = out.shape
        gqkv = torch.empty_like(qkv)
        gout = _chk(gout)
        if n == 0:
            pass
        elif ctx.tc and gout.data_ptr() % 16 == 0:
            ws = torch.empty(n * ctx.heads, dtype=qkv.dtype, device=qkv.device)
            _lib.call("hgb_mha_tc_bwd", _p(qkv), _p(out), _p(lse), _p(gout), n, f, ctx.heads, ctx.exact, _p(ws), _p(gqkv), _stream())
        else:       # either backward takes either forward's out and lse (include/hgb.h)
            _lib.call("hgb_mha_bwd", _p(qkv), _p(out), _p(lse), _p(gout), n, f, ctx.heads, _p(gqkv), _stream())
        return gqkv, None


def mha_any_order(qkv, heads):
    """Same attention from the closed MatMul primitive + ATen softmax (used when the graph is differentiated twice)."""
    n, f3 = qkv.shape
    f = f3 // 3
    d = f // heads
    outs = []
    for h in range(heads):
        q = qkv[:, h * d:(h + 1) * d].contiguous()
        k = qkv[:, f + h * d:f + (h + 1) * d].contiguous()
        v = qkv[:, 2 * f + h * d:2 * f + (h + 1) * d].contiguous()
        p = torch.softmax(ops.MatMul.apply(q, k, False, True) / math.sqrt(d), dim=-1)
        outs.append(ops.MatMul.apply(p, v, False, False))
    return torch.cat(outs, dim=1)


class GPSConv(nn.Module):
    def __init__(self, channels, conv, heads=1, dropout=0.0, attn_type="multihead"):
        super().__init__()
        if attn_type != "multihead":
            raise ValueError(f"{attn_type} is not supported")
        self.channels, self.conv, self.heads, self.dropout, self.attn_type = channels, conv, heads, dropout, attn_type
        self.attn = nn.MultiheadAttention(channels, heads, batch_first=True)       # parameter container only
        self.mlp = nn.Sequential(nn.Linear(channels, channels * 2), nn.ReLU(), nn.Dropout(dropout),
                                 nn.Linear(channels * 2, channels), nn.Dropout(dropout))
        self.norm1, self.norm2, self.norm3 = PyGBatchNorm(channels), PyGBatchNorm(channels), PyGBatchNorm(channels)

    def forward(self, inv_node_feat, equiv_node_feat, plan, higher_order=False, **kwargs):
        x = inv_node_feat
        h, equiv = self.conv(inv_node_feat=x, equiv_node_feat=equiv_node_feat, plan=plan, higher_order=higher_order, **kwargs)
        h = F.dropout(h, p=self.dropout, training=self.training) + x
        h1 = self.norm1(h)
        if higher_order:
            qkv = ops.linear_any_order(x, self.attn.in_proj_weight, self.attn.in_proj_bias)
            a = mha_any_order(qkv, self.heads)
            a = ops.linear_any_order(a, self.attn.out_proj.weight, self.attn.out_proj.bias)
        else:
            qkv = ops.linear_act(x, self.attn.in_proj_weight, self.attn.in_proj_bias)
            a = MhaFn.apply(qkv, self.heads)
            a = ops.linear_act(a, self.attn.out_proj.weight, self.attn.out_proj.bias)
        a = F.dropout(a, p=self.dropout, training=self.training) + x
        h2 = self.norm2(a)
        out = h1 + h2
        out = out + run_mlp(self.mlp, out, higher_order)
        return self.norm3(out), equiv
