"""fp64 restatements of the fused message-passing convolutions (PNAConv, PNAPlus, CGConv, GATv2Conv, SchNet's CFConv), written
from the definitions in include/hgb.h and PyG.  The model tests (test_gpu_{pna,pnaplus,cgcnn,gat,schnet}.py) and the kernel
tests (test_gpu_conv_kernels.py) both compare against these.  Every function computes on the device of its inputs."""
import math

import torch
import torch.nn.functional as F

from oracle import schnet as so
from oracle.pnaeq import DegreeScalerAggregation as ODSA


def pna_fwd(pq, ea, mt, c, ei, n):
    """PNAConv: (agg [n, 4f], first argmin / argmax in CSR order = smallest edge id, h [e, f]), all in fp64."""
    dev = pq.device
    f = pq.shape[1] // 2
    src, dst = ei[0].to(dev), ei[1].to(dev)
    h = pq[:, :f].double()[dst] + pq[:, f:].double()[src]
    if c is not None:
        h = h + c.double()
    if ea is not None:
        h = h + ea.double() @ mt.double()
    e = h.shape[0]
    cnt = torch.bincount(dst, minlength=n).double()
    inv = (1.0 / cnt.clamp(min=1))[:, None]
    idx = dst[:, None].expand(-1, f)
    mean = torch.zeros(n, f, dtype=torch.float64, device=dev).index_add_(0, dst, h) * inv
    var = torch.zeros(n, f, dtype=torch.float64, device=dev).index_add_(0, dst, h * h) * inv - mean * mean
    sd = var.clamp(min=1e-5).sqrt()
    sd = sd.masked_fill(sd <= math.sqrt(1e-5), 0.0)
    empty = (cnt == 0)[:, None]
    mn = torch.full((n, f), math.inf, dtype=torch.float64, device=dev).scatter_reduce(0, idx, h, "amin")
    mx = torch.full((n, f), -math.inf, dtype=torch.float64, device=dev).scatter_reduce(0, idx, h, "amax")
    eid = torch.arange(e, device=dev)[:, None].expand(-1, f)
    big = torch.full((n, f), e, dtype=torch.int64, device=dev)
    amin = big.scatter_reduce(0, idx, torch.where(h == mn[dst], eid, e), "amin").masked_fill(empty, -1)
    amax = big.scatter_reduce(0, idx, torch.where(h == mx[dst], eid, e), "amin").masked_fill(empty, -1)
    agg = torch.cat([mean, mn.masked_fill(empty, 0), mx.masked_fill(empty, 0), sd], dim=1)
    return agg, amin, amax, h


def pna_bwd(g, agg, amin, amax, h, ea, mt, ei, n):
    """PNAConv backward given the forward's agg / argmin / argmax: (g_h, g_P, g_Q, g_c, g_M^T or None, g_eattr or None)."""
    dev = h.device
    f = h.shape[1]
    src, dst = ei[0].to(dev), ei[1].to(dev)
    g = g.double().to(dev)
    cnt = torch.bincount(dst, minlength=n).double().clamp(min=1)[:, None]
    mean, sd = agg[:, :f], agg[:, 3 * f:]
    e = torch.arange(h.shape[0], device=dev)[:, None]
    gh = g[:, :f][dst] / cnt[dst] + (amin.long()[dst] == e) * g[:, f:2 * f][dst] + (amax.long()[dst] == e) * g[:, 2 * f:3 * f][dst]
    safe = torch.where(sd > 0, sd, torch.ones_like(sd))
    gh = gh + torch.where(sd[dst] > 0, g[:, 3 * f:][dst] / (cnt[dst] * safe[dst]) * (h - mean[dst]), torch.zeros_like(h))
    gp = torch.zeros(n, f, dtype=torch.float64, device=dev).index_add_(0, dst, gh)
    gq = torch.zeros(n, f, dtype=torch.float64, device=dev).index_add_(0, src, gh)
    gmt = ea.double().t() @ gh if ea is not None else None
    gea = gh @ mt.double().t() if ea is not None else None
    return gh, gp, gq, gh.sum(0), gmt, gea


def pnaplus_basis(dist, radius, expo, freq):
    """(x, rbf [e, r]) of the Bessel basis with the polynomial envelope: rbf = 0 for x = dist / radius >= 1."""
    x = (dist / radius)[:, None]
    p = expo + 1
    a, b, c = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    env = (1 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)) * (x < 1).to(x.dtype)
    return x, env * torch.sin(freq * x)


def pnaplus_messages(t, ei, radius, expo):
    """PNAPlus message m_e [e, f] from the tensors of t (pq, dist, eattr, freq, wr, br, wl, mr, mat, cvec)."""
    dev = t["pq"].device
    src, dst = ei[0].to(dev), ei[1].to(dev)
    f = t["pq"].shape[1] // 2
    _, rbf = pnaplus_basis(t["dist"], radius, expo, t["freq"])
    u = torch.relu(rbf @ t["wr"].t() + t["br"])
    h = t["pq"][dst, :f] + t["pq"][src, f:] + u @ t["mr"].t() + t["cvec"]
    if t["eattr"] is not None:
        h = h + t["eattr"] @ t["mat"]
    if t.get("hz") is not None:                                # a zero leaf: its gradient is dL/dh per edge
        h = h + t["hz"]
    return h * (rbf @ t["wl"].t())


def pnaplus_agg(t, ei, n, radius, expo):
    """PNAPlus: agg [n, 4f] = [mean | min | max | std] of m_e in the dtype of t."""
    return ODSA(["mean", "min", "max", "std"], ["identity"], torch.tensor([1.0]))(pnaplus_messages(t, ei, radius, expo),
                                                                                    ei[1].to(t["pq"].device), n)


def cgconv(t, ei, g_out):
    """CGConv, fp64 on the CPU: out = x + sum at the targets of sigmoid(f) softplus(s), and the gradients of <out, g_out>."""
    src, dst = ei[0].cpu(), ei[1].cpu()
    leaves = {k: (v.detach().cpu().double().requires_grad_(True) if v is not None else None) for k, v in t.items()}
    pq, ea, mt, cvec, x = (leaves[k] for k in ("pq", "ea", "mt", "cvec", "x"))
    f = x.shape[1]
    h = pq[dst, :2 * f] + pq[src, 2 * f:] + cvec
    if ea is not None:
        h = h + ea @ mt
    if leaves.get("hz") is not None:                           # a zero leaf: its gradient is g_h = [dL/df | dL/ds] per edge
        h = h + leaves["hz"]
    m = torch.sigmoid(h[:, :f]) * F.softplus(h[:, f:])
    out = x + torch.zeros_like(x).index_add(0, dst, m)
    names = [k for k in ("pq", "ea", "mt", "cvec", "hz") if leaves.get(k) is not None]
    grads = torch.autograd.grad(out, [leaves[k] for k in names], g_out.cpu().double())
    return out.detach(), dict(zip(names, grads))


def gat(t, ei, heads, c, concat, g_out, slope, keep=None, p=0.0):
    """GATv2Conv after its Linears, fp64 on the CPU (remove / add self-loops with the mean attribute, softmax with the max
    detached), and the gradients of <out, g_out> by autograd."""
    src, dst = ei[0].cpu(), ei[1].cpu()
    leaves = {k: (v.detach().cpu().double().requires_grad_(True) if v is not None else None) for k, v in t.items()}
    xlr, ea, mt, att, bias = (leaves[k] for k in ("xlr", "ea", "mt", "att", "bias"))
    n, hc = xlr.shape[0], heads * c
    xl, xr = xlr[:, :hc], xlr[:, hc:]
    e = src.numel()
    other = src != dst
    eid = torch.cat([torch.arange(e)[other], e + torch.arange(n)])
    s_, d_ = torch.cat([src[other], torch.arange(n)]), torch.cat([dst[other], torch.arange(n)])
    z = xr[d_] + xl[s_]
    if ea is not None:
        a = ea[other]
        cnt = torch.zeros(n, dtype=a.dtype).index_add_(0, dst[other], torch.ones(a.shape[0], dtype=a.dtype)).clamp(min=1)
        a = torch.cat([a, torch.zeros(n, a.shape[1], dtype=a.dtype).index_add(0, dst[other], a) / cnt[:, None]])
        z = z + a @ mt
    s = (F.leaky_relu(z, slope).view(-1, heads, c) * att.view(1, heads, c)).sum(-1)
    m = torch.full((n, heads), float("-inf"), dtype=s.dtype).scatter_reduce(0, d_[:, None].expand_as(s), s.detach(), "amax")
    ex = (s - m[d_]).exp()
    al = ex / (torch.zeros(n, heads, dtype=s.dtype).index_add(0, d_, ex) + 1e-16)[d_]
    if keep is not None:
        al = al * keep.cpu().double()[eid] / (1.0 - p)
    out = torch.zeros(n, heads, c, dtype=s.dtype).index_add(0, d_, al[:, :, None] * xl[s_].view(-1, heads, c))
    out = (out.reshape(n, hc) if concat else out.mean(1)) + bias
    names = [k for k in ("xlr", "ea", "mt", "att", "bias") if leaves[k] is not None]
    grads = torch.autograd.grad(out, [leaves[k] for k in names], g_out.cpu().double())
    return out.detach(), dict(zip(names, grads))


def cfconv(ei, pos, t, offset, coeff, cutoff=3.0, g_we=True):
    """SchNet's CFConv in fp64 on the CPU through oracle.schnet.cfconv with identity Linears: (out = sum_e xl[j] W_e, W_e, the
    gradients of <out, g_out> + <W_e, g_we> by autograd, pos included).  With g_we False the W_e term is left out."""
    leaves = {k: (v.clone().requires_grad_(True) if v is not None and k not in ("g_out", "g_we") else v) for k, v in t.items()}
    p = pos.clone().requires_grad_(True)
    a = leaves["a1t"]
    ea = leaves["r"]
    w1 = a.t()
    eye = torch.eye(a.shape[1], dtype=torch.float64)
    out, w = so.cfconv(leaves["xl"], p, ei, eye, w1, leaves["b1"], leaves["w2"], leaves["b2"], eye, torch.zeros_like(leaves["b1"]),
                       offset, coeff, cutoff, edge_attr=ea)
    obj = (out * t["g_out"]).sum() + ((w * t["g_we"]).sum() if g_we else 0.0)
    names = ["xl", "a1t", "b1", "w2", "b2"] + (["r"] if ea is not None else [])
    grads = torch.autograd.grad(obj, [leaves[k] for k in names] + [p])
    return out, w, dict(zip(names + ["pos"], grads))


def cfconv_edges(t, dist, row, col, n, mu, coeff, cutoff):
    """CFConv per edge from the edge lengths, fp64 in the dtype of t: (out [n, nf] = sum_e xl[row] W_e at col, W_e [e, nf]).
    t: xl, r (or None), a1t, b1, w2, b2; mu [g]."""
    a = torch.exp(coeff * (dist[:, None] - mu) ** 2)
    if t["r"] is not None:
        a = torch.cat([a, t["r"]], 1)
    s = F.softplus(a @ t["a1t"] + t["b1"]) - math.log(2.0)
    w = (s @ t["w2"].t() + t["b2"]) * (0.5 * (torch.cos(dist * math.pi / cutoff) + 1.0))[:, None]
    out = torch.zeros(n, w.shape[1], dtype=w.dtype).index_add(0, col, t["xl"][row] * w)
    return out, w
