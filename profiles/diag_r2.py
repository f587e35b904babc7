"""Round-2 diagnostics (needs a GPU): (1) which EGNN parameter gradients differ between the fused path, the composed path
and the fp64 oracle; (2) PNAEq+GPS gradient agreement with the tensor-core attention on / off; (3) attention kernel timings."""
import os, sys, copy
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hydragnn_b200 as hb
from hydragnn_b200 import ops, gps
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples
import oracle
from oracle.workloads import add_edges_cpu, arch_for

DEV = "cuda"


def egnn():
    name, g = "md17_egnn", 24
    cpu = add_edges_cpu(make_samples(name, g), name)
    kw = ARCH[name]
    om = oracle.base.create_model(**kw).train()
    em = hb.create_model(**kw).train()
    em.model.load_state_dict(om.model.state_dict())
    o64 = copy.deepcopy(om).double()
    c64 = cpu.clone(); c64._num_graphs = g
    for k in ("x", "pos", "energy", "forces", "edge_shifts"):
        c64[k] = c64[k].double()
    c64.pos.requires_grad_(True)
    l64, _ = o64.energy_force_loss(o64(c64), c64)
    l64.backward()
    cpu.pos.requires_grad_(True)
    l32, _ = om.energy_force_loss(om(cpu), cpu)
    l32.backward()
    res = {}
    for fused in (True, False):
        ops.FUSED_EGNN = fused
        for p in em.parameters():
            p.grad = None
        d = cpu.clone().to(DEV); d._num_graphs = g
        d.pos = d.pos.detach().requires_grad_(True)
        le, _ = em.energy_force_loss(em(d), d)
        le.backward()
        res[fused] = {n: p.grad.double().cpu() for n, p in em.model.named_parameters()}
    ops.FUSED_EGNN = True
    ref = {n: p.grad for n, p in o64.model.named_parameters()}
    o32 = {n: p.grad.double() for n, p in om.model.named_parameters()}
    print("loss fp64 %.8f  oracle32 %.8f" % (float(l64), float(l32)))
    for n in ref:
        sc = ref[n].abs().max()
        e_f = (res[True][n] - ref[n]).abs().max() / sc
        e_c = (res[False][n] - ref[n]).abs().max() / sc
        e_o = (o32[n] - ref[n]).abs().max() / sc
        print("%-48s max|diff|/max|ref|: fused %.2e  composed %.2e  oracle-fp32 %.2e" % (n, e_f, e_c, e_o))


def wd():
    """which loss term / which block of edge_mlp.0.weight carries the fused path's excess error"""
    name, g = "md17_egnn", 24
    cpu = add_edges_cpu(make_samples(name, g), name)
    kw = ARCH[name]
    om = oracle.base.create_model(**kw).train()
    em = hb.create_model(**kw).train()
    em.model.load_state_dict(om.model.state_dict())
    o64 = copy.deepcopy(om).double()

    def losses(m, d, which):
        pred = m(d)
        if which == "energy":
            return (pred[0] ** 2).sum()
        e = pred[0].sum()
        f = torch.autograd.grad(e, d.pos, create_graph=True)[0]
        return (f ** 2).sum() if which == "force" else (f ** 2).sum() + (pred[0] ** 2).sum()

    for which in ("energy", "force"):
        c64 = cpu.clone(); c64._num_graphs = g
        for k in ("x", "pos", "energy", "forces", "edge_shifts"):
            c64[k] = c64[k].double()
        c64.pos.requires_grad_(True)
        for p in o64.parameters():
            p.grad = None
        losses(o64.model, c64, which).backward()
        ref = {n: p.grad.clone() for n, p in o64.model.named_parameters() if p.grad is not None}
        for fused in (True, False):
            ops.FUSED_EGNN = fused
            for p in em.parameters():
                p.grad = None
            d = cpu.clone().to(DEV); d._num_graphs = g
            d.pos = d.pos.detach().requires_grad_(True)
            em.model.force_higher_order = True
            losses(em.model, d, which).backward()
            for n, p in em.model.named_parameters():
                if n.endswith("edge_mlp.0.weight"):
                    gr, rf = p.grad.double().cpu(), ref[n]
                    fin2 = gr.shape[1] - 1
                    e_ab = (gr[:, :fin2] - rf[:, :fin2]).abs().max() / rf[:, :fin2].abs().max()
                    e_wd = (gr[:, fin2] - rf[:, fin2]).abs().max() / rf[:, fin2].abs().max()
                    print("%-7s fused=%-5s %-44s W0a|W0b block %.2e   w_d column %.2e (max|ref| %.3e)" % (which, fused, n, e_ab, e_wd, rf[:, fin2].abs().max()))
    ops.FUSED_EGNN = True


def pna():
    name, g = "gfm_pnaeq", 12
    cpu = add_edges_cpu(make_samples(name, g), name)
    kw = arch_for(name, cpu)
    om = oracle.base.create_model(**kw).eval()
    o64 = copy.deepcopy(om).double()
    c64 = cpu.clone(); c64._num_graphs = g
    for k in ("x", "pos", "y", "pe", "rel_pe", "edge_shifts", "energy", "forces"):
        if c64[k] is not None:
            c64[k] = c64[k].double()
    hi = hb.get_head_indices(om, cpu)
    l64, _ = o64.loss(o64(c64), c64.y, hi); l64.backward()
    l32, _ = om.loss(om(cpu), cpu.y, hi); l32.backward()
    ref = dict(o64.named_parameters())

    def rel(grads):
        num = sum(float((grads[n] - ref[n].grad).pow(2).sum()) for n in grads)
        den = sum(float(ref[n].grad.pow(2).sum()) for n in grads)
        return (num / den) ** 0.5
    print("pna oracle-fp32 vs fp64: %.3e" % rel({n: p.grad.double() for n, p in om.named_parameters()}))
    for tc in (True, False):
        gps.TC_ATTENTION = tc
        em = hb.create_model(**kw).eval()
        em.load_state_dict(om.state_dict())
        d = cpu.clone().to(DEV); d._num_graphs = g
        le, _ = em.loss(em(d), d.y, [h.to(DEV) for h in hi]); le.backward()
        print("pna engine (tc attention %s) vs fp64: %.3e   loss %.8f vs %.8f" % (tc, rel({n: p.grad.double().cpu() for n, p in em.named_parameters()}), float(le), float(l64)))
    gps.TC_ATTENTION = True


def attn():
    n, f, heads = 9920, 64, 8
    qkv = torch.randn(n, 3 * f, device=DEV, requires_grad=True)
    go = torch.randn(n, f, device=DEV)
    for tc, mode in ((True, "exact"), (True, "tf32"), (False, "simt")):
        gps.TC_ATTENTION = tc
        with ops.tensor_cores(mode == "tf32"):
            for it in range(3):
                out = gps.MhaFn.apply(qkv, heads)
                out.backward(go)
            torch.cuda.synchronize()
            t0, t1, t2 = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            t0.record()
            for it in range(5):
                out = gps.MhaFn.apply(qkv, heads)
            t1.record()
            for it in range(5):
                out = gps.MhaFn.apply(qkv, heads)
                out.backward(go)
            t2.record()
            torch.cuda.synchronize()
        fwd = t0.elapsed_time(t1) / 5
        print("attention n=%d %s: fwd %.3f ms, fwd+bwd %.3f ms" % (n, mode, fwd, t1.elapsed_time(t2) / 5))
    gps.TC_ATTENTION = True


if __name__ == "__main__":
    for fn in sys.argv[1:] or ["egnn", "pna", "attn"]:
        globals()[fn]()
