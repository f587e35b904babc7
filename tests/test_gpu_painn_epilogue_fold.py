"""The encoder's ReLU after a PaiNN layer folded into the passes next to it (stacks.ReluEmbed): layer 0's node_embed_out runs with
the ReLU in its tensor-core epilogue and layer 1's scalar-message MLP adds the two gradients of s and applies the ReLU's mask in
its data-gradient epilogue (ops.ReluMlp2PhiFn); after the last layer the mean pool's backward applies the mask while it
broadcasts (ops.ReluMlp2MeanPoolFn).  Every fold is a selection or a two-term sum, so the model keeps the bits of the unfused
loop (Mlp2Fn, torch.relu, autograd's add, threshold_backward), forward and backward, and trains along the same trajectory."""
import pytest
import torch
from torch import nn

import hydragnn_b200 as hb
from hydragnn_b200 import _lib, ops, stacks
from hydragnn_b200.synthetic import ARCH, make_samples

DEV = "cuda"
gpu = pytest.mark.gpu


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


def unfused(monkeypatch):
    monkeypatch.setattr(stacks.Base, "_relu_embed_plan", lambda self, higher: [False] * len(self.graph_convs))


def fold_nodes(t):
    """names of the fold Functions in the autograd graph behind t"""
    seen, names, todo = set(), set(), [t.grad_fn]
    while todo:
        fn = todo.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.add(type(fn).__name__)
        todo.extend(f for f, _ in fn.next_functions)
    return {n for n in names if n.startswith("ReluMlp2")}


def c2(graphs, precision, **arch):
    torch.manual_seed(0)
    m = hb.set_precision(hb.create_model(**dict(ARCH["qm9_painn"], **arch)), precision).to(DEV)
    b = make_samples("qm9_painn", graphs).to(DEV)
    b._num_graphs = graphs
    return m, hb.get_radius_graph(7.0, 5)(b)


def loss_and_grads(m, b, higher=False):
    m.zero_grad(set_to_none=True)
    m.force_higher_order = higher
    loss, _ = m.loss(m(b), b.y, [torch.arange(b._num_graphs, device=DEV)])
    nodes = fold_nodes(loss)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()], nodes


# ---- whole model ------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_c2_model_same_bits_as_unfused(precision, monkeypatch):
    """TF32 (bf16 config): both folds run; fp32: neither does.  Loss and every parameter gradient keep the unfused bits."""
    m, b = c2(512, precision)
    loss_f, grads_f, nodes = loss_and_grads(m, b)
    assert nodes == ({"ReluMlp2PhiFnBackward", "ReluMlp2MeanPoolFnBackward"} if precision == "bf16" else set())
    unfused(monkeypatch)
    loss_u, grads_u, nodes = loss_and_grads(m, b)
    assert not nodes
    assert same_bits(loss_f, loss_u), (float(loss_f), float(loss_u))
    for (name, _), gf, gu in zip(m.named_parameters(), grads_f, grads_u):
        assert same_bits(gf, gu), "%s: rel-L2 %.3g" % (name, rel(gf, gu))


@gpu
def test_c2_twenty_adamw_steps_same_parameters(monkeypatch):
    runs = []
    for fold in (True, False):
        if not fold:
            unfused(monkeypatch)
        m, b = c2(512, "bf16")
        model = hb.get_distributed_model(m)
        opt = hb.FlatAdamW(model, lr=1e-3)
        losses = [hb.train_step(model, opt, b)[0].detach().clone() for _ in range(20)]
        torch.cuda.synchronize()
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    for i, (a, c) in enumerate(zip(runs[0][0], runs[1][0])):
        assert same_bits(a, c), "step %d: loss %r vs %r" % (i, float(a), float(c))
    for (name, _), a, c in zip(m.named_parameters(), runs[0][1], runs[1][1]):
        assert same_bits(a, c), "%s differs after 20 steps: rel-L2 %.3g" % (name, rel(a, c))


@gpu
def test_c2_step_runs_no_aten_kernel_over_n64():
    """one eager C2 training step: no ATen kernel is launched by an op with an operand of N * 64 elements or more (the ReLU
    forward and backward and the gradient sum of the unfused loop all were)"""
    from torch.profiler import ProfilerActivity, profile
    m, b = c2(1024, "bf16")
    n = b.x.shape[0]
    model = hb.get_distributed_model(m)
    opt = hb.FlatAdamW(model, lr=1e-3)
    hb.train_step(model, opt, b)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        hb.train_step(model, opt, b)
        torch.cuda.synchronize()
    is_aten = lambda k: "at::" in k or "at_cuda" in k or "cutlass" in k or "cublas" in k.lower()  # noqa: E731
    big = []
    for e in prof.events():
        if not any(is_aten(k.name) for k in (getattr(e, "kernels", None) or [])):
            continue
        sizes = [torch.Size(s).numel() for s in (e.input_shapes or []) if isinstance(s, (list, tuple)) and all(isinstance(x, int) for x in s)]
        if max(sizes, default=0) >= n * 64:
            big.append((e.name, e.input_shapes))
    assert not big, big


# ---- the kernels the folds use, against the ATen ops they replace -------------------------------------------------------------
def special_rows(t, g):
    """y-like tensor with +0, -0.0, NaN and negative entries at random places"""
    t = t.clone()
    k = t.numel()
    idx = torch.randperm(k, generator=g)[: max(4, k // 5)].to(t.device)
    vals = torch.tensor([0.0, -0.0, float("nan"), -1.5], device=t.device)
    t.view(-1)[idx] = vals[torch.arange(idx.numel(), device=t.device) % 4]
    return t


@gpu
@pytest.mark.parametrize("mode", ["mean", "add"])
@pytest.mark.parametrize("c", [64, 40])
def test_masked_pool_backward_equals_pool_backward_then_threshold_backward(mode, c):
    g = torch.Generator().manual_seed(c)
    sizes = torch.tensor([0, 1, 9, 0, 5, 1, 30, 0, 2, 1, 70, 9, 9, 0, 1] * 7)
    rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), sizes.cumsum(0)]).int().to(DEV)
    n, ng = int(sizes.sum()), sizes.numel()
    y = torch.relu(special_rows(torch.randn(n, c, generator=g), g)).to(DEV)
    y = special_rows(y, g)                                   # -0.0 and NaN rows survive only if set after the ReLU
    gout = torch.randn(ng, c, generator=g).to(DEV)
    gout[0, :4] = torch.tensor([float("inf"), float("-inf"), float("nan"), -0.0])
    code = ops.POOL_CODES[mode]
    gx = torch.empty(n, c, device=DEV)
    _lib.call("hgb_pool_bwd", ops._p(gout), ops._p(rowptr), None, None, n, ng, c, code, ops._p(gx), ops._stream())
    ref = torch.ops.aten.threshold_backward(gx, y, 0.0)
    got = torch.full((n, c), 7.0, device=DEV)
    _lib.call("hgb_pool_bwd", ops._p(gout), ops._p(rowptr), None, ops._p(y), n, ng, c, code, ops._p(got), ops._stream())
    torch.cuda.synchronize()
    assert same_bits(got, ref)


@gpu
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("n", [128, 129, 16897, 147456])
def test_relu_select_dgrad_equals_dgrad_add_threshold_backward(n, tc):
    """the data gradient of phi's first Linear with g_s added and the ReLU's select in the epilogue, against dgrad, add and
    threshold_backward; and the ReLU forward epilogue against torch.relu of the plain Linear"""
    g = torch.Generator().manual_seed(n)
    f = 64
    dz = torch.randn(n, f, generator=g).to(DEV)
    w = (torch.randn(f, f, generator=g) * 0.2).to(DEV)
    g_s = special_rows(torch.randn(n, f, generator=g), g).to(DEV)
    s = special_rows(torch.relu(torch.randn(n, f, generator=g)), g).to(DEV)
    x = torch.randn(n, f, generator=g)
    x[n // 3] = float("nan")
    x[n // 2] = 0.0
    x, b = x.to(DEV), torch.randn(f, generator=g).to(DEV)
    b[:4] = -0.0
    with ops.tensor_cores(tc):
        dx = ops.raw_tc_linear(dz, w, True, None, f, f)[0]
        ref = torch.ops.aten.threshold_backward(dx + g_s, s, 0.0)
        got = ops.raw_tc_linear(dz, w, True, None, f, f, addend=g_s, gsrc=s, gact=ops.RELU_SELECT)[0]
        y_ref = torch.relu(ops.raw_tc_linear(x, w, False, b, f, f)[0])
        y = ops.raw_tc_linear(x, w, False, b, f, f, code=ops.ACT_CODES["relu"])[0]
        act_bwd = ops.raw_act_bwd(dx + g_s, s, None, ops.RELU_SELECT)
    torch.cuda.synchronize()
    assert same_bits(got, ref)
    assert same_bits(act_bwd, ref)
    assert same_bits(y, y_ref)


# ---- where the folds are taken --------------------------------------------------------------------------------------------------
def plan(kw, tc, higher=False):
    m = hb.create_model(**kw)
    with ops.tensor_cores(tc):
        return m._relu_embed_plan(higher)


def test_fold_plan_c2():
    kw = dict(ARCH["qm9_painn"])
    assert plan(kw, True) == [True, True]
    assert plan(dict(kw, num_conv_layers=3), True) == [True, True, True]
    assert plan(kw, False) == [False, False]                                      # fp32 mode
    assert plan(kw, True, higher=True) == [False, False]                          # any-order path
    assert plan(dict(kw, activation_function="selu"), True) == [False, False]
    assert plan(dict(kw, graph_pooling="max"), True) == [True, False]              # the pool fold is a mean pool's
    node_head = dict(kw, output_dim=[1, 1], output_type=["graph", "node"], task_weights=[1.0, 1.0],
                     output_heads=dict(kw["output_heads"], node={"num_headlayers": 2, "dim_headlayers": [8, 8], "type": "mlp"}))
    assert plan(node_head, True) == [True, False]                                  # a node head reads the [N, F] features


def test_fold_plan_gps_and_pnaeq():
    gps = dict(ARCH["qm9_painn"], global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4, pe_dim=4)
    assert plan(gps, True) == [False, False]
    pnaeq = {k: v for k, v in ARCH["gfm_pnaeq"].items() if not k.startswith(("global_attn", "pe_dim"))}
    pnaeq.update(output_dim=[1], output_type=["graph"], task_weights=[1.0], pna_deg=[0, 4, 8, 4])
    pnaeq["output_heads"] = {"graph": pnaeq["output_heads"]["graph"]}
    assert plan(pnaeq, True) == [False] * pnaeq["num_conv_layers"]


@gpu
@pytest.mark.parametrize("hidden,higher", [(48, False), (64, True)])
def test_width_48_and_any_order_take_the_unfused_path(hidden, higher, monkeypatch):
    """F = 48 is off the tensor-core shapes: the ReluEmbed records are materialised with the unfused calls; the any-order path
    never defers"""
    m, b = c2(256, "bf16", hidden_dim=hidden)
    if higher:
        b.pos.requires_grad_(False)
    loss_f, grads_f, nodes = loss_and_grads(m, b, higher)
    assert not nodes
    unfused(monkeypatch)
    loss_u, grads_u, _ = loss_and_grads(m, b, higher)
    assert same_bits(loss_f, loss_u)
    for gf, gu in zip(grads_f, grads_u):
        assert same_bits(gf, gu)
