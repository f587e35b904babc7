"""The fp64 optimizer oracle (oracle/optim.py) against torch.optim's single-tensor implementations (foreach=False) in fp64 over 20
steps with a learning rate changed between steps, for every option combination of optim_support.CASES, and against the
trajectories of the reference's select_standard_optimizer in tests/golden/optimizers.pt."""
import pytest
import torch

from optim_support import CASES, IDS, TORCH, oracle_run
from oracle import optim as oopt

STEPS = 20


def _grads(shape, steps, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(shape, generator=g, dtype=torch.float64) for _ in range(steps)]


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_oracle_equals_torch_single_tensor_fp64(name, hp):
    gen = torch.Generator().manual_seed(3)
    p0 = torch.randn(37, generator=gen, dtype=torch.float64)
    grads = _grads(37, STEPS, 4)
    lrs = [hp["lr"] * (1.0 if t < 8 else 0.3 if t < 14 else 0.1) for t in range(STEPS)]   # a scheduler between steps
    p = torch.nn.Parameter(p0.clone())
    opt = TORCH[name]([p], foreach=False, **hp)
    for t in range(STEPS):
        opt.param_groups[0]["lr"] = lrs[t]
        p.grad = grads[t].clone()
        opt.step()
    po, so = oracle_run(name, hp, p0, grads, lrs)
    torch.testing.assert_close(po, p.detach(), rtol=1e-12, atol=1e-14)
    tst = opt.state[p]
    assert set(so) == set(k for k in tst if k != "step")
    for k, v in so.items():
        torch.testing.assert_close(v, tst[k], rtol=1e-12, atol=1e-14)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/optimizers.pt")


@pytest.mark.parametrize("name", ["SGD", "Adam", "AdamW", "Adadelta", "Adagrad", "Adamax", "RMSprop"])
def test_oracle_equals_reference_trajectories(golden, name):
    rec = golden["types"][name]
    hp = {k: rec["group"][k] for k in oopt.DEFAULTS[name]}
    assert rec["class"] == name
    for i, p0 in enumerate(golden["params0"]):
        grads = [gs[i] for gs in golden["grads"]]
        for t, step in enumerate(rec["trajectory"], start=1):
            po, so = oracle_run(name, hp, p0, grads[:t])
            torch.testing.assert_close(po, step["params"][i], rtol=1e-12, atol=1e-14)
            for k, v in so.items():
                torch.testing.assert_close(v, step["state"][i][k], rtol=1e-12, atol=1e-14)
