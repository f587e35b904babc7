"""Oracle: the engine's TF32 tensor-core rounding applied to an fp32 oracle, so a test can measure how far the reference's
arithmetic moves from fp64 at the engine's precision.  Test infrastructure only."""
import torch
from torch import nn


def _round_tf32(t):
    """fp32 -> the nearest value with a 10-bit mantissa (TF32), kept in fp32."""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


class _RoundTF32(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _round_tf32(x)

    @staticmethod
    def backward(ctx, g):
        return _round_tf32(g)


class tf32_linears:
    """Context manager: every ``nn.Linear`` of an fp32 oracle rounds its input, its weight and the incoming gradient to TF32
    before the product, as the engine's tensor-core Linears do under precision "bf16".  The rest stays fp32."""

    def __enter__(self):
        self.orig = nn.Linear.forward
        nn.Linear.forward = lambda m, x: torch.nn.functional.linear(_RoundTF32.apply(x), _RoundTF32.apply(m.weight), m.bias)
        return self

    def __exit__(self, *exc):
        nn.Linear.forward = self.orig
        return False
