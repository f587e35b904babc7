"""GPU tests of the weight-gradient pipeline's ring sizing (hgb_tc_wgrad): the TMA ring of raw slabs, the ring of K-major operand
buffers between the seven transposer warps and the MMA warpgroups, and the operand rows that are written once at start-up.

The host code picks 3 K-major buffers where they fit beside two raw stages, else 2, else 1, and gives the rest of shared memory to
the raw ring.  With the 128 + k_out + 16 operand rows of a buffer (twice that in the exact mode) and (n_out / 32 + Q) raw slabs of
4 KB per stage:
  tf32:   3 buffers (2..19 stages), except Q = 7 at n_out = 128: 2 buffers
  exact:  3 buffers for Q <= 2 and for Q = 3 at n_out <= 64, 2 buffers for Q = 3 at n_out >= 96 and Q = 4, 5, 1 buffer for
          Q = 6 at n_out >= 64 and Q = 7 (2..11 stages)
The existing width tests run each instantiation at <= 2 chunks per CTA; these run every ring around many times, and the tails where
a CTA has fewer chunks than the rings are deep.  Each case is held to the bound of tests/test_gpu_tc.py (exact: within 4x of the SIMT
fp32 GEMM; tf32: 2e-3) and must give the same bits twice."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from hydragnn_b200 import ops  # noqa: E402
from test_gpu_tc import DEV, TOL, mode_ctx, rel, traced, wgrad_ok  # noqa: E402

SMS = 132


def m_for(chunks_per_cta, ctas, tail=0):
    """rows giving `ctas` CTAs of `chunks_per_cta` 32-row chunks, the last CTA short by `tail` chunks and its last chunk 7 rows long"""
    return 32 * (chunks_per_cta * ctas - tail - 1) + 7


# (mode, n_out, k_out, m): chunks per CTA from 1 to 24, K-major rings of 3, 2 and 1 buffers, row blocks of 128, 96 (warpgroup 1 has
# 32 zero rows) and 128 + 32 (n_out = 160: the second CTA row has 32 rows, warpgroup 1 idles)
CASES = [
    ("tf32", 64, 64, m_for(1, 100)),            # one chunk per CTA: every ring deeper than the work
    ("tf32", 64, 64, m_for(2, SMS, tail=1)),    # two chunks, the last CTA one
    ("tf32", 128, 64, m_for(24, SMS, tail=5)),  # 3 buffers, 6 stages, both rings around several times
    ("tf32", 96, 32, m_for(13, SMS)),
    ("tf32", 160, 96, m_for(7, SMS // 2, tail=4)),
    ("tf32", 128, 224, m_for(5, SMS, tail=2)),  # 2 buffers, 3 stages
    ("exact", 64, 64, m_for(3, SMS, tail=2)),   # 3 buffers, 4 stages: fewer chunks than stages
    ("exact", 128, 96, m_for(17, SMS, tail=9)),   # 2 buffers, 3 stages; folds after chunks 8 and 16, the last CTA has 8 chunks
    ("exact", 128, 160, m_for(9, SMS)),         # 2 buffers, 2 stages
    ("exact", 96, 128, m_for(2, SMS)),          # 2 buffers, 3 stages: fewer chunks than either ring
    ("exact", 128, 224, m_for(20, SMS, tail=3)),  # 1 buffer, 3 stages
    ("exact", 64, 192, m_for(1, 40)),           # 1 buffer, 4 stages, one chunk per CTA
]


@pytest.mark.parametrize("mode,n,k,m", CASES)
def test_tc_wgrad_ring_depths_and_tails(mode, n, k, m):
    g = torch.Generator().manual_seed(m + n + k)
    dz, x = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g)
    dzd, xd = dz.to(DEV), x.to(DEV)
    with mode_ctx(mode):
        (dw, db), calls = traced(lambda: ops.raw_tc_wgrad(dzd, xd, want_bias=True), "hgb_tc_wgrad")
        dw2, db2 = ops.raw_tc_wgrad(dzd, xd, want_bias=True)
    assert [(c[0]["exact"], c[0]["n_out"], c[0]["k_out"], c[1]) for c in calls] == [(int(mode == "exact"), n, k, 2)]
    ref_w = dz.double().t() @ x.double()
    ok, e = wgrad_ok(dw, ref_w, rel(ops.raw_gemm(dzd, xd, True, False), ref_w), mode)
    assert ok, e
    assert rel(db, dz.double().sum(0)) < (5e-6 if mode == "exact" else TOL[mode])
    assert torch.equal(dw, dw2) and torch.equal(db, db2)
