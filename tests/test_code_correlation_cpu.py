"""code_correlation without a GPU: the fp64 oracle against the reference's codes (tests/golden/code_correlation.pt), the
cross-sum bound against the emulated arithmetics, the host-side refusals, and the ABI declarations."""
import os

import pytest
import torch

from oracle import arith_emulation as AE
from oracle import correlation_oracle as CO
from sparse_coding_b200 import _lib, metrics
from sparse_coding_b200.learned_dict import TiedSAE, UntiedSAE

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "code_correlation.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def test_oracle_reproduces_golden(golden):
    for (na, nb), want in golden["pairs"].items():
        got = CO.correlation(golden["codes"][("a", na)], golden["codes"][("b", nb)])
        for k in ("mean_a", "var_a", "mean_b", "var_b", "correlation", "max_corr_ab", "max_corr_ba"):
            assert torch.equal(torch.isnan(got[k]), torch.isnan(want[k])), (na, nb, k)
            torch.testing.assert_close(got[k].nan_to_num(), want[k].nan_to_num(), rtol=0, atol=1e-12)
        for k in ("argmax_ab", "argmax_ba"):
            assert torch.equal(got[k], want[k]), (na, nb, k)


def test_golden_has_dead_feature_and_tie(golden):
    tt = golden["pairs"][("tied", "tied")]
    dead = golden["dead"]
    assert torch.isnan(tt["correlation"][dead]).all()
    assert int(tt["argmax_ab"][dead]) == -1 and torch.isnan(tt["max_corr_ab"][dead])
    c2, c7 = golden["tie_cols"]
    torch.testing.assert_close(tt["correlation"][:, c2], tt["correlation"][:, c7], rtol=0, atol=0, equal_nan=True)
    assert int(tt["argmax_ab"][0]) == c2


def test_best_ties_and_nan():
    corr = torch.tensor([[0.5, 0.9, 0.9], [float("nan")] * 3, [float("nan"), -0.2, -0.3]], dtype=torch.float64)
    mx, ag = CO.best(corr, 1)
    assert ag.tolist() == [1, -1, 1] and torch.isnan(mx[1]) and mx[0] == 0.9
    mx, ag = CO.best(corr, 0)
    assert ag.tolist() == [0, 0, 0] and mx.tolist() == [0.5, 0.9, 0.9]


def _codes(kind, N, n, g):
    if kind == "relu":
        return torch.relu(torch.randn(N, n, generator=g, dtype=torch.float64) - 0.5).float()
    if kind == "common_mean":   # a large common mean on a small spread
        return (50.0 + torch.rand(N, n, generator=g, dtype=torch.float64)).float()
    return (torch.randn(N, n, generator=g, dtype=torch.float64) * torch.logspace(-2, 2, n, dtype=torch.float64)).float()


@pytest.mark.parametrize("kind", ["relu", "common_mean", "signed"])
@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_cross_sum_bound_holds_against_emulation(kind, arith):
    g = torch.Generator().manual_seed(7)
    ca, cb = _codes(kind, 2048, 24, g), _codes(kind, 2048, 16, g)
    mm = AE.mm_bf16x3 if arith == "bf16x3" else AE.mm_f16f8
    got = mm(ca.T.contiguous(), cb)
    want = ca.double().T @ cb.double()
    bound = CO.cross_sum_bound(ca, cb, arith)
    assert bool(((got - want).abs() <= bound).all())
    # the correlation bound follows, and stays small in absolute terms except where the mean dwarfs the spread
    cb_ = CO.correlation_bound(ca, cb, bound)
    if kind != "common_mean":
        assert float(cb_.max()) < 0.05


def test_cross_moment_bytes_and_memory_check():
    acc, ws, out = metrics._cross_moment_bytes([(2, 4096)], [(1, 16384), (3, 512)], True)
    assert acc == 8 * (2 * 1 * 4096 * 16384 + 2 * 3 * 4096 * 512)
    assert ws == 4 * 4096 * 16384 + 1024
    assert out == acc
    metrics._check_cross_memory(10, 10)
    with pytest.raises(ValueError, match="need 11 bytes"):
        metrics._check_cross_memory(11, 10)


def test_host_validation():
    g = torch.Generator().manual_seed(0)
    tied = TiedSAE(torch.randn(16, 32, generator=g), torch.zeros(16))
    x = torch.randn(64, 32, generator=g)
    with pytest.raises(ValueError, match="same number of paired rows"):
        metrics.code_correlation(tied, x, tied, torch.randn(63, 32))
    odd = UntiedSAE(torch.randn(16, 12), torch.randn(16, 12), torch.zeros(16))
    with pytest.raises(ValueError, match="multiple of 8"):
        metrics.code_correlation(tied, x, odd, torch.randn(64, 12))
    with pytest.raises(NotImplementedError, match="no engine variant"):
        metrics.code_correlation(tied, x, object())
    with pytest.raises(ValueError, match="full must be"):
        metrics.code_correlation(tied, x, tied, full=1)


def test_export_declared_and_exported():
    names = ["sce_cross_moments_workspace_bytes", "sce_cross_moments", "sce_correlation_finish"]
    header = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "sce.h")).read()
    assert "size_t sce_cross_moments_workspace_bytes(const sce_plan* plan_a, const sce_plan* plan_b, int B);" in header
    assert "int sce_cross_moments(sce_plan* plan_a, sce_plan* plan_b, int B, double* acc, void* workspace," in header
    assert "int sce_correlation_finish(const double* acc, int n_a, int n_b, int lda," in header
    for n in names:
        assert n in _lib.EXPORTS
    lib = _lib.load()
    for n in names:
        assert hasattr(lib, n)
    assert lib.sce_version() == 201
    assert lib.sce_cross_moments_workspace_bytes(None, None, 1) == 0
    assert lib.sce_cross_moments(None, None, 1, None, None, 0, None) == -1
    assert lib.sce_correlation_finish(None, 1, 1, 1, None, None, 1, None, None, None, None, None, None, None) == -1
