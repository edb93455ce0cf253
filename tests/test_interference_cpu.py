"""The expected interference without a GPU: the golden fixture (the reference's own calc_expected_interference) against
the fp64 restatement in oracle/interference_oracle.py, what the fixture covers, the argument checks of the drop-in and of
evaluate_dicts(interference=...), the two workspace queries, and the ABI refusals that are checked on the host."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import desc
from interference_cases import KINDS, cases, rel_err, workspace_bytes
from oracle import interference_oracle as IO
from sparse_coding_b200 import _lib


def test_golden_matches_fp64_oracle(golden):
    cs = cases(golden)
    assert set(cs) == set(KINDS)
    for name, c in cs.items():
        want = IO.expected_interference(c["dictionary"], c["code"])
        assert rel_err(want, c["expected"]) < 1e-5, name
        cap, nz, _ = IO.sums(c["dictionary"], c["code"])
        assert torch.equal(nz, c["nz_counts"]), name


def test_golden_covers_the_cases(golden):
    g = golden("interference")
    cs = cases(golden)
    tied = cs["tied"]
    # a zero-norm dictionary row whose feature is active: totals 0, clamped, cap = c / 1e-8
    zero = int((tied["dictionary"].norm(dim=-1) == 0).nonzero()[0])
    assert tied["nz_counts"][zero] > 0 and tied["expected"][zero] > 1e6
    # an all-zero code column: count 0, floored at 1, result 0
    assert (tied["nz_counts"] == 0).any() and (tied["expected"][tied["nz_counts"] == 0] == 0).all()
    for name in KINDS:
        nnz = (cs[name]["code"] != 0).sum(1)
        assert (nnz == 1).any(), name                  # single active features: cap = 1 (or 1e8 c for a zero row)
    ica = cs["ica"]
    assert (ica["code"] < 0).any()
    i = g["signed_feature"]
    wn = IO.normalised(ica["dictionary"])
    totals = ica["code"].double() @ (wn @ wn.T).pow(2).T
    assert ((ica["code"][:, i] != 0) & (totals[:, i] < 0)).any()    # a signed row whose totals fall below the clamp
    assert ica["expected"][i].abs() > 1e6


def test_oracle_single_feature_and_clamp():
    dictionary = torch.tensor([[3.0, 4.0], [0.0, 0.0], [1.0, 0.0]])
    code = torch.tensor([[2.0, 0.0, 0.0], [0.0, 0.5, 0.0], [1.0, 0.0, -4.0], [0.0, 0.0, 0.0]])
    cap, nz, _ = IO.sums(dictionary, code)
    assert nz.tolist() == [2, 1, 1]
    # row 0: a single feature, cap = 1; row 1: a zero row, totals 0 -> 0.5 / 1e-8; row 2: cos^2 = 0.36,
    # totals_0 = 1 - 1.44 < 0 -> 1 / 1e-8, totals_2 = 0.36 - 4 < 0 -> -4 / 1e-8
    assert cap[0].item() == pytest.approx(1.0 + 1e8)
    assert cap[1].item() == pytest.approx(0.5e8)
    assert cap[2].item() == pytest.approx(-4e8)


def test_argument_errors():
    w, c = torch.randn(16, 8), torch.rand(4, 16)
    with pytest.raises(ValueError, match="CUDA device"):
        S.calc_expected_interference(w, c)
    with pytest.raises(ValueError, match="features"):
        S.calc_expected_interference(w, torch.rand(4, 15))
    with pytest.raises(ValueError, match=r"\[n, d\]"):
        S.calc_expected_interference(w[0], c)
    with pytest.raises(ValueError, match="arith"):
        S.calc_expected_interference(w, c, arith="fp8")
    with pytest.raises(TypeError):
        S.calc_expected_interference(w.numpy(), c)
    ld = S.TiedSAE(torch.randn(16, 8), torch.zeros(16))
    with pytest.raises(ValueError, match="interference must be True or False"):
        S.evaluate_dicts([ld], torch.randn(32, 8), interference="yes")


def test_workspace_queries():
    lib = _lib.load()
    q = lambda M, n, d, B, Bmax=None, **f: lib.sce_interference_workspace_bytes(C.byref(desc(M, n, d, Bmax or B, lr=0.0, **f)), B)
    for M, n, d, B in ((1, 8, 8, 1), (16, 4096, 512, 8192), (3, 72, 40, 33), (2, 48, 64, 200)):
        assert q(M, n, d, B) == workspace_bytes(M, n, d, B), (M, n, d, B)
    assert q(16, 4096, 512, 8192) == 256 << 20
    assert q(2, 48, 32, 0, Bmax=64) == 0 and q(2, 48, 32, 65, Bmax=64) == 0
    assert q(2, 48, 32, 64, variant=_lib.SCE_TIED_LEARNED_CENTER) == 0
    assert q(2, 48, 32, 64, encoder_nonneg=1) == 0 and q(2, 48, 32, 64, input_shift=0.18) == 0
    assert q(2, 44, 32, 64) == 0                                   # n not a multiple of 8: an invalid desc
    assert lib.sce_interference_workspace_bytes(None, 4) == 0
    e = lib.sce_expected_interference_workspace_bytes
    for n, d, B in ((1, 1, 1), (13, 7, 100), (4096, 512, 8192)):
        assert e(n, d, B) == workspace_bytes(1, n, d, B), (n, d, B)
    assert e(0, 8, 8) == 0 and e(8, 0, 8) == 0 and e(8, 8, 0) == 0


def test_host_refusals():
    """Refusals that return before any device call: a NULL plan or pointer, n / d / B < 1, a short or misaligned
    workspace."""
    lib = _lib.load()
    err = lambda: lib.sce_last_error().decode()
    fake = C.c_void_p(1 << 20)
    assert lib.sce_code_interference(None, 8, fake, fake, fake, 1 << 20, None) == -1
    assert "plan is NULL" in err()
    call = lambda dic=fake, n=8, d=8, code=fake, B=4, cap=fake, nz=fake, ws=C.c_void_p(1 << 20), nb=1 << 20: \
        lib.sce_expected_interference(dic, n, d, code, B, cap, nz, ws, nb, None)
    assert call(dic=None) == -1 and "dict / code is NULL" in err()
    assert call(code=None) == -1 and "dict / code is NULL" in err()
    assert call(n=0) == -1 and "must be >= 1" in err()
    assert call(B=0) == -1 and "must be >= 1" in err()
    assert call(cap=None) == -1 and "cap_sums and nz_counts are required" in err()
    assert call(nz=None) == -1 and "cap_sums and nz_counts are required" in err()
    need = lib.sce_expected_interference_workspace_bytes(8, 8, 4)
    assert call(nb=need - 1) == -3 and "workspace too small" in err()
    assert call(ws=None) == -3
    assert call(ws=C.c_void_p((1 << 20) + 256), nb=need) == -3 and "1024-byte aligned" in err()
