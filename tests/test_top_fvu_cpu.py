"""The top- and rest-feature FVU without a GPU: the golden fixture (the reference's own
fraction_variance_unexplained_top_activating) against the fp64 restatement in oracle/top_fvu_oracle.py, the selection
order and its tie rule, the argument checks of evaluate_dicts(n_top=...) and the drop-in before any device work, and the
sce_forward_split workspace query and its checks that need no plan."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import desc
from oracle import eval_oracle as EO
from oracle import top_fvu_oracle as TO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT


def oracle_dict(e):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in e.items()}


def test_golden_matches_fp64_oracle(golden):
    g = golden("top_fvu")
    assert len(g["cases"]) == 6 * len(g["n_tops"])
    for c in g["cases"]:
        m = oracle_dict(g["dicts"][c["dict"]])
        d = (m["dict"] if m["kind"] == "topk" else m["encoder"]).shape[1]
        x = TO.rows(d, c["x_seed"]).double()
        top, rest, feats = TO.fraction_variance_unexplained_top_activating(m, x, c["n_top"])
        assert torch.equal(feats, c["top_features"]), c["dict"]
        assert abs(float(top) / c["fvu_top"] - 1) < 1e-5, (c["dict"], c["n_top"], float(top), c["fvu_top"])
        assert abs(float(rest) / c["fvu_rest"] - 1) < 1e-5, (c["dict"], c["n_top"], float(rest), c["fvu_rest"])


def test_golden_covers_the_cases(golden):
    g = golden("top_fvu")
    assert {e["kind"] for e in g["dicts"].values()} == {"tied", "untied", "topk", "random", "identity_relu"}
    cen = g["dicts"]["tied_centred"]
    assert cen["center_trans"].abs().max() > 0.1 and cen["center_scale"].std() > 0.1
    assert "center_trans" not in g["dicts"]["tied_identity"]
    assert set(g["n_tops"]) == {1, 2, 5} and g["n_eval"] % 1000
    assert {e["encoder"].shape[1] for e in g["dicts"].values() if "encoder" in e} == {32, 64}
    assert all(c["gap"] >= 1e-3 for c in g["cases"])
    assert g["ica_error"] and "RuntimeError" in g["ica_error"]
    # the quirk is visible: center, not uncenter, of the partial reconstructions of the centred TiedSAE
    m = oracle_dict(cen)
    x = TO.rows(32, 1).double()
    c = TO.code(m, x)
    feats = TO.top_features(c, 2)
    keep = torch.zeros(c.shape[1], dtype=torch.bool)
    keep[feats] = True
    w = TO.decoder(m)
    plain = (x - EO.uncenter(m, (c * keep) @ w)).pow(2).mean() / (x - x.mean(0)).pow(2).mean()
    got = [k for k in g["cases"] if k["dict"] == "tied_centred" and k["n_top"] == 2][0]["fvu_top"]
    assert abs(float(plain) / got - 1) > 1e-2


def test_selection_order_and_ties():
    sums = torch.tensor([1.0, 3.0, 3.0, 2.0, 3.0, -1.0, 0.0], dtype=torch.float64)
    assert MT._top_features(sums, 7).tolist() == [1, 2, 4, 3, 0, 6, 5]
    # padding columns past n never take part
    assert MT._top_features(torch.cat([sums[:4], torch.tensor([9.0, 9.0], dtype=torch.float64)]), 4).tolist() == [1, 2, 3, 0]
    c = torch.tensor([[1.0, 2.0, 2.0, 0.5], [1.0, 2.0, 2.0, 0.5]], dtype=torch.float64)
    assert TO.top_features(c, 3).tolist() == [1, 2, 0]


def _tied(n, d):
    return S.TiedSAE(torch.randn(n, d), torch.zeros(n))


def test_argument_errors():
    x = torch.randn(100, 64)
    lds = [_tied(16, 64), _tied(40, 64)]
    for bad in (0, -1, 65, 2.0, "2", True):
        with pytest.raises(ValueError, match="n_top"):
            MT.evaluate_dicts(lds, x, n_top=bad)
    with pytest.raises(ValueError, match="n_top = 17 exceeds dictionary 0's 16 features"):
        MT.evaluate_dicts(lds, x, n_top=17)
    with pytest.raises(ValueError, match="n_top"):
        S.fraction_variance_unexplained_top_activating(lds[0], x, n_top=0)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            S.fraction_variance_unexplained_top_activating(lds[0], x, n_top=2)


def test_split_workspace_query():
    lib = _lib.load()
    ws = lambda M, n, d, B, k, Bmax=None: lib.sce_forward_split_workspace_bytes(C.byref(desc(M, n, d, Bmax or B, lr=0.0)),
                                                                              B, k)
    # config 2: x_hat 256 MiB, code columns 1 MiB, dictionary rows 64 KiB, partials 32 KiB
    assert ws(16, 4096, 512, 8192, 2) == (256 << 20) + (1 << 20) + (64 << 10) + (32 << 10)
    up = lambda b: -(-b // 1024) * 1024
    assert ws(2, 40, 64, 33, 5) == up(2 * 33 * 64 * 4) + up(2 * 33 * 5 * 4) + up(2 * 5 * 64 * 4) + up(2 * 2 * 2 * 4)
    assert ws(2, 40, 64, 33, 1) > 0 and ws(2, 40, 64, 33, 40) > 0 and ws(2, 40, 64, 33, 8) > 0
    assert ws(2, 40, 64, 33, 0) == 0 and ws(2, 40, 64, 33, 41) == 0 and ws(2, 80, 64, 33, 65) == 0
    assert ws(2, 40, 64, 0, 2, 64) == 0 and ws(2, 40, 64, 65, 2, 64) == 0 and ws(2, 36, 64, 64, 2) == 0
    assert _lib.SCE_SPLIT_MAX_TOP == 64


def test_split_argument_errors():
    lib = _lib.load()
    rc = lib.sce_forward_split(None, 1 << 20, 16, 2, 1 << 21, 1 << 22, 1 << 23, None, None, 1 << 30, 1 << 40, None)
    assert rc == -1
    assert "forward_split: plan is NULL" in lib.sce_last_error().decode()
