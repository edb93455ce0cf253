"""Dictionary evaluation without a GPU: the golden fixture (the reference's own standard_metrics scores) against the
fp64 restatement in oracle/eval_oracle.py, grouping / padding / order of a mixed list, the errors the drop-ins raise
before any device work, and the sce_forward_stats workspace bound and argument checks."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import desc
from oracle import eval_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT


def oracle_dict(e):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in e.items()}


def test_golden_matches_fp64_oracle(golden):
    g = golden("dict_eval")
    assert len(g["cases"]) >= 50
    for c in g["cases"]:
        want = O.FUNCS[c["fn"]](oracle_dict(g["dicts"][c["dict"]]), g["acts"][c["acts"]].double(), **c["kwargs"])
        got = c["out"]
        if isinstance(got, int):
            assert got == want, c
            continue
        got, want = (got, want) if isinstance(got, tuple) else ((got,), (want,))
        for a, b in zip(got, want):
            b = torch.as_tensor(b, dtype=torch.float64)
            assert a.shape == b.shape, c["fn"]
            assert torch.allclose(a.double(), b, rtol=2e-4, atol=1e-6), (c["fn"], c["dict"], (a.double() - b).abs().max())


def test_golden_covers_the_edge_cases(golden):
    g = golden("dict_eval")
    kinds = {e["kind"] for e in g["dicts"].values()}
    assert {"tied", "untied", "topk"} <= kinds
    cen = g["dicts"]["tied_centred"]
    rot = cen["center_rot"]
    assert not torch.allclose(rot @ rot.T, torch.eye(rot.shape[0]), atol=1e-2) and cen["center_scale"].std() > 0.1
    assert g["dicts"]["tied_odd"]["encoder"].shape[0] % 8
    ns = [x.shape[0] for x in g["acts"].values()]
    assert any(n % 1000 for n in ns if n > 1000) and any(n < 1000 for n in ns)
    never = [c for c in g["cases"] if c["fn"] == "calc_moments_streaming" and c["dict"] == "tied_odd"][0]
    assert never["out"][0][3] == 0 and never["out"][1][3] == 0       # feature 3 never fires
    thr = [c for c in g["cases"] if c["kwargs"].get("threshold") is not None]
    assert thr and all(isinstance(c["out"], int) for c in thr)


def _tied(n, d, **kw):
    return S.TiedSAE(torch.randn(n, d), torch.zeros(n), **kw)


def test_grouping_padding_and_order_of_a_mixed_list():
    d = 64
    rot = torch.eye(d) * 2
    lds = [_tied(100, d), S.UntiedSAE(torch.randn(96, d), torch.randn(96, d), torch.zeros(96)), _tied(104, d),
           S.TopKLearnedDict(torch.randn(64, d), 8), _tied(100, d, centering=(None, rot, None)), _tied(96, d)]
    groups = MT._eval_groups(lds, True, 8)
    assert list(groups.items()) == [(("tied", 104, d, False), [0, 2]), (("untied", 96, d, False), [1]),
                                    (("topk", 64, d, False), [3]), (("tied", 104, d, True), [4]),
                                    (("tied", 96, d, False), [5])]
    # the raw-batch drop-ins plan without centring; f16f8 pads to a multiple of 16
    assert MT._eval_groups([lds[4]], False, 8) == {("tied", 104, d, False): [0]}
    assert MT._eval_groups([lds[0]], True, 16) == {("tied", 112, d, False): [0]}


def test_errors_name_the_constraint():
    x = torch.randn(100, 64)
    with pytest.raises(NotImplementedError, match="norm_encoder=False"):
        MT.evaluate_dicts([_tied(64, 64, norm_encoder=False)], x)

    class Other(S.LearnedDict):
        n_feats, activation_size = 8, 64

        def get_learned_dict(self):
            return torch.zeros(8, 64)

        def encode(self, b):
            return b[:, :8]

        def to_device(self, dev):
            pass

    with pytest.raises(NotImplementedError, match="Other has no engine variant"):
        MT.fraction_variance_unexplained(Other(), x)
    with pytest.raises(ValueError, match="multiple of 8"):
        MT.calc_moments_streaming(S.TopKLearnedDict(torch.randn(60, 64), 4), x)
    with pytest.raises(ValueError, match="d = 60 must be a multiple of 8"):
        MT.mean_nonzero_activations(_tied(64, 60), torch.randn(10, 60))
    with pytest.raises(ValueError, match="non-empty"):
        MT.r_squared(_tied(64, 64), torch.zeros(0, 64))
    with pytest.raises(ValueError, match=">= 1"):
        MT.batched_calc_feature_n_ever_active(_tied(64, 64), x, batch_size=0)
    with pytest.raises(ValueError, match=">= 1"):
        MT.evaluate_dicts([_tied(64, 64)], x, segment=0)


def test_stats_workspace_bound():
    lib = _lib.load()
    ws = lambda M, n, d, B, Bmax=None: lib.sce_forward_stats_workspace_bytes(C.byref(desc(M, n, d, Bmax or B, lr=0.0)), B)
    assert ws(16, 4096, 512, 8192) == 16 * 256 * 4 * 4096 * 4 == 256 << 20          # config 2
    assert ws(1, 32768, 2048, 4096) == 128 * 4 * 32768 * 4 == 64 << 20             # config 5's width
    assert ws(2, 40, 64, 33) == 1024 * -(-(2 * 2 * 4 * 40 * 4) // 1024)
    assert ws(2, 40, 64, 0, 64) == 0 and ws(2, 40, 64, 65, 64) == 0 and ws(2, 36, 64, 64) == 0


def test_forward_stats_argument_errors():
    lib = _lib.load()
    call = lambda **k: lib.sce_forward_stats(
        k.get("plan"), k.get("x", 1 << 20), k.get("B", 16), k.get("seg", 1), k.get("phase", 0), None, 1 << 21,
        1 << 22, 1 << 23, 1 << 24, k.get("open"), k.get("ws", 1 << 30), k.get("ws_bytes", 1 << 40), None)
    assert call() == -1
    assert "plan is NULL" in lib.sce_last_error().decode()
