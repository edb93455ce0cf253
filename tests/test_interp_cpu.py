"""Record selection without a GPU: the golden fixture (the reference's own make_feature_activation_dataset and
interpret, tests/golden/interp.pt) against the fp64 restatement in oracle/interp_oracle.py, the priority hash against
a plain-integer splitmix64, the errors top_activating_fragments raises before any device work, and the
sce_forward_fragments workspace bound and argument checks."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import desc
from oracle import interp_oracle as IO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

FP16_TINY = 2.0 ** -24          # fp16's smallest subnormal


def oracle_dict(e):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in e.items()}


def splitmix64_int(z):
    m = (1 << 64) - 1
    z = (z + 0x9E3779B97F4A7C15) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def test_priority_is_splitmix64():
    for seed in (0, 1, 12345, (1 << 64) - 1, -1):
        p = IO.priority(seed, torch.arange(40), torch.tensor([0, 1, 7, 49999, 1 << 40]))
        for gi, g in enumerate((0, 1, 7, 49999, 1 << 40)):
            for f in (0, 3, 39):
                want = splitmix64_int(splitmix64_int(splitmix64_int(seed & ((1 << 64) - 1)) ^ f) ^ g) >> 1
                assert int(p[gi, f]) == want


def test_golden_covers_the_edge_cases(golden):
    g = golden("interp")
    assert {e["kind"] for e in g["dicts"].values()} == {"tied", "untied", "topk"}
    assert g["dicts"]["tied_odd"]["encoder"].shape[0] % 8
    n_act = {k: (c["maxes"] > 0).sum(0) for k, c in g["cases"].items()}
    t = n_act["tied_odd"]
    assert (t == 0).any()                                   # a feature that never fires
    assert ((t > 0) & (t < 20)).any() and (t > 20).any()    # skipped features with a positive part, and kept ones
    assert g["cases"]["tied_odd"]["skipped"].any() and not g["cases"]["tied_odd"]["skipped"].all()


def test_golden_matches_fp64_oracle(golden):
    g = golden("interp")
    L, k = g["fragment_len"], g["n_examples"]
    x = g["acts"].double()
    for name, case in g["cases"].items():
        m = oracle_dict(g["dicts"][name])
        o = IO.select(m, x, L=L, n_top=k, n_random=k, seed=0)
        maxes = case["maxes"].double()
        # the reference's fp16 table is the oracle's maxima rounded to fp16
        assert torch.allclose(maxes, o["fmax"], rtol=2.0 ** -11, atol=FP16_TINY), name
        assert torch.equal(case["skipped"], o["skipped"]), name
        n = maxes.shape[1]
        for f in range(n):
            head = case["head"][f]
            pos = head[maxes[head, f] > 0]
            want = o["top_fragments"][f]
            want_pos = want[o["fmax"][want, f] > 0]
            # the positive part is the same set (the fixture has no fp16 tie at the boundary), in descending fp16 order
            assert set(pos.tolist()) == set(want_pos.tolist()), (name, f)
            assert len(head) - len(pos) == len(want) - len(want_pos), (name, f)     # same number of zero maxima
            if f in case["top"]:
                rec = case["top"][f]
                assert torch.equal(rec["fragments"], head), (name, f)
                vals = IO.fragment_values(o["code"][:, f:f + 1], rec["fragments"][None], L)[0]
                # fp16 rounding, plus the reference's fp32 encode next to the kink (|z| within 1e-5 of its scale)
                atol = FP16_TINY + 1e-5 * float(vals.abs().max())
                assert torch.allclose(rec["activations"].double(), vals, rtol=2.0 ** -11, atol=atol), (name, f)
        # every explained feature is one the oracle keeps, and the random picks are active, distinct, in draw order
        r = o["random_fragments"]
        for f in range(n):
            picks = r[f][r[f] >= 0]
            assert len(set(picks.tolist())) == len(picks) == min(k, int(o["n_active_fragments"][f]))
            assert bool(o["active"][picks, f].all())


def _tied(n, d, **kw):
    return S.TiedSAE(torch.randn(n, d), torch.zeros(n), **kw)


def test_errors_name_the_constraint():
    x = torch.randn(256, 64)
    ld = _tied(64, 64)
    for L in (0, 16, 48, 8224):
        with pytest.raises(ValueError, match="fragment_len"):
            MT.top_activating_fragments([ld], x, fragment_len=L)
    with pytest.raises(ValueError, match="whole number of fragments"):
        MT.top_activating_fragments([ld], x[:200], fragment_len=64)
    with pytest.raises(ValueError, match="n_top"):
        MT.top_activating_fragments([ld], x, n_top=65)
    with pytest.raises(ValueError, match="n_random"):
        MT.top_activating_fragments([ld], x, n_random=-1)
    with pytest.raises(ValueError, match="both 0"):
        MT.top_activating_fragments([ld], x, n_top=0, n_random=0)
    with pytest.raises(ValueError, match="no dictionaries"):
        MT.top_activating_fragments([], x)
    with pytest.raises(ValueError, match="non-empty"):
        MT.top_activating_fragments([ld], torch.zeros(0, 64))
    with pytest.raises(ValueError, match="fp32 or fp16"):
        MT.top_activating_fragments([ld], x.double())
    with pytest.raises(ValueError, match="arith"):
        MT.top_activating_fragments([ld], x, arith="tf32")
    with pytest.raises(ValueError, match="width 64, the activations 72"):
        MT.top_activating_fragments([ld], torch.randn(256, 72))
    with pytest.raises(ValueError, match="multiple of 8"):
        MT.top_activating_fragments([S.TopKLearnedDict(torch.randn(60, 64), 4)], x)
    with pytest.raises(NotImplementedError, match="norm_encoder=False"):
        MT.top_activating_fragments([_tied(64, 64, norm_encoder=False)], x)
    with pytest.raises(NotImplementedError, match="Other has no engine variant"):
        class Other(S.LearnedDict):
            n_feats, activation_size = 8, 64

            def get_learned_dict(self):
                return torch.zeros(8, 64)

            def encode(self, b):
                return b[:, :8]

            def to_device(self, dev):
                pass

        MT.top_activating_fragments([(Other(), {})], x)


def test_fragments_workspace_bound():
    lib = _lib.load()
    ws = lambda M, n, d, B, L, Bmax=None: lib.sce_fragments_workspace_bytes(C.byref(desc(M, n, d, Bmax or B, lr=0.0)), B, L)
    # config 2: 16 x 4096 features, 8192-row calls of 128 fragments: maxima + flags + open flags = 40 MiB + 256 KiB
    assert ws(16, 4096, 512, 8192, 64) == 16 * 128 * 4096 * 5 + 16 * 4096 * 4 == (40 << 20) + (256 << 10)
    assert ws(16, 4096, 512, 8192, 32) == 16 * 256 * 4096 * 5 + 16 * 4096 * 4
    # config 5's width
    assert ws(1, 32768, 2048, 8192, 64) == 128 * 32768 * 5 + 32768 * 4
    assert ws(1, 32768, 2048, 8192, 8192) == 32768 * 5 + 32768 * 4
    assert ws(2, 40, 64, 64, 32) == 1024 * 3                  # each part rounded up to 1 KiB
    for B, L, Bmax in ((64, 48, 64), (64, 16, 64), (96, 64, 96), (0, 32, 64), (128, 32, 64), (16384, 16384, 16384)):
        assert ws(2, 40, 64, B, L, Bmax) == 0, (B, L)
    assert ws(2, 36, 64, 64, 32) == 0                         # invalid desc


def test_forward_fragments_argument_errors():
    lib = _lib.load()
    rc = lib.sce_forward_fragments(None, 1 << 20, 64, 32, 0, 20, 20, 0, 1 << 21, 1 << 22, None, 1 << 23, 1 << 24, None,
                                   1 << 25, 1 << 30, 1 << 40, None)
    assert rc == -1 and "plan is NULL" in lib.sce_last_error().decode()
