"""Dictionary-similarity metrics on the H100 (libsce sce_similarity): every drop-in against the reference's own
results (golden fixture) under both arithmetics, and the batched forms at config-2 / config-5 scale against the fp64
oracle on the device. Tolerances: cosine maxima 1e-5 absolute (raw truth: 1e-5 ||a_i|| max_g ||t_g||), MMCS 1e-5,
capacity 1e-4 relative."""
import pytest
import torch

import sparse_coding_b200 as S
from oracle import metrics_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.learned_dict import TiedSAE, UntiedSAE

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
# f16f8 carries the cross terms on E5M2 planes (3 significant bits): ~2^-14 relative error per product, which at the
# fixture's small widths (d = 48) sums to ~1e-5 on a cosine (measured: 1.06e-5). The bar for it is 2.5e-5 there;
# bf16x3 (what auto runs) meets 1e-5.
F16F8_SLACK = 2.5


def ours(e):
    kind, w = e["kind"], e["w"].to(DEV)
    if kind == "tied":
        return TiedSAE(w, torch.zeros(w.shape[0], device=DEV), norm_encoder=True)
    if kind == "untied":
        return UntiedSAE(torch.zeros_like(w), w, torch.zeros(w.shape[0], device=DEV))
    if kind == "topk":
        return S.TopKLearnedDict(w, 4)
    return w


def arg(g, name):
    return [arg(g, x) for x in name] if isinstance(name, list) else ours(g["dicts"][name])


def tolerance(g, c):
    """1e-5 for cosines; scaled by the row norms of a raw truth operand."""
    raw = [g["dicts"][a]["w"] for a in c["args"] if not isinstance(a, list) and g["dicts"][a]["kind"] == "raw"]
    if not raw:
        return 1e-5
    t = raw[0]
    if c["fn"] == "representedness":
        return 1e-5 * t.norm(dim=-1).to(DEV)
    return 1e-5 * float(t.norm(dim=-1).max())


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_drop_ins_match_reference_golden(golden, arith):
    g = golden("dict_metrics")
    ran = 0
    for c in g["cases"]:
        widths = {g["dicts"][a]["w"].shape[-1] for a in (c["args"][0] if isinstance(c["args"][0], list) else c["args"])}
        if arith == "f16f8" and any(w % 16 for w in widths):
            continue                                                  # f16f8 needs d % 16 == 0 (auto takes bf16x3)
        got = getattr(MT, c["fn"])(*[arg(g, a) for a in c["args"]], arith=arith)
        want = c["out"].to(DEV)
        assert got.device == want.device and got.shape == want.shape, c["fn"]
        assert torch.equal(torch.isnan(got), torch.isnan(want)), (c["fn"], c["args"])
        ok = ~torch.isnan(want)
        if c["fn"] == "capacity_per_feature":
            assert ((got - want)[ok].abs() <= 1e-4 * want[ok].abs()).all(), (c["args"], (got - want)[ok].abs().max())
        else:
            tol = tolerance(g, c) * (F16F8_SLACK if arith == "f16f8" else 1.0)
            tol = tol[ok] if torch.is_tensor(tol) else tol
            assert ((got - want)[ok].abs() <= tol).all(), (c["fn"], c["args"], (got - want)[ok].abs().max())
        ran += 1
    assert ran >= (53 if arith == "bf16x3" else 35)


def _check_pairs(res, L, pairs, rows=None):
    """mcs_ab / mcs_ba / mmcs of dictionary_similarity against the fp64 oracle (L: learned dicts, list of [n_m, d])."""
    for q, (i, j) in enumerate(pairs):
        r, c = O.pair_maxima(L[i], L[j])
        na, nb = L[i].shape[0], L[j].shape[0]
        assert (res["mcs_ab"][q, :na].double() - r).abs().max() <= 1e-5, (i, j)
        assert (res["mcs_ba"][q, :nb].double() - c).abs().max() <= 1e-5, (i, j)
        assert abs(float(res["mmcs"][i, j]) - float(r.mean())) <= 1e-5
        assert torch.isnan(res["mcs_ab"][q, na:]).all() and torch.isnan(res["mcs_ba"][q, nb:]).all()


def _check_capacity(cap, L):
    for m, l in enumerate(L):
        want = O.capacity_blocked(l)
        got = cap[m, : l.shape[0]].double()
        assert ((got - want).abs() <= 1e-4 * want.abs()).all(), (m, ((got - want).abs() / want.abs()).max())


def _cfg2_ensemble():
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(512, 4096, a) for a in torch.logspace(-4, -2, 16).tolist()]
    return S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)


def _learned(ens):
    return [ens.sig.to_learned_dict(p, b).get_learned_dict().double() for p, b in ens.unstack()]


def test_config2_all_pairs_and_capacity_fresh_and_trained():
    ens = _cfg2_ensemble()
    gen = torch.Generator(device=DEV).manual_seed(1)
    for steps in (0, 30):
        for _ in range(steps):
            ens.step_batch(torch.randn(2048, 512, device=DEV, generator=gen))
        res = MT.dictionary_similarity(ens)                           # all 120 lower-triangle pairs, both directions
        assert res["pairs"].shape == (120, 2)
        L = _learned(ens)
        pairs = [tuple(p) for p in res["pairs"].tolist()]
        _check_pairs(res, L, pairs)
        for i, j in pairs:                                            # the mirror entries come from the column maxima
            assert abs(float(res["mmcs"][j, i]) - float(O.pair_maxima(L[j], L[i])[0].mean())) <= 1e-5
        _check_capacity(MT.capacity(ens), L)


def test_config5_width():
    torch.manual_seed(2)
    lds = [TiedSAE(torch.randn(32768, 2048, device=DEV), torch.zeros(32768, device=DEV)) for _ in range(2)]
    res = MT.dictionary_similarity(lds, pairs=[(1, 0)])
    L = [ld.get_learned_dict().double() for ld in lds]
    _check_pairs(res, L, [(1, 0)])
    _check_capacity(MT.capacity(lds), L)


def test_masked_stack_grid_as_in_log_standard_metrics():
    """big_sweep.py:108-138: the smallest dictionary against every larger one, per L1 value, in one call."""
    torch.manual_seed(3)
    sizes, l1s = (1024, 2048, 4096), (1e-3, 3e-3)
    models = [S.FunctionalMaskedTiedSAE.init(512, k, 4096, a) for a in l1s for k in sizes]
    ens = S.FunctionalEnsemble(models, S.FunctionalMaskedTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    ens.step_batch(torch.randn(1024, 512, device=DEV))
    # (larger, smallest): mcs_ab = each atom of the larger dictionary, its best match in the smallest =
    # standard_metrics.mcs_duplicates(small, larger)
    pairs = [(li * 3 + s, li * 3) for li in range(len(l1s)) for s in (1, 2)]
    res = MT.dictionary_similarity(ens, pairs=pairs)
    L = _learned(ens)
    assert [l.shape[0] for l in L] == list(sizes) * 2
    _check_pairs(res, L, pairs)
    grid = [[float(res["mmcs"][i, j]) for i, j in pairs[2 * li: 2 * li + 2]] for li in range(len(l1s))]
    for li in range(len(l1s)):
        for s in (1, 2):
            small, larger = L[li * 3], L[li * 3 + s]
            assert abs(grid[li][s - 1] - float(O.mmcs(small, larger))) <= 1e-5
    _check_capacity(MT.capacity(ens), L)


def test_raw_truth_beyond_fp16_range():
    torch.manual_seed(4)
    model = TiedSAE(torch.randn(300, 64, device=DEV), torch.zeros(300, device=DEV))
    truth = torch.randn(200, 64, device=DEV) * 1e5                    # |v| > 65504: fp16 cannot hold it
    assert truth.abs().max() > 65504
    want = O.mcs_to_fixed(model.get_learned_dict().double(), truth.double())
    got = MT.mcs_to_fixed(model, truth)                              # auto: bf16x3
    assert torch.isfinite(got).all()
    assert (got.double() - want).abs().max() <= 1e-5 * float(truth.norm(dim=-1).max())
    with pytest.raises(_lib.SceError, match="fp16"):
        MT.mcs_to_fixed(model, truth, arith="f16f8")


def test_repeated_calls_are_bitwise_equal():
    ens = _cfg2_ensemble()
    pairs = [(i, j) for i in range(16) for j in range(16)]
    a = MT.dictionary_similarity(ens, pairs=pairs)
    b = MT.dictionary_similarity(ens, pairs=pairs)
    for k in ("mcs_ab", "mcs_ba", "mmcs"):
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
    assert torch.equal(MT.capacity(ens).view(torch.int32), MT.capacity(ens).view(torch.int32))


@pytest.mark.parametrize("masked", [False, True])
def test_ensemble_and_exported_dicts_agree_bitwise(masked):
    torch.manual_seed(5)
    if masked:
        sig, models = S.FunctionalMaskedSAE, [S.FunctionalMaskedSAE.init(256, k, 1024, 1e-3) for k in (1024, 300, 777)]
    else:
        sig, models = S.FunctionalSAE, [S.FunctionalSAE.init(256, 1024, a) for a in (1e-3, 2e-3, 4e-3)]
    ens = S.FunctionalEnsemble(models, sig, S.adam, {"lr": 1e-3}, device=DEV)
    lds = [sig.to_learned_dict(p, b) for p, b in ens.unstack()]
    for fn in (lambda x: MT.dictionary_similarity(x, pairs="all"), lambda x: {"capacity": MT.capacity(x)}):
        a, b = fn(ens), fn(lds)
        for k in a:
            if k != "pairs":
                assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
