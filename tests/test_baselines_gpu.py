"""The baseline dictionaries through the public API on the GPU: evaluate_dicts and its drop-ins against the reference's own
metrics (tests/golden/baselines.pt), an ICAEncoder fitted by the engine scored and interpreted end to end against fp64,
and the existing kinds giving the same bits alone and next to the baselines."""
import io

import numpy as np
import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import DEV, tied, topk, untied
from oracle import baselines_oracle as BO
from oracle.ica_oracle import mixed_sources
from sparse_coding_b200.ica import ICAEncoder
from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict

pytestmark = pytest.mark.gpu
ARITHS = ["bf16x3", "f16f8"]
GOLDEN = BO.load_golden()


def cases():
    return BO.golden_cases(GOLDEN)


def _moment_tol(ref):
    return 2e-4 * float(ref.abs().max()) + 1e-7


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_parity_with_the_reference(case, arith):
    name, ld, m, x, want = case
    seg, thr = GOLDEN["segment"], GOLDEN["threshold"]
    xd = x.to(DEV)
    r = S.evaluate_dicts([ld], xd, segment=seg, threshold=thr, arith=arith)[0]
    md = BO.to(m, DEV)
    c, z = BO.encode(md, xd), BO.pre_activations(md, xd)
    # activity flips only where the fp64 pre-activation lies within the engine's rounding of 0
    near = (z.abs() < 1e-5 * float(z.abs().max())).sum(0)
    counts = (c != 0).sum(0)
    assert bool(((r["feature_counts"].long() - counts).abs() <= near).all()), name
    assert torch.allclose(r["feature_frequency"].double().cpu(), want["mean_nonzero_activations"],
                          atol=1e-6 + float(near.max()) / x.shape[0])
    if int(near.sum()) == 0:
        assert int(r["n_ever_active"]) == want["n_ever_active"]
        assert torch.equal(r["times_active"].double().cpu(), want["moments"]["times_active"])
    for k in ("mean", "var", "m4"):
        ref = want["moments"][k]
        assert torch.allclose(r[k].double().cpu(), ref, rtol=2e-4, atol=_moment_tol(ref)), (name, k)
    if "fvu_error" in want:
        assert bool(r["fvu"].isnan()) and bool(S.fraction_variance_unexplained(ld, xd, arith=arith).isnan())
        assert bool(S.r_squared(ld, xd, arith=arith).isnan())
        for k in ("mean_l0", "skew", "kurtosis"):
            assert bool(torch.isfinite(r[k]).all()), k
    else:
        assert abs(float(r["fvu"]) - want["fvu"]) <= 2e-4 * abs(want["fvu"]), (name, float(r["fvu"]), want["fvu"])
    # the raw-batch drop-ins apply ICA's translation too (it belongs to encode)
    times, mean, var, skew, kurt, m4 = S.calc_moments_streaming(ld, xd, batch_size=seg, arith=arith)
    assert torch.allclose(mean.double().cpu(), want["moments"]["mean"], rtol=2e-4,
                          atol=_moment_tol(want["moments"]["mean"]))
    if int(near.sum()) == 0:
        assert S.batched_calc_feature_n_ever_active(ld, xd, seg, thr, arith=arith) == want["n_ever_active"]


def _fragment_maxima(c, L):
    return c.view(-1, L, c.shape[1]).amax(dim=1)          # [G, n]


@pytest.mark.parametrize("arith", ARITHS)
def test_engine_fitted_ica_end_to_end(arith):
    d, N, L = 64, 16384, 64
    x64, _ = mixed_sources(d, N, 5)
    x = (x64 + 40.0 * torch.linspace(-1, 1, d, dtype=torch.float64)).float().to(DEV)   # a large offset on some columns
    np.random.seed(3)
    ica = ICAEncoder(d, device=DEV, arith="bf16x3").fit(x)
    c = ica.encode(x)                                      # fp64 on the device
    assert bool((c < 0).any())
    r = S.evaluate_dicts([ica], x, segment=1000, arith=arith)[0]
    assert bool(r["fvu"].isnan())
    # (the streaming moments weight the last partial segment like a full one, as the reference does)
    m = BO.to(BO.ica(ica.scaler.mean_, ica.scaler.scale_, ica.ica.components_, ica.ica.mean_), DEV)
    times, mean, var, _, _, m4 = BO.calc_moments_streaming(m, x, 1000)
    assert torch.allclose(r["mean"].double(), mean, rtol=0, atol=1e-5 * float(c.abs().max()))
    assert torch.allclose(r["var"].double(), var, rtol=1e-4)
    assert torch.allclose(r["m4"].double(), m4, rtol=1e-3)
    assert torch.equal(r["times_active"].double(), times)
    assert int(r["n_ever_active"]) == d
    # record selection: negative maxima are kept, the lists are ordered, and every value is its row's maximum
    out = S.top_activating_fragments([ica], x, fragment_len=L, n_top=20, n_random=8, arith=arith)[0]
    fm = _fragment_maxima(c, L)                            # [G, n] fp64
    tv, tf, ta = out["top_values"], out["top_fragments"], out["top_activations"]
    assert bool((tf >= 0).all()) and bool((tv[:, :-1] >= tv[:, 1:]).all())
    assert torch.equal(tv, ta.amax(dim=-1))
    scale = 1e-4 * float(c.abs().max())
    got = fm.T.gather(1, tf)                               # the fp64 maxima of the chosen fragments
    assert bool(((got - tv.double()).abs() <= scale).all())
    kth = fm.T.sort(dim=1, descending=True).values[:, 19]
    assert bool((got[:, -1] >= kth - 2 * scale).all())
    # fragments with only negative values: their maximum is negative, and a feature's list may consist of them
    neg = -c
    ica_neg = ICAEncoder(d)
    ica_neg.scaler, ica_neg.ica = ica.scaler, type(ica.ica)(-ica.ica.components_, ica.ica.mixing_, ica.ica.mean_,
                                                            None, None, 0)
    o2 = S.top_activating_fragments([ica_neg], x, fragment_len=L, n_top=4, n_random=0, arith=arith)[0]
    fm2 = _fragment_maxima(neg, L)
    assert bool((o2["top_values"].double() - fm2.T.gather(1, o2["top_fragments"])).abs().max() <= scale)


@pytest.mark.parametrize("arith", ARITHS)
def test_existing_kinds_unchanged_next_to_the_baselines(arith):
    d, N = 64, 6000
    x = torch.randn(N, d, device=DEV) + 0.1
    sae = [tied(96, d, 1), untied(80, d, 2), topk(96, d, 5, 3)]
    torch.manual_seed(7)
    rd, ir = RandomDict(d, 128), IdentityReLU(d)
    alone = S.evaluate_dicts(sae, x, arith=arith)
    mixed = S.evaluate_dicts([rd, sae[0], ir, sae[1], sae[2]], x, arith=arith)
    for a, b in zip(alone, [mixed[1], mixed[3], mixed[4]]):
        for k in a:
            va, vb = a[k], b[k]
            assert (va == vb) if not torch.is_tensor(va) else torch.equal(va, vb), k
    L = 64
    x2 = x[:64 * 64]
    fa = S.top_activating_fragments(sae, x2, fragment_len=L, arith=arith)
    fb = S.top_activating_fragments([sae[0], rd, sae[1], ir, sae[2]], x2, fragment_len=L, arith=arith)
    for a, b in zip(fa, [fb[0], fb[2], fb[4]]):
        for k in a:
            assert (a[k] == b[k]) if not torch.is_tensor(a[k]) else torch.equal(a[k], b[k]), k
    # IdentityReLU is the untied SAE with E = D = I: the same plan, the same bits
    eye = torch.eye(d, device=DEV)
    u = S.UntiedSAE(eye, eye, ir.bias.to(DEV))
    ra, rb = S.evaluate_dicts([ir], x, arith=arith)[0], S.evaluate_dicts([u], x, arith=arith)[0]
    for k in ra:
        assert (ra[k] == rb[k]) if not torch.is_tensor(ra[k]) else torch.equal(ra[k], rb[k]), k


def _golden_selection(kind):
    e = next(e for e in GOLDEN[kind] if e["interp"] is not None)
    ld = BO.ica_from_golden(e) if kind == "ica" else torch.load(io.BytesIO(e["pickle"]), weights_only=False)
    return ld, e["interp"]


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", ["ica", "random"])
def test_record_selection_matches_the_reference(kind, arith):
    """top_activating_fragments against the reference's interpret.py on the same fragments (tests/golden/baselines.pt):
    per feature the same 20 top fragments with the same fp16 maxima in the same order (fragments whose fp16 maxima tie
    may come in either order: the reference's quicksort leaves it unspecified), the same skipped features, and for ICA
    negative maxima among them."""
    ld, ref = _golden_selection(kind)
    acts = ref["acts"].to(DEV)
    out = S.top_activating_fragments([ld], acts, fragment_len=64, n_top=20, n_random=20, arith=arith)[0]
    maxes = ref["maxes"].float().T.to(DEV)                 # [n, G], the reference's fp16 table
    head = ref["head"].to(DEV)
    frags = out["top_fragments"]
    assert torch.equal(maxes.gather(1, frags), maxes.gather(1, head))
    assert torch.equal(frags.sort(1).values, head.sort(1).values)
    # the engine's fp32 maxima, rounded to fp16, are the reference's fp16 maxima to one fp16 step
    want = maxes.gather(1, frags)
    step = torch.where(want == 0, torch.full_like(want, 2.0 ** -24), want.abs() * 2.0 ** -10)
    assert bool(((out["top_values"].half().float() - want).abs() <= step).all())
    assert torch.equal(out["skipped"].cpu(), ref["skipped"])
    if kind == "ica":
        assert bool((out["top_values"] < 0).any()) and bool((maxes < 0).all(dim=1).any())
        assert int(out["n_active_fragments"].min()) == maxes.shape[1]    # signed codes: every fragment is active
