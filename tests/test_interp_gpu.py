"""Record selection on the H100 (libsce sce_forward_fragments): top_activating_fragments against the reference's own
records (golden fixture) under both arithmetics, against the fp64 oracle at config-2 / config-5 / config-3 scale, for
L = 32 and L = 8192 and host-streamed input, plus internal consistency, repeatability and the ABI's error codes.

Tolerances. Each code value carries the error of its pre-activation z: below 2^-16 |x| |w| under bf16x3 (2^-14 on the
f16f8 cross terms), so at scale (bf16x3) values are compared within 1e-5 of the feature's largest fragment maximum plus
2^-16 max|x| |w|. Two fragments whose maxima lie inside that window may swap, so the top list may differ from the
oracle's only around its n_top-th value.
A coefficient inside the kink window (|z| < max(1e-5, 1e-4 rms(z)), DESIGN §5; top-k: also next to the row's k-th
score) may be active on one side and not the other; activity differences are allowed only where such a coefficient
exists, and their number is reported."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from oracle import eval_oracle as E
from oracle import interp_oracle as IO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FP16_TINY = 2.0 ** -24


def to_ld(m):
    f = lambda t: t.float().to(DEV)
    if m["kind"] == "tied":
        return S.TiedSAE(f(m["encoder"]), f(m["encoder_bias"]), norm_encoder=True)
    if m["kind"] == "untied":
        return S.UntiedSAE(f(m["encoder"]), f(m["decoder"]), f(m["encoder_bias"]))
    return S.TopKLearnedDict(f(m["dict"]), int(m["sparsity"]))


def from_ld(ld):
    g = lambda t: t.double().to(DEV)
    if isinstance(ld, S.TopKLearnedDict):
        return {"kind": "topk", "dict": g(ld.dict), "sparsity": int(ld.sparsity)}
    if isinstance(ld, S.UntiedSAE):
        return {"kind": "untied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias), "decoder": g(ld.decoder)}
    return {"kind": "tied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias)}


def kink_fragments(m, x, L, rows=8192):
    """[G, n] bool: fragments holding a coefficient inside the kink window."""
    z = torch.cat([E.pre_activations(m, x[i:i + rows]) for i in range(0, x.shape[0], rows)])
    w = max(1e-5, 1e-4 * float(z.pow(2).mean().sqrt()))
    near = z.abs() < w
    if m["kind"] == "topk":
        near |= (z - torch.topk(z, int(m["sparsity"]), dim=-1).values[:, -1:]).abs() < w
    return near.reshape(x.shape[0] // L, L, -1).any(1)


def check_against_oracle(ld, x, r, L, n_top, n_random, seed=0, values=True):
    m, xd = from_ld(ld), x.double().to(DEV)
    o = IO.select(m, xd, L=L, n_top=n_top, n_random=n_random, seed=seed)
    fmax = o["fmax"]                                                         # [G, n]
    n = fmax.shape[1]
    # 1e-5 of the feature's largest maximum, plus the arithmetic's error on z: 2^-16 |x| |w| (bf16x3)
    wn = m["encoder"].norm(dim=1) if m["kind"] == "untied" else torch.ones(n, dtype=torch.float64, device=DEV)
    tol = 1e-5 * fmax.amax(0).clamp(min=1e-30) + 2.0 ** -16 * float(xd.norm(dim=1).max()) * wn + FP16_TINY    # [n]
    tf, tv = r["top_fragments"].to(DEV), r["top_values"].to(DEV).double()
    assert tf.shape == (n, n_top) and bool((tf >= 0).all())
    # a top-k score next to its row's k-th largest may be selected on the other side and move its fragment's maximum by
    # a whole value: such fragments, and the lists of features that have one, are exempt from the value bounds
    kink = kink_fragments(m, xd, L)
    exempt = kink.T.gather(1, tf) if m["kind"] == "topk" else torch.zeros_like(tf, dtype=torch.bool)
    loose = kink.any(0) if m["kind"] == "topk" else torch.zeros(n, dtype=torch.bool, device=DEV)
    assert bool(((tv - fmax.T.gather(1, tf)).abs() <= tol[:, None]).logical_or(exempt).all())
    want_v = fmax.T.gather(1, o["top_fragments"])
    assert bool(((tv - want_v).abs() <= 2 * tol[:, None])[~loose].all())  # the k-th value is the oracle's k-th
    # a fragment the oracle does not keep lies inside the window around the n_top-th value
    swapped = (tf != o["top_fragments"]) & ~loose[:, None]
    edge = want_v[:, -1]
    for f in swapped.any(1).nonzero().flatten().tolist():
        extra = set(tf[f].tolist()) - set(o["top_fragments"][f].tolist())
        for g in extra:
            assert abs(float(fmax[g, f]) - float(edge[f])) <= 2 * float(tol[f]), (f, g)
    if values and r["top_activations"] is not None:
        ta = r["top_activations"].to(DEV).double()
        assert torch.equal(r["top_values"], r["top_activations"].amax(-1))   # bitwise
        want = IO.fragment_values(o["code"], tf, L)
        assert bool(((ta - want).abs() <= tol[:, None, None]).logical_or(exempt[..., None]).all())
    # activity: differences only where a coefficient lies in the kink window
    got_n = r["n_active_fragments"].to(DEV)
    diff = (got_n - o["n_active_fragments"]).abs()
    assert bool((diff <= kink.sum(0)).all())
    rf = r["random_fragments"].to(DEV)
    bad = 0
    for f in range(n):
        picks = rf[f][rf[f] >= 0]
        assert len(set(picks.tolist())) == len(picks) == min(n_random, int(got_n[f]))
        assert bool((o["active"][picks, f] | kink[picks, f]).all())
        if not torch.equal(rf[f], o["random_fragments"][f]):
            bad += 1
            assert bool(kink[:, f].any()), f
    assert torch.equal(r["skipped"].to(DEV), got_n < n_random)
    print(f"n = {n}: {int((diff > 0).sum())} features with an activity difference, {bad} with different random picks, "
          f"{int(exempt.sum())} top records exempt from the value bound")


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_golden_records(golden, arith):
    g = golden("interp")
    L, k = g["fragment_len"], g["n_examples"]
    x = g["acts"].to(DEV)
    names = list(g["cases"])
    res = MT.top_activating_fragments([to_ld(g["dicts"][nm]) for nm in names], x, fragment_len=L, n_top=k, n_random=k,
                                      arith=arith)
    # the fixture's fp16 rounding (2^-11 relative), plus the arithmetic's error on z: below 2^-14 (f16f8, E5M2 cross
    # terms) or 2^-16 (bf16x3) of |x| |w| per cross term
    eps_z = 2 * (2.0 ** -14 if arith == "f16f8" else 2.0 ** -16) * float(x.double().norm(dim=1).max())
    for nm, r in zip(names, res):
        case, m = g["cases"][nm], from_ld(to_ld(g["dicts"][nm]))
        maxes = case["maxes"].to(DEV).double()
        assert torch.equal(r["skipped"].cpu(), case["skipped"]), nm
        assert r["fragments"] == x.shape[0] // L
        o = IO.select(m, x.double(), L=L, n_top=k, n_random=k, seed=0)
        for f in range(maxes.shape[1]):
            head = case["head"][f].to(DEV)
            pos = head[maxes[head, f] > 0]
            tf = r["top_fragments"][f]
            mine = tf[r["top_values"][f] > 0]
            assert set(mine.tolist()) == set(pos.tolist()), (nm, f)
            assert len(tf) - len(mine) == len(head) - len(pos), (nm, f)
            if f in case["top"]:
                rec = case["top"][f]
                want = rec["activations"].to(DEV).double()
                got = r["top_activations"][f].double()
                # same fragments, possibly in another order where fp16 ties: compare per fragment
                idx = [tf.tolist().index(gg) for gg in rec["fragments"].tolist()]
                got = got[idx]
                w = m["encoder"] if m["kind"] == "untied" else None
                atol = FP16_TINY + 1e-5 * float(want.abs().max()) + eps_z * (float(w[f].norm()) if w is not None else 1.0)
                assert bool(((got - want).abs() <= 2.0 ** -11 * want.abs() + atol).all()), (nm, f)
            # random picks: distinct, active, and exactly the oracle's hash selection
            assert torch.equal(r["random_fragments"][f], o["random_fragments"][f]), (nm, f)
        assert torch.equal(r["n_active_fragments"], o["n_active_fragments"]), nm


def test_config2_fresh_and_trained():
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(512, 4096, a) for a in torch.logspace(-4, -2, 16).tolist()]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    x = (torch.randn(64 * 400, 512, device=DEV, generator=gen) * 0.5).half()
    for steps in (0, 30):
        for s in range(steps):
            ens.step_batch(x[(s % 12) * 2048:(s % 12 + 1) * 2048].float())
        lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in ens.unstack()]
        res = MT.top_activating_fragments(lds, x)
        for ld, r in zip(lds[::5], res[::5]):
            check_against_oracle(ld, x, r, 64, 20, 20)


def test_config5_width():
    torch.manual_seed(2)
    ld = S.TiedSAE(torch.randn(32768, 2048, device=DEV), torch.randn(32768, device=DEV) * 0.1 - 0.3)
    x = torch.randn(64 * 160, 2048, device=DEV)
    r = MT.top_activating_fragments([ld], x, n_top=8, n_random=8)[0]
    check_against_oracle(ld, x, r, 64, 8, 8)


def test_config3_topk_shapes():
    torch.manual_seed(4)
    lds = [S.TopKEncoder.to_learned_dict(*S.TopKEncoder.init(768, n, k)) for n, k in ((3072, 16), (6144, 32), (12288, 64))]
    for ld in lds:
        ld.to_device(DEV)
    x = torch.randn(64 * 150, 768, device=DEV)
    for ld, r in zip(lds, MT.top_activating_fragments(lds, x)):
        check_against_oracle(ld, x, r, 64, 20, 20)


@pytest.mark.parametrize("L", [32, 8192])
def test_fragment_lengths(L):
    torch.manual_seed(5)
    ld = S.TiedSAE(torch.randn(512, 256, device=DEV), torch.randn(512, device=DEV) * 0.3 - 1.0)
    x = torch.randn(L * (40 if L == 32 else 5), 256, device=DEV)
    k = 20 if L == 32 else 3
    r = MT.top_activating_fragments([ld], x, fragment_len=L, n_top=k, n_random=k, seed=7)[0]
    check_against_oracle(ld, x, r, L, k, k, seed=7)


def test_host_input_matches_device_input():
    torch.manual_seed(6)
    ld = S.UntiedSAE(torch.randn(1024, 128, device=DEV) * 0.2, torch.randn(1024, 128, device=DEV),
                     torch.randn(1024, device=DEV) * 0.1 - 0.4)
    x = torch.randn(64 * 300, 128).half()
    host = MT.top_activating_fragments([ld], x)[0]
    dev = MT.top_activating_fragments([ld], x.to(DEV))[0]
    assert host["top_values"].device.type == "cpu"
    for k in ("top_values", "top_fragments", "top_activations", "random_fragments", "n_active_fragments", "skipped"):
        assert torch.equal(host[k], dev[k].cpu()), k
    check_against_oracle(ld, x.to(DEV), dev, 64, 20, 20)


def test_consistency_grouping_repeatability_and_counts():
    torch.manual_seed(7)
    d = 128
    lds = [S.TiedSAE(torch.randn(100, d, device=DEV), torch.randn(100, device=DEV) * 0.2 - 0.8),
           S.UntiedSAE(torch.randn(96, d, device=DEV) * 0.2, torch.randn(96, d, device=DEV), torch.zeros(96, device=DEV) - 0.3),
           S.TopKLearnedDict(torch.nn.functional.normalize(torch.randn(64, d, device=DEV), dim=-1), 8),
           S.TiedSAE(torch.randn(104, d, device=DEV), torch.randn(104, device=DEV) * 0.2 - 0.8)]
    x = torch.randn(64 * 200, d, device=DEV)
    a = MT.top_activating_fragments(lds, x, seed=3)
    b = MT.top_activating_fragments(lds, x, seed=3)
    for i, ld in enumerate(lds):
        one = MT.top_activating_fragments([ld], x, seed=3)[0]
        for k in a[i]:
            if torch.is_tensor(a[i][k]):
                assert torch.equal(a[i][k], b[i][k]), (i, k)              # repeatable
                assert torch.equal(a[i][k], one[k]), (i, k)               # grouping does not matter
        assert torch.equal(a[i]["top_values"], a[i]["top_activations"].amax(-1))
        ta = MT.evaluate_dicts([ld], x, segment=64)[0]["times_active"]
        assert torch.equal(a[i]["n_active_fragments"].float(), ta), i
    # another seed draws other random records; the top records do not depend on it
    c = MT.top_activating_fragments(lds[:1], x, seed=4)[0]
    assert torch.equal(c["top_fragments"], a[0]["top_fragments"])
    assert not torch.equal(c["random_fragments"], a[0]["random_fragments"])
    # without the per-token copies the lists are the same
    n = MT.top_activating_fragments(lds[:1], x, seed=3, return_activations=False)[0]
    assert n["top_activations"] is None and torch.equal(n["top_fragments"], a[0]["top_fragments"])
    assert torch.equal(n["random_fragments"], a[0]["random_fragments"])


def test_f16f8_range_rule():
    ld = S.TiedSAE(torch.randn(64, 64, device=DEV), torch.zeros(64, device=DEV))
    x = torch.randn(128, 64, device=DEV)
    x[5, 3] = 1e6
    with pytest.raises(ValueError, match="f16f8"):
        MT.top_activating_fragments([ld], x, arith="f16f8")
    MT.top_activating_fragments([ld], x)          # auto runs bf16x3


def test_fragment_plan_abi_error_paths():
    ld = S.TiedSAE(torch.randn(64, 64, device=DEV), torch.zeros(64, device=DEV))
    p = MT._FragmentPlan(("tied", 64, 64, False), [ld], 128, 32, 4, 4, 0, True, "bf16x3", DEV)
    lib = _lib.load()
    x = torch.randn(128, 64, device=DEV)
    f = lambda t: t.data_ptr()

    def call(B=128, L=32, frag0=0, nt=4, nr=4, tv=f(p.top_val), rk=f(p.rnd_key), na=f(p.n_active), ws=p.ws_ptr,
             nb=p.ws_bytes):
        rc = lib.sce_forward_fragments(p.plan, f(x), B, L, frag0, nt, nr, 0, tv, f(p.top_frag), f(p.top_act), rk,
                                       f(p.rnd_frag), f(p.rnd_act), na, ws, nb, p.stream)
        return rc, lib.sce_last_error().decode()

    try:
        assert call()[0] == 0
        assert call(B=0) == (-1, "forward_fragments: B = 0 outside [1, batch_max = 128]")
        assert call(B=160)[0] == -1
        assert call(L=48)[0] == -1 and "L = 48" in call(L=48)[1]
        assert call(B=96, L=64)[0] == -1 and "not a multiple" in call(B=96, L=64)[1]
        assert call(frag0=-1)[0] == -1
        assert call(nt=65)[0] == -1 and call(nr=-1)[0] == -1 and call(nt=0, nr=0)[0] == -1
        assert call(tv=None)[0] == -1 and call(rk=None)[0] == -1 and call(na=None)[0] == -1
        assert call(nt=0, tv=None)[0] == 0
        assert call(nb=p.ws_bytes - 1)[0] == -3 and "too small" in call(nb=p.ws_bytes - 1)[1]
        assert call(ws=p.ws_ptr + 256)[0] == -3 and "aligned" in call(ws=p.ws_ptr + 256)[1]
        torch.cuda.synchronize()
    finally:
        p.close()
