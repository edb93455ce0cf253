"""Dictionary evaluation on the H100 (libsce sce_forward_stats): every drop-in against the reference's own results
(golden fixture) under both arithmetics, evaluate_dicts at config-2 / config-5 / config-3 scale against the fp64 oracle
on the device, bitwise agreement with evaluate_batches, repeatability, the fp16 range rule and the ABI's error paths.

Tolerances, from the arithmetic's error model. Both arithmetics give each pre-activation z with an error below
~1e-6 |x| |w| (bf16x3: 2^-16 per split product; f16f8: 2^-14 on the cross terms), i.e. ~1e-6 relative on each c,
~4e-6 on c^4. The moments add these fp32 values in 32-row fp32 partials (relative error <= 32 * 2^-24 = 2e-6) and then
in fp64. So sums of powers carry <= ~1e-5 relative error; the bar is 1e-4 (of the largest value of the vector, so that
near-dead features are not judged on a relative scale). FVU is a ratio of two such sums: 1e-4 relative. Counts are
exact outside the kink window (DESIGN §5, |z| < max(1e-5, 1e-4 rms(z))): any difference is bounded by the number of
coefficients inside it. A top-k score inside the window around its row's k-th largest may be selected on the other
side and move its feature's sums by a whole value: at scale that value is added to the feature's bar. skew / kurtosis divide by var^1.5 / var^2 and are compared where var >= 1e-3 max(var)."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from oracle import eval_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
RTOL = 1e-4


def kink_window(z):
    return max(1e-5, 1e-4 * float(z.double().pow(2).mean().sqrt()))


def kink_coefficients(m, x, centred, rows=8192):
    """[N, n] mask of the coefficients whose pre-activation lies inside the kink window (top-k: also the scores next to
    the k-th largest, where the selection may take the other side)."""
    xs = O.center(m, x) if centred else x
    z = torch.cat([O.pre_activations(m, xs[i:i + rows]) for i in range(0, x.shape[0], rows)])
    w = kink_window(z)
    near = z.abs() < w
    if m["kind"] == "topk":
        near |= (z - torch.topk(z, int(m["sparsity"]), dim=-1).values[:, -1:]).abs() < w
    return near


def n_kink(m, x, centred):
    return int(kink_coefficients(m, x, centred).sum())


def selection_slack(m, x, centred, segment, rows=8192):
    """Top-k: per feature and power p, how far a selection on the other side of the k-th largest score can move the
    moment: the sum of |score|^p over the scores inside the window around their row's k-th largest, weighted as the
    streaming average weights a row (at most segment / rows of the last segment, over N). None for the SAE variants,
    whose near-kink coefficients are themselves below the window."""
    if m["kind"] != "topk":
        return None
    xs = O.center(m, x) if centred else x
    z = torch.cat([O.pre_activations(m, xs[i:i + rows]) for i in range(0, x.shape[0], rows)])
    near = (z - torch.topk(z, int(m["sparsity"]), dim=-1).values[:, -1:]).abs() < kink_window(z)
    N = x.shape[0]
    r_last = N - (-(-N // segment) - 1) * segment
    w = max(1.0, segment / r_last) / N
    a = torch.where(near, z.abs(), torch.zeros((), dtype=z.dtype, device=z.device))
    return [a.pow(p).sum(0) * w for p in (1, 2, 3, 4)]


def to_ld(m):
    f = lambda t: t.float().to(DEV)
    if m["kind"] == "tied":
        cen = tuple(f(m[k]) if k in m else None for k in ("center_trans", "center_rot", "center_scale"))
        return S.TiedSAE(f(m["encoder"]), f(m["encoder_bias"]), centering=cen, norm_encoder=True)
    if m["kind"] == "untied":
        return S.UntiedSAE(f(m["encoder"]), f(m["decoder"]), f(m["encoder_bias"]))
    return S.TopKLearnedDict(f(m["dict"]), int(m["sparsity"]))


def from_ld(ld):
    g = lambda t: t.double().to(DEV)
    if isinstance(ld, S.TopKLearnedDict):
        return {"kind": "topk", "dict": g(ld.dict), "sparsity": int(ld.sparsity)}
    if isinstance(ld, S.UntiedSAE):
        return {"kind": "untied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias), "decoder": g(ld.decoder)}
    return {"kind": "tied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias), "center_trans": g(ld.center_trans),
            "center_rot": g(ld.center_rot), "center_scale": g(ld.center_scale)}


def close(got, want, what, rtol=RTOL):
    got, want = got.double().to(want.device), want.double()
    scale = float(want.abs().max()) if want.numel() > 1 else abs(float(want))
    err = float((got - want).abs().max())
    assert err <= rtol * max(scale, 1e-30) + 1e-12, (what, err, scale)


def check_moments(got, want, kink, what, slack=None):
    """``slack``: selection_slack (top-k), added per feature to the bars of mean, var and m4; skew and kurtosis are
    then compared on the features without any."""
    times, mean, var, skew, kurt, m4 = got
    wt, wm, wv, ws, wk, w4 = want
    assert float((times.double().cpu() - wt.double().cpu()).abs().sum()) <= kink, (what, "times_active")
    if slack is None:
        for a, b, k in ((mean, wm, "mean"), (var, wv, "var"), (m4, w4, "m4")):
            close(a, b, (what, k))
        ok = wv >= 1e-3 * wv.max()
    else:
        s1, s2, _, s4 = slack
        sv = s2 + 2 * wm.abs() * s1 + s1 * s1
        for a, b, sl, k in ((mean, wm, s1, "mean"), (var, wv, sv, "var"), (m4, w4, s4, "m4")):
            err = (a.double().to(b.device) - b).abs()
            assert (err <= RTOL * b.abs().max() + sl + 1e-12).all(), (what, k, float((err - sl).max()))
        ok = (wv >= 1e-3 * wv.max()) & (s1 == 0)
    for a, b, k in ((skew, ws, "skew"), (kurt, wk, "kurtosis")):
        a, b = a.double().to(b.device)[ok], b[ok]
        assert ((a - b).abs() <= 1e-3 * b.abs() + 1e-6).all(), (what, k, ((a - b).abs() / b.abs()).max())


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_drop_ins_match_reference_golden(golden, arith):
    g = golden("dict_eval")
    for c in g["cases"]:
        m = {k: (v.double().to(DEV) if torch.is_tensor(v) else v) for k, v in g["dicts"][c["dict"]].items()}
        x = g["acts"][c["acts"]].to(DEV)
        raw = c["fn"] in ("batched_calc_feature_n_ever_active", "calc_moments_streaming")
        kink = n_kink(m, x.double(), centred=not raw)
        got = getattr(MT, c["fn"])(to_ld(g["dicts"][c["dict"]]), x, **c["kwargs"], arith=arith)
        want = c["out"]
        what = (c["fn"], c["dict"], c["acts"], c["kwargs"])
        if c["fn"] == "batched_calc_feature_n_ever_active":
            assert isinstance(got, int) and abs(got - want) <= kink, (what, got, want, kink)
        elif c["fn"] == "mean_nonzero_activations":
            assert got.device == x.device and got.shape == want.shape
            assert float((got.double().cpu() - want.double()).abs().sum()) * x.shape[0] <= kink + 1e-6, what
        elif c["fn"] == "calc_moments_streaming":
            assert len(got) == 6 and all(t.device == x.device and t.dtype == torch.float32 for t in got)
            check_moments(got, tuple(w.to(DEV) for w in want), kink, what)
        else:
            assert got.device == x.device and got.dim() == 0
            close(got, want.to(DEV), what)


def score_against_oracle(lds, x, segment=1000, threshold=10, arith="auto"):
    res = MT.evaluate_dicts(lds, x, segment=segment, threshold=threshold, arith=arith)
    xd = x.double()
    for i, (ld, r) in enumerate(zip(lds, res)):
        m = from_ld(ld)
        kink = n_kink(m, xd, centred=True)
        close(r["fvu"], O.fraction_variance_unexplained(m, xd), (i, "fvu"))
        counts = O.feature_counts(m, xd, centred=True)
        assert int((r["feature_counts"].long() - counts).abs().sum()) <= kink, (i, "counts", kink)
        assert int((r["n_ever_active"] - (counts > threshold).sum()).abs()) <= kink
        want = O.calc_moments_streaming(m, xd, segment, centred=True)
        check_moments([r[k] for k in ("times_active", "mean", "var", "skew", "kurtosis", "m4")], want, kink, i,
                      slack=selection_slack(m, xd, True, segment))
        print(f"dict {i}: fvu {float(r['fvu']):.5f} mean_l0 {float(r['mean_l0']):.2f} kink {kink}")
    return res


def synth(N, d, seed, half=True):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn(2048, d, generator=gen, device=DEV)
    feats /= feats.norm(dim=-1, keepdim=True)
    code = (torch.rand(N, 2048, generator=gen, device=DEV) < 0.01) * torch.rand(N, 2048, generator=gen, device=DEV)
    x = code @ feats + 0.05 * torch.randn(N, d, generator=gen, device=DEV)
    return x.half() if half else x


def test_config2_fresh_and_trained():
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(512, 4096, a) for a in torch.logspace(-4, -2, 16).tolist()]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    x = synth(65536 + 500, 512, 1)                                   # fp16 chunk format, partial last segment
    for steps in (0, 30):
        for s in range(steps):
            ens.step_batch(x[s * 2048:(s + 1) * 2048].float())
        lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in ens.unstack()]
        score_against_oracle(lds, x)


def test_config5_width():
    torch.manual_seed(2)
    ld = S.TiedSAE(torch.randn(32768, 2048, device=DEV), torch.randn(32768, device=DEV) * 0.1 - 0.3)
    score_against_oracle([ld], synth(10000, 2048, 3))


def test_config3_topk_shapes():
    torch.manual_seed(4)
    lds = [S.TopKEncoder.to_learned_dict(*S.TopKEncoder.init(768, n, k)) for n in (3072, 6144, 12288) for k in (16, 32, 64)]
    for ld in lds:
        ld.to_device(DEV)
    score_against_oracle(lds, synth(8192 + 300, 768, 5))


def test_centred_tied_with_nonuniform_scale_and_host_input():
    torch.manual_seed(6)
    d = 512
    cen = (torch.randn(d, device=DEV) * 0.1, torch.eye(d, device=DEV) + 0.05 * torch.randn(d, d, device=DEV) / d ** 0.5,
           torch.rand(d, device=DEV) * 1.5 + 0.5)
    ld = S.TiedSAE(torch.randn(2048, d, device=DEV), torch.randn(2048, device=DEV) * 0.05 - 0.1, centering=cen)
    x = synth(20000, d, 7, half=False).cpu()                          # host input: streamed
    res = score_against_oracle([ld, S.TiedSAE(ld.encoder, ld.encoder_bias)], x.to(DEV))
    host = MT.evaluate_dicts([ld], x)
    assert host[0]["fvu"].device.type == "cpu"
    assert torch.equal(host[0]["fvu"], res[0]["fvu"].cpu()) and torch.equal(host[0]["mean"], res[0]["mean"].cpu())


def test_segment_longer_than_an_engine_call():
    torch.manual_seed(8)
    ld = S.TiedSAE(torch.randn(1024, 256, device=DEV), torch.randn(1024, device=DEV) * 0.1 - 0.45)
    x = synth(50000, 256, 9)
    m, xd = from_ld(ld), x.double()
    kink = n_kink(m, xd, centred=False)
    for bs in (20000, 8193, 1000, 1):
        got = MT.calc_moments_streaming(ld, x, batch_size=bs)
        want = O.calc_moments_streaming(m, xd, bs) if bs > 1 else None
        if want is None:                                              # every row its own segment: row counts
            assert torch.equal(got[0].long(), O.feature_counts(m, xd)) or \
                float((got[0].double() - O.feature_counts(m, xd).double()).abs().sum()) <= kink
        else:
            check_moments(got, want, kink, bs)


@pytest.mark.parametrize("sig", ["tied", "untied", "masked"])
def test_exported_dicts_agree_bitwise_with_evaluate_batches(sig):
    torch.manual_seed(10)
    if sig == "tied":
        S_, models = S.FunctionalTiedSAE, [S.FunctionalTiedSAE.init(256, 1024, a) for a in (1e-3, 3e-3)]
    elif sig == "untied":
        S_, models = S.FunctionalSAE, [S.FunctionalSAE.init(256, 1024, a) for a in (1e-3, 3e-3)]
    else:
        S_, models = S.FunctionalMaskedSAE, [S.FunctionalMaskedSAE.init(256, k, 1024, 1e-3) for k in (1024, 300, 777)]
    ens = S.FunctionalEnsemble(models, S_, S.adam, {"lr": 1e-3}, device=DEV, arith="bf16x3")
    x = synth(24000, 256, 11, half=False)
    for s in range(10):
        ens.step_batch(x[s * 2000:(s + 1) * 2000])
    batches = [x[i:i + 8000] for i in range(0, 24000, 8000)]
    want = MT.evaluate_batches(ens, batches)
    got = MT.evaluate_dicts([(S_.to_learned_dict(p, b), {}) for p, b in ens.unstack()], x, segment=8000, arith="bf16x3")
    for m, r in enumerate(got):
        n = r["feature_counts"].shape[0]
        assert torch.equal(r["fvu"], want["fvu"][m]) and torch.equal(r["mean_l0"], want["mean_l0"][m]), m
        assert torch.equal(r["feature_counts"], want["feature_counts"][m, :n]), m


def test_repeated_calls_are_bitwise_equal():
    torch.manual_seed(12)
    lds = [S.TiedSAE(torch.randn(1000, 256, device=DEV), torch.zeros(1000, device=DEV)),
           S.TopKLearnedDict(torch.nn.functional.normalize(torch.randn(512, 256, device=DEV), dim=-1), 16)]
    x = synth(30000, 256, 13)
    a, b = MT.evaluate_dicts(lds, x), MT.evaluate_dicts(lds, x)
    for ra, rb in zip(a, b):
        for k, v in ra.items():
            assert (v == rb[k]) if not torch.is_tensor(v) else torch.equal(v, rb[k]), k


def test_out_of_fp16_range():
    torch.manual_seed(14)
    ld = S.TiedSAE(torch.randn(512, 128, device=DEV), torch.zeros(512, device=DEV))
    x = torch.randn(3000, 128, device=DEV) * 1e5
    assert x.abs().max() > 65504
    r = MT.evaluate_dicts([ld], x)[0]
    assert all(torch.isfinite(r[k]).all() for k in ("fvu", "mean", "m2", "m4"))
    close(r["fvu"], O.fraction_variance_unexplained(from_ld(ld), x.double()), "fvu")
    with pytest.raises(ValueError, match="fp16"):
        MT.evaluate_dicts([ld], x, arith="f16f8")


def test_stats_plan_abi_error_paths():
    ld = S.TiedSAE(torch.randn(64, 64, device=DEV), torch.zeros(64, device=DEV))
    p = MT._StatsPlan(("tied", 64, 64, False), [ld], 64, "bf16x3", DEV)
    lib = _lib.load()
    x = torch.randn(64, 64, device=DEV)
    f = lambda t: t.data_ptr()

    def call(B=64, seg=1, phase=0, losses=f(p.losses), sums=f(p.sums), open_=f(p.seg_open), ws=p.ws_ptr, nb=p.ws_bytes):
        rc = lib.sce_forward_stats(p.plan, f(x), B, seg, phase, None, losses, f(p.nnz), sums, f(p.seg_counts), open_,
                                   ws, nb, p.stream)
        return rc, lib.sce_last_error().decode()

    try:
        assert call()[0] == 0
        assert call(B=0) == (-1, "forward_stats: B = 0 outside [1, batch_max = 64]")
        assert call(B=65)[0] == -1
        assert call(seg=0)[0] == -1 and "seg = 0" in call(seg=0)[1]
        assert call(seg=4, phase=4)[0] == -1 and "seg_phase" in call(seg=4, phase=4)[1]
        assert call(losses=None)[0] == -1 and call(sums=None)[0] == -1
        assert call(seg=2, open_=None)[0] == -1 and "seg_open" in call(seg=2, open_=None)[1]
        assert call(nb=p.ws_bytes - 1)[0] == -3 and "too small" in call(nb=p.ws_bytes - 1)[1]
        assert call(ws=p.ws_ptr + 256)[0] == -3 and "aligned" in call(ws=p.ws_ptr + 256)[1]
        torch.cuda.synchronize()
    finally:
        p.close()
