"""Dictionary evaluation on the H100 (libsce sce_forward_stats): every drop-in against the reference's own results
(golden fixture) under both arithmetics, evaluate_dicts at config-2 / config-5 / config-3 scale against the fp64 oracle
on the device, bitwise agreement with evaluate_batches, repeatability, the fp16 range rule and the ABI's error paths.

Tolerances, per feature. Counts are exact outside the kink window (DESIGN §5, |z| < max(1e-5, 1e-4 rms(z))): feature
j's row count may differ by at most its own coefficients inside the window (kink_j), and its times_active by at most
its segments holding one. The moments (mean, var, m4, as the streaming average weights each row: 1 / (n_seg seg), the
last partial segment's rows seg / r_last times that) are held to oracle/eval_bounds.py's bound of the sums under the
same weights: e sum_b w_b p (c_b + e S_b)^(p-1) S_b + K sum_b w_b c_b^p, with e the code's element bar and S_b its
absolute-product scale, plus (SAE variants) sum over feature j's kink coefficients of w_b window^p, and the final fp32
rounding. A top-k score inside the window around its row's k-th largest may be selected on the other side and move its
feature's sums by a whole value: that value (selection_slack) is added to the feature's bound. The drop-ins' golden
results, which the reference computed in fp32, are held to the same per-feature bounds against the fp64 oracle on the
same activations, and to 1e-4 of the largest value against the golden values themselves. FVU is a ratio of two sums:
1e-4 relative. skew / kurtosis divide by var^1.5 / var^2 and are compared where var >= 1e-3 max(var)."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from engine_cases import DEV, as_oracle, synth
from oracle import eval_bounds as EB
from oracle import eval_oracle as O
from oracle import tile_bounds as T
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def kink_coefficients(m, x, centred, rows=8192):
    """[N, n] mask of the coefficients whose pre-activation lies inside the kink window (top-k: also the scores next to
    the k-th largest, where the selection may take the other side)."""
    xs = O.center(m, x) if centred else x
    z = torch.cat([O.pre_activations(m, xs[i:i + rows]) for i in range(0, x.shape[0], rows)])
    w = T.kink_window(z)
    near = z.abs() < w
    if m["kind"] == "topk":
        near |= (z - torch.topk(z, int(m["sparsity"]), dim=-1).values[:, -1:]).abs() < w
    return near


def n_kink(m, x, centred):
    return int(kink_coefficients(m, x, centred).sum())


def feature_bounds(m, x, centred, segment, arith="bf16x3", rows=8192):
    """Per feature of dictionary ``m`` on the fp64 activations ``x`` for a pass at ``segment`` (module docstring):
    ``kink`` [n] its coefficients inside the kink window, ``seg_kink`` [n] its segments holding one, and ``moments``
    [n, 4] the bound on its streaming means of c, c^2, c^3, c^4."""
    xs = O.center(m, x) if centred else x
    N, topk = x.shape[0], m["kind"] == "topk"
    near = kink_coefficients(m, x, centred, rows)
    z2 = sum(float(O.pre_activations(m, xs[i:i + rows]).pow(2).sum()) for i in range(0, N, rows))
    window = max(1e-5, 1e-4 * (z2 / (N * near.shape[1])) ** 0.5)
    n_seg = -(-N // segment)
    last = (n_seg - 1) * segment
    weight = torch.full((N,), 1.0 / (n_seg * segment), dtype=torch.float64, device=x.device)
    weight[last:] *= segment / (N - last)
    pad = torch.zeros(n_seg * segment - N, near.shape[1], dtype=torch.bool, device=x.device)
    seg_kink = torch.cat([near, pad]).reshape(n_seg, segment, -1).any(1).sum(0)
    if topk:
        e, K = T.TOPK_BARS[arith]["code"][1], EB.K_RUNNING
        W = torch.nn.functional.normalize(m["dict"], dim=-1)
    else:
        e, K = T.BARS[arith]["signed"]["code"][1], EB.K_TREE
        W = O.learned(m) if m["kind"] == "tied" else m["encoder"]
    bound = torch.zeros(near.shape[1], 4, dtype=torch.float64, device=x.device)
    for i in range(0, N, rows):
        xr, sr = x[i:i + rows], xs[i:i + rows]
        c = O.encode(m, sr)
        if topk:
            S_c = (sr.abs() @ W.abs().T) * (c != 0)
        else:
            cen = centred and "center_trans" in m
            Xabs = T.centered_input_scale(xr, m["center_trans"], m["center_rot"], m["center_scale"]) if cen else sr.abs()
            S_c = T.code_scale(Xabs, W, m["encoder_bias"])
        bound += EB.moment_bound(c, S_c, e, K, weight[i:i + rows])
        del c, S_c
    if not topk:
        wk = (weight[:, None] * near).sum(0)
        bound += torch.stack([wk * window ** p for p in (1, 2, 3, 4)], dim=-1)
    return {"kink": near.sum(0), "seg_kink": seg_kink, "moments": bound}


def check_counts(got, want, kink, what):
    """Per feature: |got_j - want_j| <= kink_j."""
    diff = (got.double().to(want.device) - want.double()).abs()
    bad = diff > kink.double().to(want.device)
    assert not bool(bad.any()), (what, int(bad.sum()), float((diff - kink.double().to(want.device)).max()))


def selection_slack(m, x, centred, segment, rows=8192):
    """Top-k: per feature and power p, how far a selection on the other side of the k-th largest score can move the
    moment: the sum of |score|^p over the scores inside the window around their row's k-th largest, weighted as the
    streaming average weights a row (at most segment / rows of the last segment, over N). None for the SAE variants,
    whose near-kink coefficients are themselves below the window."""
    if m["kind"] != "topk":
        return None
    xs = O.center(m, x) if centred else x
    z = torch.cat([O.pre_activations(m, xs[i:i + rows]) for i in range(0, x.shape[0], rows)])
    near = (z - torch.topk(z, int(m["sparsity"]), dim=-1).values[:, -1:]).abs() < T.kink_window(z)
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


def close(got, want, what, rtol=RTOL):
    got, want = got.double().to(want.device), want.double()
    scale = float(want.abs().max()) if want.numel() > 1 else abs(float(want))
    err = float((got - want).abs().max())
    assert err <= rtol * max(scale, 1e-30) + 1e-12, (what, err, scale)


def check_moments(got, want, fb, what, slack=None):
    """Per feature against the fp64 ``want`` (oracle.eval_oracle.calc_moments_streaming): times_active within its
    kink-holding segments, mean / var / m4 within feature_bounds' moment bound (``fb``), plus ``slack``
    (selection_slack, top-k) per feature; skew and kurtosis are then compared on the features without any."""
    times, mean, var, skew, kurt, m4 = (t.double().to(want[0].device) for t in got)
    wt, wm, wv, ws, wk, w4 = (t.double() for t in want)
    check_counts(times, wt, fb["seg_kink"], (what, "times_active"))
    b1, b2, _, b4 = fb["moments"].unbind(-1)
    if slack is not None:
        s1, s2, _, s4 = slack
        b1, b2, b4 = b1 + s1, b2 + s2, b4 + s4
    bv = b2 + 2 * wm.abs() * b1 + b1 * b1 + 2.0 ** -50 * (wv.abs() + 2 * wm * wm)
    for a, b, bd, k in ((mean, wm, b1, "mean"), (var, wv, bv, "var"), (m4, w4, b4, "m4")):
        err = (a - b).abs()
        lim = bd + 2.0 ** -23 * (b.abs() + bd)            # (+ the result's rounding to fp32)
        assert bool((err <= lim).all()), (what, k, int((err > lim).sum()), float((err / lim).max()))
    ok = wv >= 1e-3 * wv.max()
    if slack is not None:
        ok &= slack[0] == 0
    for a, b, k in ((skew, ws, "skew"), (kurt, wk, "kurtosis")):
        a, b = a[ok], b[ok]
        assert ((a - b).abs() <= 1e-3 * b.abs() + 1e-6).all(), (what, k, ((a - b).abs() / b.abs()).max())


def check_moments_golden(got, want, kink, what):
    """Against the reference's own fp32 results: mean, var and m4 within 1e-4 of the vector's largest value, and
    times_active within the kink coefficients in total."""
    times, mean, var, skew, kurt, m4 = got
    wt, wm, wv, ws, wk, w4 = want
    assert float((times.double().cpu() - wt.double().cpu()).abs().sum()) <= kink, (what, "times_active")
    for a, b, k in ((mean, wm, "mean"), (var, wv, "var"), (m4, w4, "m4")):
        close(a, b, (what, k))


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
            # both are counts / N rounded to fp32: back to whole counts, then per feature within its kink coefficients
            n_got, n_want = got.double() * x.shape[0], want.double().to(DEV) * x.shape[0]
            assert float((n_got - n_got.round()).abs().max()) < 1e-3 and float((n_want - n_want.round()).abs().max()) < 1e-3
            check_counts(n_got.round(), n_want.round(), kink_coefficients(m, x.double(), centred=True).sum(0), what)
        elif c["fn"] == "calc_moments_streaming":
            assert len(got) == 6 and all(t.device == x.device and t.dtype == torch.float32 for t in got)
            check_moments_golden(got, tuple(w.to(DEV) for w in want), kink, what)
            bs = c["kwargs"].get("batch_size", 1000)
            check_moments(got, O.calc_moments_streaming(m, x.double(), bs), feature_bounds(m, x.double(), False, bs, arith),
                          what, slack=selection_slack(m, x.double(), False, bs))
        else:
            assert got.device == x.device and got.dim() == 0
            close(got, want.to(DEV), what)


def score_against_oracle(lds, x, segment=1000, threshold=10, arith="auto"):
    res = MT.evaluate_dicts(lds, x, segment=segment, threshold=threshold, arith=arith)
    xd = x.double()
    for i, (ld, r) in enumerate(zip(lds, res)):
        m = as_oracle(ld)
        fb = feature_bounds(m, xd, True, segment, "bf16x3" if arith == "auto" else arith)
        kink = int(fb["kink"].sum())
        close(r["fvu"], O.fraction_variance_unexplained(m, xd), (i, "fvu"))
        counts = O.feature_counts(m, xd, centred=True)
        check_counts(r["feature_counts"], counts, fb["kink"], (i, "feature_counts"))
        assert int((r["n_ever_active"] - (counts > threshold).sum()).abs()) <= kink
        want = O.calc_moments_streaming(m, xd, segment, centred=True)
        check_moments([r[k] for k in ("times_active", "mean", "var", "skew", "kurtosis", "m4")], want, fb, i,
                      slack=selection_slack(m, xd, True, segment))
        print(f"dict {i}: fvu {float(r['fvu']):.5f} mean_l0 {float(r['mean_l0']):.2f} kink {kink}")
    return res


def test_config2_fresh_and_trained():
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(512, 4096, a) for a in torch.logspace(-4, -2, 16).tolist()]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    x = synth(65536 + 500, 512, 1).half()                            # fp16 chunk format, partial last segment
    for steps in (0, 30):
        for s in range(steps):
            ens.step_batch(x[s * 2048:(s + 1) * 2048].float())
        lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in ens.unstack()]
        score_against_oracle(lds, x)


def test_config5_width():
    torch.manual_seed(2)
    ld = S.TiedSAE(torch.randn(32768, 2048, device=DEV), torch.randn(32768, device=DEV) * 0.1 - 0.3)
    score_against_oracle([ld], synth(10000, 2048, 3).half())


def test_config3_topk_shapes():
    torch.manual_seed(4)
    lds = [S.TopKEncoder.to_learned_dict(*S.TopKEncoder.init(768, n, k)) for n in (3072, 6144, 12288) for k in (16, 32, 64)]
    for ld in lds:
        ld.to_device(DEV)
    score_against_oracle(lds, synth(8192 + 300, 768, 5).half())


def test_centred_tied_with_nonuniform_scale_and_host_input():
    torch.manual_seed(6)
    d = 512
    cen = (torch.randn(d, device=DEV) * 0.1, torch.eye(d, device=DEV) + 0.05 * torch.randn(d, d, device=DEV) / d ** 0.5,
           torch.rand(d, device=DEV) * 1.5 + 0.5)
    ld = S.TiedSAE(torch.randn(2048, d, device=DEV), torch.randn(2048, device=DEV) * 0.05 - 0.1, centering=cen)
    x = synth(20000, d, 7, False).cpu()                               # host input: streamed
    res = score_against_oracle([ld, S.TiedSAE(ld.encoder, ld.encoder_bias)], x.to(DEV))
    host = MT.evaluate_dicts([ld], x)
    assert host[0]["fvu"].device.type == "cpu"
    assert torch.equal(host[0]["fvu"], res[0]["fvu"].cpu()) and torch.equal(host[0]["mean"], res[0]["mean"].cpu())


def test_segment_longer_than_an_engine_call():
    torch.manual_seed(8)
    ld = S.TiedSAE(torch.randn(1024, 256, device=DEV), torch.randn(1024, device=DEV) * 0.1 - 0.45)
    x = synth(50000, 256, 9).half()
    m, xd = as_oracle(ld), x.double()
    for bs in (20000, 8193, 1000, 1):
        got = MT.calc_moments_streaming(ld, x, batch_size=bs)
        fb = feature_bounds(m, xd, False, bs)
        if bs == 1:                                                   # every row its own segment: row counts
            check_counts(got[0], O.feature_counts(m, xd), fb["kink"], (bs, "times_active"))
        else:
            check_moments(got, O.calc_moments_streaming(m, xd, bs), fb, bs)


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
    x = synth(24000, 256, 11, False)
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
    x = synth(30000, 256, 13).half()
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
    close(r["fvu"], O.fraction_variance_unexplained(as_oracle(ld), x.double()), "fvu")
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
