"""GPU tests of the round-2 additions around the step: the device-side health flag / range contract of the f16f8
arithmetic, language-model-style outlier dimensions, fused per-feature activation counts, host-batch prefetching and
the staged chunk upload."""
import warnings

import pytest
import torch

from engine_cases import clone_models, relnorm
from oracle import sae_oracle as O

pytestmark = pytest.mark.gpu

REL = 1e-4


def _tied(M, d, n, seed=0):
    import sparse_coding_b200 as S
    torch.manual_seed(seed)
    return [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2, 3e-3)[:M]]


def test_out_of_range_batch_never_poisons_the_parameters():
    """|x| beyond fp16 in an EXPLICIT f16f8 plan: the update of that step (and of every later one) is skipped on the
    device — parameters, Adam moments bit-identical to before — and step_batch raises at its health check."""
    import sparse_coding_b200 as S
    models = _tied(2, 64, 128)
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="f16f8",
                               health_check_every=4)
    gen = torch.Generator().manual_seed(1)
    good = torch.randn(96, 64, generator=gen)
    for _ in range(2):
        ens.step_batch(good.cuda())
    snap = {k: v.clone() for k, v in ens.params.items()}
    mu = ens.optim_states["mu"]["encoder"].clone()
    bad = good.clone()
    bad[7, 3] = 1.0e5
    ens.step_batch(bad.cuda())                  # step 3: flagged on the device, not yet looked at by the host
    ens.step_batch(good.cuda())                 # step 4: a good batch after the flag — still no update (sticky)
    for k in snap:
        assert torch.equal(ens.params[k], snap[k]), k
    assert torch.equal(ens.optim_states["mu"]["encoder"], mu)
    with pytest.raises(FloatingPointError, match="bf16x3"):
        ens.step_batch(good.cuda())             # 4 steps since the last check: the host reads the flag
    assert ens.health()[0] is True
    for k in snap:
        assert torch.equal(ens.params[k], snap[k]) and torch.isfinite(ens.params[k]).all()


def test_auto_plan_falls_back_to_bf16x3_and_retakes_the_step():
    """arith='auto' (f16f8 for this shape): an out-of-range FIRST batch switches the ensemble to bf16x3, the step is
    taken again on the new plan, and the result is exactly what an ensemble built with arith='bf16x3' computes."""
    import sparse_coding_b200 as S
    models = _tied(2, 64, 128, seed=3)
    gen = torch.Generator().manual_seed(2)
    X = 300.0 * torch.randn(128, 64, generator=gen)
    X[5, 9] = 9.0e4
    auto = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    ref = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="bf16x3")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        la, _ = auto.step_batch(X.cuda())
    assert any("bf16x3" in str(x.message) for x in w)
    lr_, _ = ref.step_batch(X.cuda())
    assert auto.resolved_arith() == "bf16x3" and auto._arith_fallback == "bf16x3"
    assert torch.equal(la["loss"], lr_["loss"]) and torch.isfinite(la["loss"]).all()
    assert torch.equal(auto.params["encoder"], ref.params["encoder"])
    la2, _ = auto.step_batch(X.cuda())           # and it keeps training
    lr2, _ = ref.step_batch(X.cuda())
    assert torch.equal(la2["loss"], lr2["loss"])
    assert auto.state_dict()["arith_fallback"] == "bf16x3"


def test_nonfinite_loss_is_caught_in_bf16x3_too():
    import sparse_coding_b200 as S
    models = _tied(1, 32, 64)
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="bf16x3")
    X = torch.randn(64, 32)
    X[0, 0] = float("nan")
    snap = ens.params["encoder"].clone()
    with pytest.raises(FloatingPointError, match="not finite"):
        ens.step_batch(X.cuda())                 # first step of the plan: checked immediately
    assert torch.equal(ens.params["encoder"], snap)


@pytest.mark.parametrize("d,n", [(512, 2048), (768, 3072)])
def test_lm_residual_outlier_dimensions(d, n):
    """Residual streams of Pythia / GPT-2 carry a few dimensions 100-1000x larger than the rest. The f16f8 planes are
    floating point, so their relative precision does not depend on the scale of a dimension: x_hat / loss / code stay
    within 1e-4 of the fp64 oracle and the pattern-pinned gradient within 2e-4, no fall-back needed."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    B = 1024
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    gen = torch.Generator().manual_seed(7)
    X = torch.randn(B, d, generator=gen)
    X[:, 17] *= 1000.0
    X[:, 130] *= 300.0
    X[:, d - 5] *= 100.0
    X[:, 200] += 40.0                              # a dimension with a large mean, as massive activations have
    X = X.half().float()
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    assert_arith = ens.resolved_arith()
    grads, (loss, aux) = ens.grads_batch(X.cuda())
    code = aux["c"].dense()
    _, _, x_hat = ens.forward_batch(X.cuda(), return_x_hat=True)
    assert ens.resolved_arith() == "f16f8" and assert_arith in (None, "f16f8")
    assert ens.health()[0] is False
    for i, (p, b) in enumerate(models):
        Xd = X.double().cuda()
        E, bias = p["encoder"].double().cuda(), p["encoder_bias"].double().cuda()
        f0 = O.tied_forward(E, bias, Xd, float(b["l1_alpha"]))
        w = max(1e-5, 1e-4 * float(f0["Z"].pow(2).mean().sqrt()))
        active = torch.where(f0["Z"].abs() < w, code[i] > 0, f0["Z"] > 0)
        f = O.tied_grads(E, bias, Xd, float(b["l1_alpha"]), active=active)
        assert relnorm(x_hat[i], f0["x_hat"]) <= REL, relnorm(x_hat[i], f0["x_hat"])
        assert relnorm(code[i], f0["c"]) <= REL
        assert abs(float(loss["loss"][i]) - float(f0["loss"])) <= REL * float(f0["loss"])
        assert relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 2e-4
        assert relnorm(grads["encoder_bias"][i], f["grads"]["encoder_bias"]) <= 2e-4


@pytest.mark.parametrize("kind", ["tied", "masked_tied", "topk"])
def test_active_counts_match_the_dense_code(kind):
    """sce_active_counts (column sums of the activity-mask plane) == (c != 0).sum(0) of the dense code, accumulated
    over batches of different sizes, including n not a multiple of 32 and a short last batch."""
    import sparse_coding_b200 as S
    torch.manual_seed(1)
    d, n = 64, 328
    if kind == "tied":
        models, sig = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)], S.FunctionalTiedSAE
    elif kind == "masked_tied":
        models, sig = [S.FunctionalMaskedTiedSAE.init(d, m, n, 1e-3) for m in (200, 328)], S.FunctionalMaskedTiedSAE
    else:
        models, sig = [S.TopKEncoder.init(d, n, k) for k in (5, 17)], S.TopKEncoder
    ens = S.FunctionalEnsemble(models, sig, S.adam, {"lr": 1e-3}, device="cuda", no_stacking=(kind == "topk"))
    gen = torch.Generator().manual_seed(2)
    counts, want = None, torch.zeros(2, n, dtype=torch.int64)
    for B in (300, 300, 77):
        X = torch.randn(B, d, generator=gen)
        _, aux = ens.forward_batch(X.cuda())
        want += (aux["c"].dense() != 0).sum(dim=1).cpu()
        counts = ens.active_counts(B, counts)
    assert torch.equal(counts.cpu().long(), want)
    assert counts.dtype == torch.int32 and tuple(counts.shape) == (2, n)
    if kind == "masked_tied":
        assert int(counts[0, 200:].sum()) == 0                # masked coefficients never fire


def test_evaluate_batches_streams_a_held_out_set():
    """metrics.evaluate_batches over ragged batches == the reference's metrics on the concatenated set computed from
    the exported LearnedDicts (FVU about the set's column means, mean L0, features active on more than 10 rows)."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.metrics import evaluate_batches
    torch.manual_seed(0)
    d, n = 64, 256
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 3e-2)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    gen = torch.Generator().manual_seed(3)
    for _ in range(40):
        ens.step_batch((torch.randn(256, d, generator=gen) + 0.3).cuda())
    parts = [torch.randn(b, d, generator=gen) + 0.3 for b in (500, 500, 123)]
    ev = evaluate_batches(ens, [p.pin_memory() for p in parts])
    held = torch.cat(parts)
    assert ev["rows"] == 1123
    for i, (p, b) in enumerate(ens.unstack(device="cpu")):
        ld = S.FunctionalTiedSAE.to_learned_dict(p, b)
        c = ld.encode(ld.center(held))
        assert abs(float(ev["fvu"][i]) - float(O.fvu(held, ld.predict(held)))) <= 2e-4 * float(ev["fvu"][i]) + 1e-6
        assert abs(float(ev["mean_l0"][i]) - float((c != 0).float().sum(-1).mean())) <= 0.02
        assert abs(int(ev["n_ever_active"][i]) - int(((c != 0).sum(0) > 10).sum())) <= 1
        freq = (c != 0).float().mean(0)
        assert float((ev["feature_frequency"][i].cpu() - freq).abs().max()) <= 2.5 / 1123


def test_refresh_recopies_engine_side_buffers():
    """Editing a buffer the engine keeps a converted copy of (bool coef_mask -> uint8) takes effect after refresh()."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    d, n = 32, 64
    models = [S.FunctionalMaskedTiedSAE.init(d, 48, n, 1e-3)]
    ens = S.FunctionalEnsemble(models, S.FunctionalMaskedTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    X = torch.randn(128, d).cuda()
    _, aux = ens.forward_batch(X)
    assert int((aux["c"].dense()[0, :, 48:] != 0).sum()) == 0
    ens.buffers["coef_mask"][0, 48:56] = False            # open eight more coefficients
    ens.refresh()
    _, aux = ens.forward_batch(X)
    c = aux["c"].dense()[0]
    assert int((c[:, 48:56] != 0).sum()) > 0 and int((c[:, 56:] != 0).sum()) == 0


def test_host_batch_prefetcher_feeds_identical_steps():
    """HostBatchPrefetcher (side-stream H2D of batch i+1 during step i) == stepping on the same batches directly."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import HostBatchPrefetcher
    models = _tied(2, 64, 128, seed=5)
    gen = torch.Generator().manual_seed(6)
    host = [torch.randn(200 if i != 4 else 77, 64, generator=gen).pin_memory() for i in range(7)]
    a = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    b = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    la = [a.step_batch(x.cuda())[0]["loss"].cpu() for x in host]
    lb = [b.step_batch(x)[0]["loss"].cpu() for x in HostBatchPrefetcher(host, "cuda")]
    assert len(lb) == 7 and all(torch.equal(p, q) for p, q in zip(la, lb))
    assert torch.equal(a.params["encoder"], b.params["encoder"])


def test_staged_upload_is_bit_exact():
    from sparse_coding_b200.train_loop import _to_device_staged
    t = torch.randn(3001, 257).half()                     # pageable, odd sizes, several staging pieces
    out = _to_device_staged(t, torch.device("cuda"), piece_bytes=256 << 10)
    assert torch.equal(out.cpu(), t)
    small = torch.randn(10, 8)
    assert torch.equal(_to_device_staged(small, torch.device("cuda")).cpu(), small)


def test_chunk_streamer_ring_of_pinned_pieces(tmp_path):
    """ChunkStreamer moves a chunk through a small ring of pinned pieces; with pieces much smaller than the chunk
    (ring reused many times, ragged last piece) the device copy is bit-exact and chunks arrive in order."""
    from sparse_coding_b200.train_loop import ChunkStreamer
    gen = torch.Generator().manual_seed(0)
    chunks = [torch.randn(1000 + 37 * i, 96, generator=gen).half() for i in range(3)]
    for i, c in enumerate(chunks):
        torch.save(c, tmp_path / f"{i}.pt")
    st = ChunkStreamer(str(tmp_path), [2, 0, 1, 0], "cuda")
    st.PIECE_BYTES = 10_000                                   # 20+ pieces per chunk through a ring of 4
    seen = []
    for idx, dev in st:
        assert torch.equal(dev.cpu(), chunks[idx])
        seen.append(idx)
    assert seen == [2, 0, 1, 0] and len(st.stage_seconds) == 4
