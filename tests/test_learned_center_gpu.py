"""FunctionalTiedCenteredSAE in the engine (a tied SAE on x - center, the centre a trained parameter), under both
operand arithmetics: the reference's recorded gradients, trajectories against the restated reference step, config 2's
size against the fp64 oracle, training quality, and the run properties (repeatability, resume, range guard, export).

The centre gradient d_center = sum_b g_b - db W is the difference of two terms that nearly cancel once the centre has
converged, so its error is measured relative to ||sum_b g_b|| + ||db W||. Pre-activations within the engine's rounding
of the ReLU kink (|z| < kink_window) may land on either side; gradient checks pin those coefficients to the engine's
side, as tests/test_engine_gpu.py does."""
import math

import pytest
import torch

from engine_cases import clone_models, relnorm, synth
from oracle import learned_center_oracle as LC
from oracle import sae_oracle as O
from oracle.tile_bounds import kink_window

pytestmark = pytest.mark.gpu

REL = 1e-4
ARITHS = ["bf16x3", "f16f8"]
CASES = ["three_models", "mean_offset", "f64", "zero_center"]


def sig():
    import sparse_coding_b200 as S
    return S.FunctionalTiedCenteredSAE


def ensemble(models, **kw):
    import sparse_coding_b200 as S
    kw.setdefault("device", "cuda")
    return S.FunctionalEnsemble(clone_models(models), sig(), S.adam, {"lr": 1e-3}, **kw)


def fixture_models(fx):
    M = fx["params"]["encoder"].shape[0]
    return [({k: v[i].float().clone() for k, v in fx["params"].items()},
             {k: v[i].float().clone() for k, v in fx["buffers"].items()}) for i in range(M)]


def center_err(got, f):
    """d_center error relative to the two terms it is the difference of."""
    scale = float(f["G"].sum(0).norm() + (f["grads"]["encoder_bias"] @ f["W"]).norm())
    return float((got.double() - f["grads"]["center"].to(got.device)).norm()) / scale


def check_against_oracle(ens, X, expand_dims=True, near_frac=None):
    """grads_batch / forward_batch of every model against the fp64 oracle (on X's device), with near-kink coefficients
    pinned to the engine's side. Returns the per-model pinned oracle results."""
    grads, (loss, aux) = ens.grads_batch(X, expand_dims=expand_dims)
    code = aux["c"].dense()
    _, _, x_hat = ens.forward_batch(X, expand_dims=expand_dims, return_x_hat=True)
    out = []
    for m in range(ens.n_models):
        P = {k: v[m].double() for k, v in ens.params.items()}
        Xm = (X if expand_dims else X[m]).double()
        alpha = float(ens.buffers["l1_alpha"][m])
        f0 = O.tied_forward(P["encoder"], P["encoder_bias"], Xm - P["center"], alpha)
        Z = f0["Z"]
        near = Z.abs() < kink_window(Z)
        assert int(((code[m] > 0) != (Z > 0))[~near].sum()) == 0, m   # nothing outside the window on the wrong side
        if near_frac is not None:
            assert int(near.sum()) <= near_frac * Z.numel(), (m, int(near.sum()))
        f = LC.tied_center_grads(P["encoder"], P["encoder_bias"], P["center"], Xm, alpha,
                                active=torch.where(near, code[m] > 0, Z > 0))
        ref_loss = {"loss": f0["l_reconstruction"] + f0["l_l1"], "l_reconstruction": f0["l_reconstruction"],
                    "l_l1": f0["l_l1"]}
        for k, v in ref_loss.items():
            assert abs(float(loss[k][m]) - float(v)) <= REL * abs(float(v)), (m, k, float(loss[k][m]), float(v))
        assert relnorm(code[m], f0["c"]) <= REL, (m, relnorm(code[m], f0["c"]))
        assert relnorm(x_hat[m], f0["x_hat"]) <= REL, (m, relnorm(x_hat[m], f0["x_hat"]))
        for k in ("encoder", "encoder_bias"):
            assert relnorm(grads[k][m], f["grads"][k]) <= 2e-4, (m, k, relnorm(grads[k][m], f["grads"][k]))
        assert center_err(grads["center"][m], f) <= 2e-4, (m, center_err(grads["center"][m], f))
        out.append(f)
    return grads, loss, out


@pytest.mark.parametrize("per_model", [False, True])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("name", CASES)
def test_golden(golden, name, arith, per_model):
    """The reference's recorded losses, code and gradients; a batch shared by the models and per-model batches."""
    fx = golden("tied_learned_center")[name]
    ens = ensemble(fixture_models(fx), arith=arith)
    X = fx["batch"].float().cuda()
    M = ens.n_models
    Xin = X.expand(M, *X.shape).contiguous() if per_model else X
    grads, loss, fs = check_against_oracle(ens, Xin, expand_dims=not per_model)
    assert ens.resolved_arith() == arith
    for k, ref in fx["loss_data"].items():
        assert torch.allclose(loss[k].cpu().double(), ref.double(), rtol=REL, atol=1e-9), (k, loss[k], ref)
    for m, f in enumerate(fs):
        near = int((f["Z"].abs() < kink_window(f["Z"])).sum())
        for k in ("encoder", "encoder_bias"):
            err = relnorm(grads[k][m].cpu(), fx["grads"][k][m])
            assert err <= 2e-4 or near > 0, (k, m, err)   # only a pinned near-kink coefficient excuses a miss
        assert center_err(grads["center"][m], {**f, "grads": {**f["grads"], "center": fx["grads"]["center"][m].double()}}) <= 2e-4
    if name == "zero_center":
        for k in ("encoder", "encoder_bias"):
            assert relnorm(grads[k].cpu(), fx["tied_grads"][k]) <= 2e-4


def _trajectory_models(M, d, n, seed):
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed + 1)
    return [sig().init(d, n, a, center=0.1 * torch.randn(d, generator=gen))
            for a in torch.logspace(-4, -2, M).tolist()]


def _mix(B, d, gen, offset):
    feats = torch.randn(512, d, generator=gen)
    feats /= feats.norm(dim=-1, keepdim=True)
    codes = (torch.rand(B, 512, generator=gen) < 0.02).float() * torch.rand(B, 512, generator=gen)
    return codes @ feats + 0.01 * torch.randn(B, d, generator=gen) + offset


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("mode", ["frozen_t1", "standard"])
def test_trajectory_matches_ref_port(arith, mode):
    """30 Adam steps against RefPortEnsemble (fp32) on identical batches with a mean offset, at a launch-bound shape:
    under frozen_t1 the step replays as a CUDA graph, under standard it runs eagerly. Every tenth batch is short, after
    full ones left stale rows in the workspace."""
    M, d, n, B = 3, 64, 256, 256
    models = _trajectory_models(M, d, n, 5)
    ens = ensemble(models, adam_count_mode=mode, arith=arith)
    ref = O.RefPortEnsemble(clone_models(models), LC.sig_loss_tied_learned_center, lr=1e-3, count_mode=mode)
    gen = torch.Generator().manual_seed(6)
    offset = 0.5 * torch.randn(d, generator=gen)
    for step in range(30):
        X = _mix(B if step % 10 != 9 else 37, d, gen, offset)
        loss, _ = ens.step_batch(X.cuda())
        rloss, _ = ref.step_batch(X)
        for k in rloss:
            assert torch.allclose(loss[k].cpu(), rloss[k], rtol=1e-3, atol=1e-7), (step, k, loss[k], rloss[k])
    for k in ref.params:
        assert relnorm(ens.params[k], ref.params[k]) <= 2e-3, (k, relnorm(ens.params[k], ref.params[k]))
    assert relnorm(ens.optim_states["mu"]["center"], ref.mu["center"]) <= 3e-3


def test_launch_count_and_graph_replay():
    """The step adds four launches to the tied step (centring, three centre-gradient kernels), replayed in the graph."""
    import sparse_coding_b200 as S
    M, d, n, B = 3, 64, 256, 256
    models = _trajectory_models(M, d, n, 7)
    ident = {"center_rot": torch.eye(d), "center_trans": torch.zeros(d), "center_scale": torch.ones(d)}
    tied = S.FunctionalEnsemble([({"encoder": p["encoder"].clone(), "encoder_bias": p["encoder_bias"].clone()},
                                  {"l1_alpha": b["l1_alpha"].clone(), **ident}) for p, b in models],
                                S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="bf16x3")
    ens = ensemble(models, arith="bf16x3")
    X = torch.randn(B, d).cuda()
    counts = []
    for e in (tied, ens):
        seen = []
        for _ in range(3):   # eager, eager (capture), replay
            e.step_batch(X)
            seen.append(e.gpu_launches_last_call())
        assert seen[0] == seen[2], seen   # the replayed graph holds every launch of the eager step
        counts.append(seen[2])
    # tied with a shared batch splits one batch; the learned centre splits M centred batches
    assert counts[1] == counts[0] + 4 + (M - 1), counts
    ens.forward_batch(X)
    grads, _ = ens.grads_batch(X)
    assert torch.isfinite(grads["center"]).all()


def _offset_data(B, d, seed, offset_scale=4.0):
    """fp16-representable sparse-mixture activations whose column mean lies several spreads from the origin."""
    x = synth(B, d, seed, fp16_values=False)
    mu = torch.randn(d, generator=torch.Generator().manual_seed(seed)).cuda()
    x = x + offset_scale * float(x.std()) * mu / float(mu.abs().mean())
    return x.half().float()


@pytest.mark.parametrize("arith", ARITHS)
def test_config2_scale_against_fp64(arith):
    """Config 2's size per model (d = 512, n = 4096, B = 8192; both ends of its L1 grid) on mean-offset fp16 data,
    full batch, at initialisation and after 30 steps, against the fp64 oracle on the device."""
    d, n, B = 512, 4096, 8192
    torch.manual_seed(0)
    models = [sig().init(d, n, a) for a in (1e-4, 1e-2)]
    ens = ensemble(models, arith=arith)
    X = _offset_data(B, d, 11)
    check_against_oracle(ens, X, near_frac=5e-4)
    for s in range(30):
        ens.step_batch(_offset_data(B, d, 100 + s))
    check_against_oracle(ens, X, near_frac=5e-4)


def test_quality_against_ref_port():
    """300 steps at d = 512, n = 4096, B = 8192 on data with a known mean offset: FVU and mean L0 of the exported
    dictionaries within 1 % of the fp32 reference port's on the same batches, and the learned centre where the reference
    port's is. Where it goes is the signature's own dynamics: with 8 times more features than dimensions, db W outweighs
    sum_b g at initialisation, and in these 300 steps neither centre closes on the data mean (|c - mean| / |mean| stays
    near 1 in both, also at L1 = 1e-2 and 3e-2)."""
    import sparse_coding_b200 as S
    d, n, B = 512, 4096, 8192
    torch.manual_seed(1)
    models = [sig().init(d, n, a) for a in (3e-4, 1e-3)]
    ens = ensemble(models)
    ref = O.RefPortEnsemble([({k: v.cuda() for k, v in p.items()}, {k: v.cuda() for k, v in b.items()})
                             for p, b in clone_models(models)], LC.sig_loss_tied_learned_center, lr=1e-3)
    for s in range(300):
        X = _offset_data(B, d, 1000 + s)
        ens.step_batch(X)
        ref.step_batch(X)
    held = _offset_data(B, d, 7)
    mean = held.mean(0)
    for m in range(2):
        lds = [sig().to_learned_dict({k: v[m] for k, v in P.items()}, {k: v[m] for k, v in Bf.items()})
               for P, Bf in ((ens.params, ens.buffers), (ref.params, ref.buffers))]
        fvu = [float(O.fvu(held, ld.predict(held))) for ld in lds]
        l0 = [float((ld.encode(ld.center(held)) != 0).float().sum(-1).mean()) for ld in lds]
        assert abs(fvu[0] - fvu[1]) <= 0.01 * fvu[1], (m, fvu)
        assert abs(l0[0] - l0[1]) <= 0.01 * l0[1], (m, l0)
        c, c_ref = ens.params["center"][m], ref.params["center"][m]   # both initialised at 0
        cos = lambda a, b: float(a @ b / (a.norm() * b.norm()))
        print(f"model {m}: fvu {fvu}, l0 {l0}, |c - mean| / |mean| engine {float((c - mean).norm() / mean.norm()):.4f} "
              f"ref {float((c_ref - mean).norm() / mean.norm()):.4f}, cos(c, mean) engine {cos(c, mean):.3f} ref "
              f"{cos(c_ref, mean):.3f}, cos(c, c_ref) {cos(c, c_ref):.4f}")
        assert cos(c, c_ref) > 0.99 and relnorm(c, c_ref) <= 0.1, m


@pytest.mark.parametrize("arith", ARITHS)
def test_repeatable_and_resume(arith):
    """Two identical runs are bitwise equal; state_dict -> from_state resumes bitwise."""
    import sparse_coding_b200 as S
    M, d, n, B = 2, 256, 2048, 1024
    models = _trajectory_models(M, d, n, 9)
    data = [_offset_data(B, d, 50 + s, 2.0) for s in range(8)]
    runs = []
    for _ in range(2):
        ens = ensemble(models, adam_count_mode="standard", arith=arith)
        for X in data:
            ens.step_batch(X)
        runs.append(ens)
    for k in runs[0].params:
        assert torch.equal(runs[0].params[k], runs[1].params[k]), k
        assert torch.equal(runs[0].optim_states["nu"][k], runs[1].optim_states["nu"][k]), k
    a = ensemble(models, adam_count_mode="standard", arith=arith)
    for X in data[:4]:
        a.step_batch(X)
    deep = lambda v: {k: deep(x) for k, x in v.items()} if isinstance(v, dict) else v.clone() if torch.is_tensor(v) else v
    b = S.FunctionalEnsemble.from_state(deep(a.state_dict()))
    for X in data[4:]:
        b.step_batch(X)
    for k in runs[0].params:
        assert torch.equal(b.params[k], runs[0].params[k]), k
    unstacked = b.unstack()
    assert torch.equal(unstacked[1][0]["center"], b.params["center"][1])


def test_out_of_range_batch_skips_the_update():
    """A batch fp16 cannot hold: under f16f8 the update of centre, encoder and bias is skipped and raised; under auto
    the ensemble falls back to bf16x3 and takes the step."""
    M, d, n, B = 2, 64, 256, 128
    models = _trajectory_models(M, d, n, 11)
    X = torch.randn(B, d)
    X[3, 5] = 1e6
    ens = ensemble(models, arith="f16f8")
    before = {k: v.clone() for k, v in ens.params.items()}
    with pytest.raises(FloatingPointError):
        ens.step_batch(X.cuda())
    for k in before:
        assert torch.equal(ens.params[k], before[k]), k
    auto = ensemble(models)
    with pytest.warns(RuntimeWarning):
        auto.step_batch(X.cuda())
    assert auto.resolved_arith() == "bf16x3"
    assert not torch.equal(auto.params["center"], before["center"])
    assert torch.isfinite(auto.params["center"]).all()


def test_exported_dicts_evaluate_like_the_ensemble():
    """metrics.evaluate_dicts on the exported TiedSAEs (residual in the raw space) against metrics.evaluate_batches on
    the ensemble (centred space): feature counts equal outside the kink window, FVU within 1e-5 relative."""
    import sparse_coding_b200 as S
    from sparse_coding_b200 import metrics
    M, d, n, B = 2, 256, 1024, 2048
    models = _trajectory_models(M, d, n, 13)
    ens = ensemble(models, arith="bf16x3")
    for s in range(5):
        ens.step_batch(_offset_data(B, d, 200 + s, 2.0))
    held = [_offset_data(B, d, 300 + s, 2.0) for s in range(2)]
    eb = metrics.evaluate_batches(ens, held)
    lds = [sig().to_learned_dict(p, b) for p, b in ens.unstack()]
    ed = S.evaluate_dicts(lds, torch.cat(held))
    allx = torch.cat(held).double()
    for m in range(M):
        fvu_d = float(ed[m]["fvu"]) if isinstance(ed, list) else float(ed["fvu"][m])
        assert abs(fvu_d - float(eb["fvu"][m])) <= 1e-5 * float(eb["fvu"][m]), (m, fvu_d, float(eb["fvu"][m]))
        P = {k: v[m].double() for k, v in ens.params.items()}
        Z = (allx - P["center"]) @ O.unit_rows(P["encoder"])[0].T + P["encoder_bias"]
        near = (Z.abs() < kink_window(Z)).sum(0)
        got = ed[m]["feature_counts"] if isinstance(ed, list) else ed["feature_counts"][m]
        diff = (got.cpu().long() - eb["feature_counts"][m].cpu().long()).abs()
        assert bool((diff <= near.cpu()).all()), m
