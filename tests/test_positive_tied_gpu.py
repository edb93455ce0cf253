"""FunctionalPositiveTiedSAE in the engine (a tied SAE on max(E, 0), trained on x + 0.18 with bias decay), under both
operand arithmetics: the reference's recorded gradients, trajectories against the restated reference step, the
reference's catalogue shape against the fp64 oracle, training quality, and the run properties (graph replay,
repeatability, resume, range guard, similarity of the exports).

Pre-activations within the engine's rounding of the ReLU kink (|z| < kink_window) may land on either side; gradient
checks pin those coefficients to the engine's side, as tests/test_engine_gpu.py does. A dictionary row with no positive
entry is normalised by the 1e-8 floor, so its gradient is dW / 1e-8: it is checked on its own, relative to its own
norm, so that it does not hide the error of the other rows."""
import ctypes as C

import numpy as np
import pytest
import torch

from engine_cases import clone_models, relnorm
from oracle import positive_tied_oracle as PT
from oracle import sae_oracle as O
from oracle.tile_bounds import kink_window

pytestmark = pytest.mark.gpu

REL = 1e-4
ARITHS = ["bf16x3", "f16f8"]
CASES = ["fresh", "signed_encoder", "f64", "ratio1"]
LOSS_KEYS = ("loss", "l_reconstruction", "l_l1", "l_bias_decay")
# the reference's run_positive sweep (big_sweep_experiments.py:1034-1092): Pythia-70m MLP width, dict ratio 1
CAT_D = CAT_N = CAT_B = 2048
CAT_L1 = [0.0] + np.logspace(-5, -3.5, 8).tolist()


def sig():
    import sparse_coding_b200 as S
    return S.FunctionalPositiveTiedSAE


def ensemble(models, lr=1e-3, **kw):
    import sparse_coding_b200 as S
    kw.setdefault("device", "cuda")
    return S.FunctionalEnsemble(clone_models(models), sig(), S.adam, {"lr": lr}, **kw)


def fixture_models(fx):
    M = fx["params"]["encoder"].shape[0]
    return [({k: v[i].float().clone() for k, v in fx["params"].items()},
             {k: v[i].float().clone() for k, v in fx["buffers"].items()}) for i in range(M)]


def mlp_data(B, d, seed, n_feat=4096):
    """fp16-representable MLP-like activations: GELU of a sparse mixture plus noise (the smallest value is about -0.17,
    as for GELU outputs)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    feats = torch.randn(n_feat, d, generator=gen, device="cuda")
    feats /= feats.norm(dim=-1, keepdim=True)
    codes = (torch.rand(B, n_feat, generator=gen, device="cuda") < 0.005).float() * \
        torch.rand(B, n_feat, generator=gen, device="cuda")
    z = 3.0 * codes @ feats + 0.5 * torch.randn(B, d, generator=gen, device="cuda")
    return torch.nn.functional.gelu(z).half().float()


def catalogue_models(seed):
    torch.manual_seed(seed)
    return [sig().init(CAT_D, CAT_N, a, 0.01) for a in CAT_L1]


def check_grad_rows(got, ref, E, tol=2e-4, what=""):
    """Encoder gradients: the rows with a positive entry together, each row without one (gradient dW / 1e-8) alone."""
    zero = (E <= 0).all(-1)
    assert relnorm(got[~zero], ref[~zero]) <= tol, (what, relnorm(got[~zero], ref[~zero]))
    for r in torch.nonzero(zero).flatten().tolist():
        assert relnorm(got[r], ref[r]) <= tol, (what, r, relnorm(got[r], ref[r]))


def check_against_oracle(ens, X, expand_dims=True, near_frac=None):
    """grads_batch / forward_batch of every model against the fp64 oracle (on X's device), with near-kink coefficients
    pinned to the engine's side. x_hat is compared in the shifted space the engine writes it in. Returns the per-model
    pinned oracle results."""
    grads, (loss, aux) = ens.grads_batch(X, expand_dims=expand_dims)
    code = aux["c"].dense()
    _, _, x_hat = ens.forward_batch(X, expand_dims=expand_dims, return_x_hat=True)
    out = []
    for m in range(ens.n_models):
        P = {k: v[m].double() for k, v in ens.params.items()}
        Xm = (X if expand_dims else X[m]).double()
        alpha, bd = float(ens.buffers["l1_alpha"][m]), float(ens.buffers["bias_decay"][m])
        f0 = O.tied_forward(P["encoder"].clamp(min=0.0), P["encoder_bias"], Xm + PT.SHIFT, alpha, bd)
        Z = f0["Z"]
        near = Z.abs() < kink_window(Z)
        assert int(((code[m] > 0) != (Z > 0))[~near].sum()) == 0, m   # nothing outside the window on the wrong side
        if near_frac is not None:
            assert int(near.sum()) <= near_frac * Z.numel(), (m, int(near.sum()))
        f = PT.positive_tied_grads(P["encoder"], P["encoder_bias"], Xm, alpha, bd,
                                   active=torch.where(near, code[m] > 0, Z > 0))
        for k in LOSS_KEYS:
            v = float(f0[k])
            assert abs(float(loss[k][m]) - v) <= REL * abs(v) + 1e-12, (m, k, float(loss[k][m]), v)
        assert relnorm(code[m], f0["c"]) <= REL, (m, relnorm(code[m], f0["c"]))
        assert relnorm(x_hat[m], f0["x_hat"]) <= REL, (m, relnorm(x_hat[m], f0["x_hat"]))
        check_grad_rows(grads["encoder"][m], f["grads"]["encoder"], P["encoder"], what=m)
        assert relnorm(grads["encoder_bias"][m], f["grads"]["encoder_bias"]) <= 2e-4, m
        out.append(f)
    return grads, loss, out


@pytest.mark.parametrize("per_model", [False, True])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("name", CASES)
def test_golden(golden, name, arith, per_model):
    """The reference's recorded losses, code and gradients; a batch shared by the models and per-model batches."""
    fx = golden("positive_tied")[name]
    ens = ensemble(fixture_models(fx), arith=arith)
    X = fx["batch"].float().cuda()
    M = ens.n_models
    Xin = X.expand(M, *X.shape).contiguous() if per_model else X
    grads, loss, fs = check_against_oracle(ens, Xin, expand_dims=not per_model)
    assert ens.resolved_arith() == arith
    assert set(loss) == set(LOSS_KEYS)
    for k, ref in fx["loss_data"].items():
        assert torch.allclose(loss[k].cpu().double(), ref.double(), rtol=REL, atol=1e-9), (k, loss[k], ref)
    for m, f in enumerate(fs):
        near = int((f["Z"].abs() < kink_window(f["Z"])).sum())
        E = fx["params"]["encoder"][m]
        if near == 0:   # only a pinned near-kink coefficient excuses a miss
            check_grad_rows(grads["encoder"][m].cpu(), fx["grads"]["encoder"][m], E, what=(name, m))
            assert relnorm(grads["encoder_bias"][m].cpu(), fx["grads"]["encoder_bias"][m]) <= 2e-4, (name, m)
        if name == "signed_encoder":   # straight-through: the negative entries get the reference's gradient
            neg = E < 0
            assert float(grads["encoder"][m].cpu()[neg].abs().max()) > 0


def _trajectory_models(M, d, n, seed):
    torch.manual_seed(seed)
    return [sig().init(d, n, a, bd) for a, bd in zip(torch.logspace(-4, -2, M).tolist(), (0.0, 0.01, 0.01))]


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("mode", ["frozen_t1", "standard"])
def test_trajectory_matches_ref_port(arith, mode):
    """30 Adam steps against RefPortEnsemble (fp32) on identical batches at a launch-bound shape: under frozen_t1 the
    step replays as a CUDA graph, under standard it runs eagerly. Every tenth batch is short, after full ones left stale
    rows in the workspace. The learning rate drives encoder entries below zero, where only the straight-through
    gradient moves them, and the test checks that it did."""
    M, d, n, B = 3, 64, 256, 256
    lr = 3e-3
    models = _trajectory_models(M, d, n, 5)
    ens = ensemble(models, lr=lr, adam_count_mode=mode, arith=arith)
    ref = O.RefPortEnsemble(clone_models(models), PT.sig_loss_positive_tied, lr=lr, count_mode=mode)
    for step in range(30):
        X = mlp_data(B if step % 10 != 9 else 37, d, 100 + step).cpu()
        loss, _ = ens.step_batch(X.cuda())
        rloss, _ = ref.step_batch(X)
        assert set(loss) == set(rloss)
        for k in rloss:
            assert torch.allclose(loss[k].cpu(), rloss[k], rtol=1e-3, atol=1e-7), (step, k, loss[k], rloss[k])
    for k in ref.params:
        assert relnorm(ens.params[k], ref.params[k]) <= 2e-3, (k, relnorm(ens.params[k], ref.params[k]))
    neg = ens.params["encoder"] < 0
    assert int(neg.sum()) > 0.01 * neg.numel(), int(neg.sum())
    assert bool((ref.params["encoder"] < 0).any())


def _runtime_calls(fn):
    """Names of the CUDA runtime calls made while running fn(), from torch.profiler's CUDA activity trace."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


def test_launch_count_and_graph_replay():
    """The shift and the clamp add no launch to the tied step (a shared batch is split once, shifted on the way). At this
    launch-bound shape a frozen_t1 step is replayed as a CUDA graph from the third step on: the replay makes one
    cudaGraphLaunch and no kernel launches, holds every launch of the eager step, and trains like the eager steps of a
    standard-mode plan (whose bias correction moves, so it never replays) at step 1, where the two modes agree."""
    import sparse_coding_b200 as S
    M, d, n, B = 3, 64, 256, 256
    models = _trajectory_models(M, d, n, 7)
    ident = {"center_rot": torch.eye(d), "center_trans": torch.zeros(d), "center_scale": torch.ones(d)}
    tied = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, {**{k: v.clone() for k, v in b.items()}, **ident})
                                 for p, b in models], S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda",
                                arith="bf16x3")
    ens = ensemble(models, arith="bf16x3")
    X = mlp_data(B, d, 1)
    counts = []
    for e in (tied, ens):
        seen = []
        for _ in range(3):   # eager, eager (capture), replay
            e.step_batch(X)
            seen.append(e.gpu_launches_last_call())
        assert seen[0] == seen[2], seen
        counts.append(seen[2])
    assert counts[1] == counts[0], counts
    replay = _runtime_calls(lambda: ens.step_batch(X))
    assert any("cudaGraphLaunch" in c for c in replay), sorted(set(replay))
    assert not any("LaunchKernel" in c for c in replay), sorted(set(replay))
    eager = ensemble(models, arith="bf16x3", adam_count_mode="standard")
    for _ in range(2):
        eager.step_batch(X)
    calls = _runtime_calls(lambda: eager.step_batch(X))
    assert any("LaunchKernel" in c for c in calls) and not any("cudaGraphLaunch" in c for c in calls)
    # the shifted batch the graph reads is the one fed to this step: a replayed first step equals an eager one
    a, b = ensemble(models, arith="bf16x3"), ensemble(models, arith="bf16x3", adam_count_mode="standard")
    Xs = [mlp_data(B, d, 20 + s) for s in range(3)]
    for x in Xs[:2]:
        a.step_batch(x)
    b.params = {k: v.clone() for k, v in a.params.items()}   # (same parameters and moments before the step)
    b.optim_states = {k: {q: t.clone() for q, t in v.items()} for k, v in a.optim_states.items()}
    b._steps = 0
    b._destroy_plan()
    b._plan_key = None
    la, _ = a.step_batch(Xs[2])
    lb, _ = b.step_batch(Xs[2])
    for k in la:
        assert torch.equal(la[k], lb[k]), k
    for k in a.params:
        assert torch.equal(a.params[k], b.params[k]), k


@pytest.mark.parametrize("arith", ARITHS)
def test_catalogue_scale_against_fp64(arith):
    """The reference's run_positive shape (9 models, d = n = 2048, B = 2048, its L1 grid, bias decay 0.01) on MLP-like
    fp16 data, at initialisation and after 30 steps, against the fp64 oracle on the device; coefficients inside the kink
    window are bounded as in tests/test_scale_parity_gpu.py."""
    ens = ensemble(catalogue_models(0), arith=arith)
    X = mlp_data(CAT_B, CAT_D, 11)
    check_against_oracle(ens, X, near_frac=5e-4)
    for s in range(30):
        ens.step_batch(mlp_data(CAT_B, CAT_D, 100 + s))
    check_against_oracle(ens, X, near_frac=5e-4)


def _training_stats(params, buffers, held):
    """FVU of the training objective (x̂ - 0.18 against x), mean L0 and features ever active on `held`, per model."""
    out = []
    for m in range(params["encoder"].shape[0]):
        f = O.tied_forward(params["encoder"][m].double().clamp(min=0.0), params["encoder_bias"][m].double(),
                           held + PT.SHIFT, 0.0)
        out.append((float(O.fvu(held, f["x_hat"] - PT.SHIFT)), float((f["c"] > 0).double().sum(-1).mean()),
                    int(((f["c"] > 0).sum(0) > 0).sum())))
    return out


def test_quality_against_ref_port():
    """300 steps at the catalogue shape: FVU, mean L0 and features ever active on held-out data within 1 % of the fp32
    reference port's, trained on the same batches."""
    models = catalogue_models(1)
    ens = ensemble(models)
    ref = O.RefPortEnsemble([({k: v.cuda() for k, v in p.items()}, {k: v.cuda() for k, v in b.items()})
                             for p, b in clone_models(models)], PT.sig_loss_positive_tied, lr=1e-3)
    for s in range(300):
        X = mlp_data(CAT_B, CAT_D, 1000 + s)
        ens.step_batch(X)
        ref.step_batch(X)
    held = mlp_data(CAT_B, CAT_D, 7).double()
    got, want = _training_stats(ens.params, ens.buffers, held), _training_stats(ref.params, ref.buffers, held)
    for m, (g, w) in enumerate(zip(got, want)):
        print(f"model {m} (l1 {CAT_L1[m]:.2e}): engine fvu {g[0]:.5f} l0 {g[1]:.1f} alive {g[2]}, "
              f"ref port fvu {w[0]:.5f} l0 {w[1]:.1f} alive {w[2]}")
        for i in range(3):
            assert abs(g[i] - w[i]) <= 0.01 * abs(w[i]), (m, i, g, w)
    assert bool((ens.params["encoder"] < 0).any())


@pytest.mark.parametrize("arith", ARITHS)
def test_repeatable_and_resume(arith):
    """Two identical runs are bitwise equal; state_dict -> from_state resumes bitwise."""
    import sparse_coding_b200 as S
    M, d, n, B = 3, 256, 2048, 1024
    models = _trajectory_models(M, d, n, 9)
    data = [mlp_data(B, d, 50 + s) for s in range(8)]
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


def test_out_of_range_batch_skips_the_update():
    """A batch fp16 cannot hold: under f16f8 the update is skipped and raised; under auto the ensemble falls back to
    bf16x3 and takes the step."""
    M, d, n, B = 3, 64, 256, 128
    models = _trajectory_models(M, d, n, 11)
    X = mlp_data(B, d, 3).cpu()
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
    assert not torch.equal(auto.params["encoder"], before["encoder"].cuda())
    assert torch.isfinite(auto.params["encoder"]).all()


def test_similarity_of_exports_and_forward_only_refusal():
    """dictionary_similarity of the ensemble is bitwise that of its exported TiedSAEs (both the raw encoder, negative
    entries kept); the forward-only evaluation entry points refuse the plan."""
    from sparse_coding_b200 import _lib, metrics
    M, d, n, B = 3, 256, 1024, 1024
    ens = ensemble(_trajectory_models(M, d, n, 13), lr=1e-2)
    for s in range(10):
        ens.step_batch(mlp_data(B, d, 200 + s))
    assert bool((ens.params["encoder"] < 0).any())
    lds = [sig().to_learned_dict(p, b) for p, b in ens.unstack()]
    a, b = metrics.dictionary_similarity(ens), metrics.dictionary_similarity(lds)
    assert set(a) == set(b)
    for k in a:
        torch.testing.assert_close(a[k], b[k], rtol=0, atol=0, equal_nan=True)
    lib = _lib.load()
    X = mlp_data(B, d, 5)
    # (the refusal comes before any argument is read)
    assert lib.sce_forward_stats(ens._plan, X.data_ptr(), B, 1, 0, *([None] * 7), 0, None) == -1
    assert "encoder_nonneg" in lib.sce_last_error().decode()
    assert lib.sce_forward_fragments(ens._plan, X.data_ptr(), B, 32, 0, 4, 0, C.c_ulonglong(0), *([None] * 8), 0,
                                     None) == -1
    assert "encoder_nonneg" in lib.sce_last_error().decode()
