"""Every element of every Adam step output of the engine (the train tail of sce_step: center_grad_kernel,
dict_rows_kernel and bias_kernel in MODE_ADAM) against the fp64 step of oracle/adam_bounds.py, fed with the gradient the
engine itself reports.

Each checked step is: clone params, mu and nu; g = grads_batch(X) (with sce_read_center_grad for the learned centre);
step_batch(X); then every element of every parameter, mu and nu is held to its per-element bar against
adam_bounds.reference at the step number the count mode prescribes (1 under frozen_t1, steps taken + 1 under standard).
Every checked step also asserts:
  - from zero moments (a plan's first step), mu = fp32((1 - b1) g) and nu = fp32(fp32((1 - b2) g) g) exactly, whatever
    the FMA contraction (tests/test_adam_bounds_cpu.py): the step applied exactly the gradient grads_batch reports, so
    the fp64 tile bounds on that gradient (test_tile_bounds_gpu.py, test_topk_tile_bounds_gpu.py) carry over to the
    step. It would fail if the centre gradient ran after dict_rows_kernel<MODE_ADAM> rewrote the encoder, if the
    MODE_GRAD and MODE_ADAM instantiations of the row-norm Jacobian rounded differently, or if the f16f8 gradient scale
    2 / (B d) differed between them;
  - the learned centre's gradient read back after the step equals grads_batch's exactly;
  - the rows and biases of masked dictionaries beyond dict_size are bitwise unchanged, their moments exactly 0;
  - sce_get_step_count is the number of steps taken.

Cases: every signature (tied, tied with centring, untied, masked tied and untied, learned centre, positive tied, top-k
on the gather and on the dense decode path, each pinned by its launch count) under both arithmetics with a shared and
per-model batches at the ragged M = 4, d = 400, n = 1040, B = 4001, whose frozen_t1 step is replayed as a CUDA graph
(steps 1-4: the eager first step, the captured one and replays); B = 8001, which runs eagerly; config 2 at full size;
d = 4096 and 5120 (dict_rows_kernel's NV = 8 and 16 instantiations, the latter with a partial float4 tail); non-default
lr, betas, eps and an eps_root near the median of v-hat. Count paths: standard over t = 1-4, a run resumed through
state_dict / from_state with the count in ``steps`` or only in optim_states["count"], a plan rebuilt because the batch
grew, and the f16f8 -> bf16x3 rerun of arith="auto", which must equal an explicit-bf16x3 twin resumed from the
pre-step state bit for bit. Negative controls: a step counter one off, hyper-parameters other than the oracle's and
a frozen_t1 step checked as standard at t = 3 each fail the bars at most elements.

Worst ratio (error / bar) measured over every case, H100 SXM (80 GB HBM3, 700 W power limit):

  arith    p'      m'      v'
  bf16x3   0.999   0.974   0.958
  f16f8    0.999   0.971   0.959

p' comes this close to its bar because the last rounding, p - lr r, can cost half an ulp of p', which is u |p'| where
p' lies just above a power of two, and lr |r| is small next to |p'|. Each negative control fails its bar at every
element of the dictionary. The whole file runs in about 20 s on an H100.

The closed-form check at step 1 found that MODE_GRAD and MODE_ADAM of dict_rows_kernel contracted the row sums and
the row-norm Jacobian into FMAs differently in the instantiation for d <= 512 (one float4 per thread), so the step
applied a gradient a rounding away from the one grads_batch returned. Those sums, and the centre and bias gradients,
are now rounded explicitly, in the order the step's kernel was compiled to.
"""
import pytest
import torch

import engine_cases as EC
from oracle import adam_bounds as A
from oracle.plan_paths import gather_classes, launch_bound, launches

pytestmark = pytest.mark.gpu

ARITHS = EC.ARITHS
RAGGED, RAGGED_EAGER = EC.RAGGED, EC.RAGGED_EAGER
TOPK = {"topk_gather": (1, (3, 8, 5, 8)), "topk_dense": (0, (16, 33, 17, 40))}   # gather launches, k per model
SIGNATURES = EC.VARIANTS + list(TOPK)
OTHER_HYPER = {"lr": 3e-3, "betas": (0.8, 0.99), "eps": 1e-6}
WORST = {}   # (arith, output) -> worst ratio over the passing cases


def lib():
    import sparse_coding_b200 as S
    return S._lib.load()


def check_call(rc, name):
    import sparse_coding_b200 as S
    S._lib.check(rc, name)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    """Prints the worst ratio of each bar over the cases of this module that ran."""
    yield
    for arith in ARITHS:
        print(f"worst {arith:6s} " + " ".join(f"{o}' {WORST.get((arith, o), float('nan')):.3f}" for o in "pmv"))


def make(variant, arith, shape, seed=0, optim=None, **kw):
    """A fresh ensemble of `variant` at `shape` (M, d, n, B)."""
    import sparse_coding_b200 as S
    M, d, n, _ = shape
    optim = dict(optim or {"lr": 1e-3})
    if variant in TOPK:
        torch.manual_seed(seed)
        models = [S.TopKEncoder.init(d, n, k) for k in TOPK[variant][1]]
        return S.FunctionalEnsemble(models, S.TopKEncoder, S.adam, optim, device="cuda", arith=arith,
                                    no_stacking=True, **kw)
    models, sig = EC.make_models(variant, M, d, n, seed)
    return S.FunctionalEnsemble(models, sig, S.adam, optim, device="cuda", arith=arith, **kw)


def clone(tree):
    return {k: clone(v) if isinstance(v, dict) else v.clone() for k, v in tree.items()}


def snapshot(ens):
    """A state_dict of `ens` whose tensors are copies."""
    s = dict(ens.state_dict())
    for k in ("params", "buffers", "optim_states"):
        s[k] = clone(s[k])
    return s


def take_step(ens, X, per_model):
    """grads_batch, then step_batch, on X: (params, mu, nu before the step, gradient)."""
    before = (clone(ens.params), clone(ens.optim_states["mu"]), clone(ens.optim_states["nu"]))
    g, _ = ens.grads_batch(X, expand_dims=not per_model)
    ens.step_batch(X, expand_dims=not per_model)
    return before, g


def ratios(ens, before, g, t, hyper=None):
    """Per-element ratio tensors {(param, "p" | "m" | "v"): error / bar} of the step just taken against fp64 step t."""
    P0, M0, V0 = before
    out = {}
    for k in ens.params:
        ref = A.reference(P0[k], g[k], M0[k], V0[k], t, hyper or ens.optimizer)
        got = {"p": ens.params[k], "m": ens.optim_states["mu"][k], "v": ens.optim_states["nu"][k]}
        for o in ("p", "m", "v"):
            out[(k, o)] = A.ratios(got[o], ref[o], ref["bar_" + o])
        del ref
    return out


def bits(t):
    return t.contiguous().view(torch.int32)


def checked_step(ens, X, per_model, steps, tag, launches_expected=None):
    """One step on X after `steps` steps of `ens` (of this object's history), checked element by element."""
    before, g = take_step(ens, X, per_model)
    arith = ens.resolved_arith()
    P0, M0, V0 = before
    t = A.step_number(ens.adam_count_mode, steps)
    assert int(lib().sce_get_step_count(ens._plan)) == steps + 1, tag
    if launches_expected is not None:
        assert ens.gpu_launches_last_call() == launches_expected, tag
    h = A.fp32_hyper(ens.optimizer)
    mu, nu = ens.optim_states["mu"], ens.optim_states["nu"]
    if all(bool((M0[k] == 0).all()) and bool((V0[k] == 0).all()) for k in M0):
        for k in g:
            assert torch.equal(mu[k], g[k] * (1.0 - h["b1"])), (tag, k, "mu is not (1 - b1) g")
            assert torch.equal(nu[k], (g[k] * (1.0 - h["b2"])) * g[k]), (tag, k, "nu is not ((1 - b2) g) g")
    if "center" in ens.params:
        cg = torch.empty_like(ens.params["center"])
        check_call(lib().sce_read_center_grad(ens._plan, cg.data_ptr(), ens._stream()), "sce_read_center_grad")
        assert torch.equal(bits(cg), bits(g["center"])), (tag, "centre gradient of the step != grads_batch's")
    if "coef_mask" in ens.buffers:
        pad = ens.buffers["coef_mask"].bool()
        for k in ("encoder", "decoder", "encoder_bias"):
            if k in ens.params:
                assert torch.equal(bits(ens.params[k][pad]), bits(P0[k][pad])), (tag, k, "padding moved")
                assert bool((mu[k][pad] == 0).all()) and bool((nu[k][pad] == 0).all()), (tag, k, "padding moments")
    worst = {}
    for (k, o), r in ratios(ens, before, g, t).items():
        worst[(k, o)] = float(r.max())
        WORST[(arith, o)] = max(WORST.get((arith, o), 0.0), worst[(k, o)])
    print(f"{tag:48s} {arith:6s} t={t:<2d} " + " ".join(f"{k}.{o} {v:.2f}" for (k, o), v in worst.items()))
    for key, v in worst.items():
        assert v <= 1.0, (tag, t, key, v)
    return worst


def walk(ens, batches, per_model, tag, steps=0, launches_expected=None):
    for X in batches:
        checked_step(ens, X, per_model, steps, f"{tag} step {steps + 1}", launches_expected)
        steps += 1
    return steps


def batches(shape, per_model, seed, count, fp16_values=True):
    M, d, _, B = shape
    return [EC.batch(M, B, d, seed + s, per_model, fp16_values) for s in range(count)]


def topk_launches(variant, shape, per_model, arith):
    classes, ks = TOPK[variant]
    M, d, n, _ = shape
    assert gather_classes(d, n, ks) == classes, variant
    return launches("step", classes, M if per_model else 1, arith)


@pytest.mark.parametrize("per_model", [False, True], ids=["shared", "per_model"])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", SIGNATURES)
def test_every_signature_ragged_graph(variant, arith, per_model):
    """Steps 1-4 under frozen_t1 at the ragged shape: the eager first step, the captured second and two replays."""
    assert launch_bound(*RAGGED)
    ens = make(variant, arith, RAGGED)
    n_launch = topk_launches(variant, RAGGED, per_model, arith) if variant in TOPK else None
    walk(ens, batches(RAGGED, per_model, 10, 4, fp16_values=False), per_model,
         f"ragged {variant} {'per-model' if per_model else 'shared'}", launches_expected=n_launch)
    assert ens.resolved_arith() == arith


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied", "positive_tied"])
def test_eager_shape(variant, arith):
    """B = 8001: above the launch-bound rule, every step runs eagerly (under f16f8 with the native weight gradient)."""
    assert not launch_bound(*RAGGED_EAGER)
    walk(make(variant, arith, RAGGED_EAGER), batches(RAGGED_EAGER, False, 20, 2), False, f"eager {variant}")


@pytest.mark.parametrize("arith", ARITHS)
def test_config2_full_size(arith):
    shape = (16, 512, 4096, 8192)
    walk(make("tied", arith, shape, seed=2), batches(shape, False, 30, 2), False, "cfg2 tied 16 models")


@pytest.mark.parametrize("d", [4096, 5120])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied"])
def test_wide_rows(variant, arith, d):
    """dict_rows_kernel's NV = 8 (d = 4096) and NV = 16 (d = 5120: the last float4 slots of a row past d)."""
    shape = (2, d, 256, 512)
    walk(make(variant, arith, shape, seed=3), batches(shape, False, 40, 2), False, f"d={d} {variant}")


def median_v_hat(variant, arith, shape, X, per_model):
    """The median over the main dictionary of v-hat at t = 1, which is g^2."""
    ens = make(variant, arith, shape)
    g, _ = ens.grads_batch(X, expand_dims=not per_model)
    return float(g[ens._engine_sig.main].double().pow(2).median())


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied", "learned_center", "positive_tied", "topk_dense"])
def test_non_default_hyper_parameters(variant, arith):
    """lr = 3e-3, betas = (0.8, 0.99), eps = 1e-6 and eps_root near the median v-hat, standard counting over t = 1-3."""
    xs = batches(RAGGED, False, 50, 3)
    eps_root = median_v_hat(variant, arith, RAGGED, xs[0], False)
    ens = make(variant, arith, RAGGED, optim=dict(OTHER_HYPER, eps_root=eps_root), adam_count_mode="standard")
    walk(ens, xs, False, f"hyper {variant} eps_root {eps_root:.1e}")


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied", "learned_center"])
def test_standard_count(variant, arith):
    ens = make(variant, arith, RAGGED, adam_count_mode="standard")
    walk(ens, batches(RAGGED, False, 60, 4), False, f"standard {variant}")


@pytest.mark.parametrize("carrier", ["steps", "count"])
@pytest.mark.parametrize("arith", ARITHS)
def test_standard_resumed_from_state(arith, carrier):
    """state_dict -> from_state after two standard steps continues at t = 3, with the count in ``steps`` or, as a
    worker handed only the shared optimiser state sees it, in optim_states["count"] alone."""
    import sparse_coding_b200 as S
    xs = batches(RAGGED, False, 70, 4)
    ens = make("untied", arith, RAGGED, adam_count_mode="standard")
    walk(ens, xs[:2], False, "resume before")
    state = snapshot(ens)
    if carrier == "count":
        del state["steps"]
    walk(S.FunctionalEnsemble.from_state(state), xs[2:], False, f"resumed ({carrier})", steps=2)


@pytest.mark.parametrize("mode", ["frozen_t1", "standard"])
@pytest.mark.parametrize("arith", ARITHS)
def test_plan_rebuilt_for_a_larger_batch(arith, mode):
    """Two steps at B = 2000, then B = 4001: the plan is built anew and must continue the count."""
    M, d, n, _ = RAGGED
    ens = make("tied", arith, RAGGED, adam_count_mode=mode)
    steps = walk(ens, batches((M, d, n, 2000), False, 80, 2), False, f"small batch {mode}")
    key = ens._plan_key
    steps = walk(ens, batches(RAGGED, False, 90, 2), False, f"grown batch {mode}", steps=steps)
    assert ens._plan_key[0] == RAGGED[3] and key[0] == 2000


def test_auto_rerun_applies_one_update():
    """arith="auto" resolves to f16f8 here; a batch beyond the fp16 range makes the step skip its update on the device,
    the plan is rebuilt on bf16x3 and the batch stepped again: exactly one update at t = steps + 1, bit for bit what an
    explicit-bf16x3 ensemble resumed from the state before that step computes (itself checked element by element)."""
    import sparse_coding_b200 as S
    xs = batches(RAGGED, False, 100, 3)
    ens = make("tied", "auto", RAGGED, adam_count_mode="standard", health_check_every=1)
    walk(ens, xs[:2], False, "auto before")
    assert ens.resolved_arith() == "f16f8"
    X = xs[2].clone()
    X[7, 11] = 1.0e5
    state = snapshot(ens)
    with pytest.warns(RuntimeWarning, match="bf16x3"):
        ens.step_batch(X)
    assert ens.resolved_arith() == "bf16x3"
    assert int(lib().sce_get_step_count(ens._plan)) == 3 and ens._steps == 3
    assert all(bool((c == 3).all()) for c in ens.optim_states["count"].values())
    twin = S.FunctionalEnsemble.from_state(dict(state, arith="bf16x3", arith_fallback=None))
    walk(twin, [X], False, "explicit bf16x3 twin", steps=2)
    for tree in ("params", "mu", "nu"):
        a = ens.params if tree == "params" else ens.optim_states[tree]
        b = twin.params if tree == "params" else twin.optim_states[tree]
        for k in a:
            assert torch.equal(bits(a[k]), bits(b[k])), (tree, k)


def failing_share(r):
    return float((r > 1).double().mean())


@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_counter_one_off(arith):
    """A standard step whose counter was set one off (t = 3 run as step 2, t = 2 run as step 3) fails the p' bar at most
    elements of the dictionary."""
    xs = batches(RAGGED, False, 110, 3)
    ens = make("tied", arith, RAGGED, adam_count_mode="standard")
    walk(ens, xs[:1], False, "counter control")
    for i, (t, set_to) in enumerate(((2, 2), (3, 1))):
        check_call(lib().sce_set_step_count(ens._plan, set_to), "sce_set_step_count")
        before, g = take_step(ens, xs[1 + i], False)
        share = failing_share(ratios(ens, before, g, t)[("encoder", "p")])
        print(f"counter one off at t={t} {arith}: share of encoder elements failing the p' bar {share:.3f}")
        assert share > 0.5, (t, share)


@pytest.mark.parametrize("which", ["eps_root", "betas", "eps"])
@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_hyper_parameters(arith, which):
    """An ensemble built with a non-default eps_root, betas or eps, checked against an oracle given the defaults: the
    output the hyper-parameter moves fails its bar at most elements (betas: m' at t = 1; eps_root and eps: p')."""
    import sparse_coding_b200 as S
    xs = batches(RAGGED, False, 120, 1)
    value = {"eps_root": median_v_hat("tied", arith, RAGGED, xs[0], False), "betas": OTHER_HYPER["betas"],
             "eps": OTHER_HYPER["eps"]}[which]
    ens = make("tied", arith, RAGGED, optim={"lr": 1e-3, which: value}, adam_count_mode="standard")
    before, g = take_step(ens, xs[0], False)
    out = "m" if which == "betas" else "p"
    share = failing_share(ratios(ens, before, g, 1, hyper=S.optim.AdamConfig())[("encoder", out)])
    print(f"{which} {value} against the default oracle {arith}: share of encoder elements failing the {out}' bar "
          f"{share:.3f}")
    assert share > 0.5, share


@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_frozen_checked_as_standard(arith):
    """A frozen_t1 run's third step passes at t = 1 and fails the p' bar at t = 3 at most elements."""
    xs = batches(RAGGED, False, 130, 3)
    ens = make("tied", arith, RAGGED)
    walk(ens, xs[:2], False, "frozen control")
    before, g = take_step(ens, xs[2], False)
    r = ratios(ens, before, g, 1)
    assert max(float(v.max()) for v in r.values()) <= 1.0
    share = failing_share(ratios(ens, before, g, 3)[("encoder", "p")])
    print(f"frozen_t1 step 3 checked at t=3 {arith}: share of encoder elements failing the p' bar {share:.3f}")
    assert share > 0.5, share

